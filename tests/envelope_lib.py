"""Inputs from the edges of what the C ABI accepts, shared by tests/test_emu_envelope.py and tests/test_gpu_z_envelope.py —
test infrastructure only.

- irregular_graph: a CSR whose out-degrees differ (isolated nodes, degrees below and above the fan-out, hubs of thousands
  of edges, optionally self-loops and duplicate edges).  Such a topology takes the kernels' general row-offset path
  (row_ptr is loaded instead of computed from a uniform degree).
- tma_span_graph: the largest 256-node tile's CSR span exactly at the 48 KB stage of the TMA pipeline, or just over it.
- envelope_fuzz: scenarios.fuzz over the whole fan-out (1–8) and slot (1–16) range, on regular, small-world or irregular
  graphs.
- kernel_lines: the kernel and grid the library prints for each topology under SERFSIM_VERBOSE.
- product_run: a run's parity outputs (parity_lib.outputs) with the product-only getters beside them.
- run_jobs / grid_for: product runs / a handle's kernel and grid under a set of run-time switches, in this process (every handle reads
  the switches when it is created).
- run_isolated: product_run in a fresh process, for the host build's lane and CTA schedule (SERFSIM_EMU_SCHED), which the host build
  reads once per process.
"""
import contextlib
import os
import pickle
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import parity_lib as P                                                       # noqa: E402
from serf_b200 import scenarios                                              # noqa: E402
from serf_b200.scenarios import Scenario                                     # noqa: E402
from serf_b200.sim import Op, random_regular_graph, small_world_graph         # noqa: E402

TILE = 256
TMA_STAGE_BYTES = 48 * 1024          # the largest CSR span of a tile a TMA stage holds (serfsim_set_topology_csr)
ON_EMU = bool(os.environ.get("SERFSIM_GPU_TESTS_ON_EMU"))


def _rng(seed):
    return np.random.Generator(np.random.Philox(seed))


def _draw_peers(rng, n, deg):
    """For every node v, deg[v] uniform peers other than v."""
    src = np.repeat(np.arange(n, dtype=np.int64), deg)
    col = rng.integers(0, n - 1, size=src.size, dtype=np.int64)
    return col + (col >= src)


def irregular_graph(n, seed, mean_degree=8, zero_frac=0.05, low_frac=0.2, hubs=3, hub_degree=(1000, 4000),
                    self_loops=0.0, duplicates=0.0):
    """CSR (row_ptr uint64[n+1], col uint32) with per-node out-degrees from a wide distribution: `zero_frac` of the nodes
    have none, `low_frac` have 1–2 (below most fan-outs), the rest 1 … 2·mean_degree, and `hubs` nodes have hub_degree
    (drawn from the range; more edges than the graph has nodes means repeated peers).  self_loops / duplicates: the
    fraction of edges replaced by an edge to the node itself / by a copy of the row's previous edge (the ABI accepts both)."""
    assert n >= 2
    rng = _rng(seed)
    deg = rng.integers(1, 2 * mean_degree + 1, size=n)
    deg = np.where(rng.random(n) < low_frac, rng.integers(1, 3, size=n), deg)
    deg[rng.random(n) < zero_frac] = 0
    if hubs:
        hub_ids = rng.choice(n, size=min(hubs, n), replace=False)
        deg[hub_ids] = rng.integers(hub_degree[0], hub_degree[1] + 1, size=hub_ids.size)
    deg = np.minimum(deg, 65535)
    col = _draw_peers(rng, n, deg)
    row_ptr = np.zeros(n + 1, dtype=np.uint64)
    row_ptr[1:] = np.cumsum(deg)
    src = np.repeat(np.arange(n, dtype=np.int64), deg)
    if self_loops:
        m = rng.random(col.size) < self_loops
        col[m] = src[m]
    if duplicates:
        first = np.zeros(col.size, dtype=bool)
        first[row_ptr[:-1][deg > 0].astype(np.int64)] = True                  # the first edge of a row has no predecessor in it
        for i in np.nonzero((rng.random(col.size) < duplicates) & ~first)[0]:
            col[i] = col[i - 1]                                                # in order: a run of marked edges repeats one peer
    return row_ptr, col.astype(np.uint32)


def tma_span_graph(n, target_tile_bytes, degree=8, seed=5):
    """Every node has `degree` uniform peers except one node of the middle tile, whose degree makes that tile's CSR span
    target_tile_bytes / 4 edges.  The preceding tiles hold multiples of 4 edges, so the span's ends are 16-byte aligned and
    the span the library computes is exactly target_tile_bytes; target_tile_bytes = 48 KB + 4 is one edge over the stage."""
    assert target_tile_bytes % 4 == 0 and (TILE * degree) % 4 == 0
    tiles = (n + TILE - 1) // TILE
    assert tiles >= 3
    mid = tiles // 2
    want = target_tile_bytes // 4
    assert (mid + 1) * TILE <= n and want - (TILE - 1) * degree <= 65535
    deg = np.full(n, degree, dtype=np.int64)
    deg[mid * TILE + 17] = want - (TILE - 1) * degree
    rng = _rng(seed)
    col = _draw_peers(rng, n, deg)
    row_ptr = np.zeros(n + 1, dtype=np.uint64)
    row_ptr[1:] = np.cumsum(deg)
    return row_ptr, col.astype(np.uint32)


def max_tile_span_bytes(row_ptr):
    """The largest 16-byte-aligned CSR span of one 256-node tile, in bytes — what sizes the TMA stage."""
    rp = np.asarray(row_ptr, dtype=np.int64)
    b = np.arange(0, rp.size - 1, TILE)
    e = np.minimum(b + TILE, rp.size - 1)
    return int((((rp[e] + 3) & ~3) - (rp[b] & ~3)).max()) * 4


TOPOLOGIES = ("regular", "small_world", "irregular")


def envelope_fuzz(seed, n=None, topology=None, slots=None):
    """scenarios.fuzz with the whole parameter range of the ABI: fan-out 1–8, slots 1–16, and the topology drawn from a
    random regular graph, a small world and an irregular graph (or the one named by `topology`; `slots` fixes the slot count).
    The same seed gives the same scenario everywhere: every draw comes from Philox streams of the seed.  Irregular graphs get
    at most two hubs of at most 3000 edges, so a tile's CSR span (≤ 2·3000 + 256·24 edges) stays within a TMA stage."""
    rng = _rng(seed + 7_000_003)
    drawn = int(rng.integers(1, 17))
    sc = scenarios.fuzz(seed, n=n, slots=slots or drawn)
    kind = TOPOLOGIES[int(rng.integers(0, 3))]
    kind = topology or kind
    degree = int(sc.row_ptr[1])
    if kind == "small_world":
        sc.row_ptr, sc.col = small_world_graph(sc.n, max(2, degree // 2 * 2), 0.2, seed + 17)
    elif kind == "irregular":
        sc.row_ptr, sc.col = irregular_graph(sc.n, seed + 17, mean_degree=max(2, degree), hubs=int(rng.integers(0, 3)), hub_degree=(1000, 3000),
                                             self_loops=0.05 if rng.random() < 0.3 else 0.0,
                                             duplicates=0.05 if rng.random() < 0.3 else 0.0)
    else:
        sc.row_ptr, sc.col = random_regular_graph(sc.n, degree, seed + 17)
    sc.cfg["fanout"] = int(rng.integers(1, 9))
    sc.max_ticks = 300                                   # (isolated nodes that received mail keep the run from going quiet)
    sc.name = f"envelope_fuzz_{seed}_{kind}_f{sc.cfg['fanout']}_r{sc.slots}"
    sc.topology = kind
    return sc


# ---- studies ------------------------------------------------------------------------------------------------
# A node with no out-edges never drains what it has queued, so a run on an irregular graph whose isolated nodes receive mail
# never becomes quiescent: such runs stop at max_ticks on both sides (the comparison covers every tick up to there).
def leave_study(n, topo, fanout=4, seed=3, subject=3, max_ticks=400):
    return Scenario(f"leave_{n}", n, 1, topo, [subject], [(0, Op.LEAVE, subject, 0)], dict(fanout=fanout, seed=seed), max_ticks=max_ticks)


def crash_study(n, topo, fanout=4, seed=3, subject=3, short_timers=False, max_ticks=400):
    """One tracked subject crashes at tick 0.  Default timers are the memberlist LAN profile: suspicion timers run for many
    ticks in which views sleep and tiles are woken by the timer wheel.  short_timers: random_graph_fail's probing setup."""
    cfg = dict(fanout=fanout, seed=seed)
    if short_timers:
        cfg.update(suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)
    return Scenario(f"crash_{n}" + ("_short" if short_timers else "_lan"), n, 1, topo, [subject], [(0, Op.FAIL, subject, 0)], cfg,
                    max_ticks=max_ticks)


def crash_and_leave_study(n, topo, fanout=4, seed=3, slots=2, max_ticks=400):
    """Multi-slot: every subject leaves at tick 0 except the last, which crashes (dissemination_storm(with_fail=True) on `topo`)."""
    subjects = (np.arange(slots, dtype=np.int64) * max(1, n // slots) + 3).astype(np.uint32)
    ops = [(0, Op.LEAVE, int(s), 0) for s in subjects[:-1]] + [(0, Op.FAIL, int(subjects[-1]), 0)]
    return Scenario(f"crash_leave_{n}_r{slots}", n, slots, topo, subjects, ops, dict(fanout=fanout, seed=seed), max_ticks=max_ticks)


# ---- what the library reports -------------------------------------------------------------------------------
_KERNEL_RE = re.compile(r"tick kernel = (\w+) \(stage_col_bytes (\d+), grid (\d+)\)")


def kernel_lines(stderr_text):
    """[(kernel name, grid)] from the `tick kernel = …` lines SERFSIM_VERBOSE printed, one per topology set.  On the host build
    of the kernels (SERFSIM_GPU_TESTS_ON_EMU=1) the TMA pipeline is compiled out, whatever the line says: the name is "selected"
    there."""
    return [("selected" if ON_EMU else name, int(grid)) for name, _, grid in _KERNEL_RE.findall(stderr_text)]


def is_kernel(name, expected):
    return name == "selected" or name == expected


def tiles_per_cta(n, grid):
    tiles = (n + TILE - 1) // TILE
    return (tiles + grid - 1) // grid


def busy_ctas(n, grid):
    """CTAs that own at least one tile under the ceiling split (the others return after the tile scan)."""
    tiles = (n + TILE - 1) // TILE
    per = tiles_per_cta(n, grid)
    return (tiles + per - 1) // per


# ---- runs of the product -------------------------------------------------------------------------------------
def product_run(sim, sc):
    """Runs sim (built from sc) to convergence: {"out": its parity outputs, "view_kinds": the per-view kind counters, "launches":
    the kernel launches of the last step call}."""
    out = P.outputs(sim, sc, sim.run_until_converged(sc.max_ticks))
    return dict(out=out, view_kinds=sim.tick_view_kinds(), launches=sim.last_step_device_ms()[1])


@contextlib.contextmanager
def switches(env=None):
    """The run-time switches `env` and SERFSIM_VERBOSE=1 for the handles created inside.  On the host build of the kernels
    (SERFSIM_GPU_TESTS_ON_EMU=1) the device has 4 SMs unless SERFSIM_EMU_SMS says otherwise: 12 CTAs of the single-slot kernel at
    SERFSIM_GRIDMUL=1."""
    with pytest.MonkeyPatch.context() as mp:
        for k, v in (env or {}).items():
            mp.setenv(k, v)
        mp.setenv("SERFSIM_VERBOSE", "1")
        if ON_EMU and not os.environ.get("SERFSIM_EMU_SMS"):
            mp.setenv("SERFSIM_EMU_SMS", "4")
        yield


def run_jobs(jobs, capfd, env=None):
    """Run jobs — dict(sc=Scenario, trace=0/1, cfg={...}) — through the product library (the host build under
    SERFSIM_GPU_TESTS_ON_EMU=1) under the switches `env`.  Returns one product_run dict per job, with "kernel": (kernel name, grid)
    of the job's topology (kernel_lines, read from the captured stderr)."""
    from serf_b200 import GossipSim
    res = []
    with switches(env):
        for job in jobs:
            capfd.readouterr()
            sim = job["sc"].build(GossipSim, trace=job["trace"], **job.get("cfg", {}))
            r = product_run(sim, job["sc"])
            sim.close()
            lines = kernel_lines(capfd.readouterr().err)
            assert len(lines) == 1, lines                  # every job sets one topology
            res.append(dict(r, kernel=lines[0]))
    return res


def grid_for(factory, n, capfd, env=None):
    """(kernel name, grid) an n-node single-slot handle made by `factory` picks under the switches `env`."""
    with switches(env):
        capfd.readouterr()
        g = factory(n, 1)
        g.set_topology(np.arange(n + 1, dtype=np.uint64), ((np.arange(n) + 1) % n).astype(np.uint32))
        g.close()
        (line,) = kernel_lines(capfd.readouterr().err)
    return line


def _child(job_path, out_path):
    from emu_lib import emu_sim
    with open(job_path, "rb") as f:
        jobs = pickle.load(f)
    res = []
    for job in jobs:
        sc = job["sc"]
        g = sc.build(emu_sim, trace=job["trace"], **job.get("cfg", {}))
        res.append(product_run(g, sc))
        g.close()
    with open(out_path, "wb") as f:
        pickle.dump(res, f)


def run_isolated(jobs, env=None, timeout=1200):
    """Run jobs — dict(sc=Scenario, trace=0/1, cfg={...}) — through the host build of the kernels in a new Python process with `env`
    added to this one's.  The host build reads its lane and CTA schedule (SERFSIM_EMU_SCHED, tests/emu/emu_engine.cpp) once per
    process, so a run under another schedule needs a process of its own.  Returns one product_run dict per job."""
    e = dict(os.environ)
    e.update(env or {})
    with tempfile.TemporaryDirectory(prefix="serfsim_envelope_") as d:
        jp, op = os.path.join(d, "jobs.pkl"), os.path.join(d, "out.pkl")
        with open(jp, "wb") as f:
            pickle.dump(jobs, f)
        p = subprocess.run([sys.executable, os.path.abspath(__file__), jp, op], env=e, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
        assert p.returncode == 0, f"child run failed ({p.returncode}):\n{p.stderr[-4000:]}"
        with open(op, "rb") as f:
            return pickle.load(f)


if __name__ == "__main__":
    _child(sys.argv[1], sys.argv[2])
