"""What a run must reproduce to equal the oracle, in one place — test infrastructure only.

Every parity test and campaign tool compares the product (device or host build, one rank or several) with the CPU oracle
through this module:

- outputs(sim, sc, run): everything a run computed that both the oracle and the product report, as a plain picklable dict.
- merge_ranks(per_rank): the global outputs of a sharded run, from the outputs of its ranks.
- assert_same(got, ref, with_hash=...): the comparison.
- run_against_oracle / run_ranks: harnesses that run a scenario and return its outputs.  ThreadComm: the host collectives of
  ranks that are threads of this process.
"""
import threading

import numpy as np

from emu_lib import emu_sim
from oracle_lib import oracle_sim

# Per-node outputs: a rank of a sharded run reports the nodes of its own shard.
PER_NODE = ("lamport_time", "lamport_time_u32", "records", "member_status", "status_ltime", "status_ltime_u32", "incarnation", "ml_state",
            "user_event_records", "event_time", "user_event_seen", "anomaly_flags")
# The agreement summary of stats() is taken over a rank's own shard; the other stats are run totals, all-reduced over the ranks.
SHARD_STATS = ("member_time", "intent_queue", "disagree_slots")


def outputs(sim, sc, run, *, records=True):
    """Everything a run of `sc` computed: `run` (the run_until_converged result), stats, trace rows, state hash, clocks, every slot's
    records and getters, and the user-event and injector outputs when the scenario has them.

    Some getters are collective in sharded runs, so every rank calls them in this one order.  The oracle's reference for a 32-bit
    getter is its 64-bit getter: a truncation in the product's compact path shows as a difference.  records=False leaves the raw
    records out (full-size runs, where the state hash covers every byte of them)."""
    wide = sim._prefix == "oracle_sim_"
    out = dict(run=run, stats=sim.stats(), trace=sim.tick_trace(), state_hash=sim.state_hash(), lamport_time=sim.lamport_time())
    out["lamport_time_u32"] = out["lamport_time"] if wide else sim.lamport_time_u32()
    per_slot = ["member_status", "status_ltime", "status_ltime_u32", "incarnation", "ml_state"]
    if records:
        per_slot.insert(0, "records")
    for k in per_slot:
        out[k] = []
    for s in range(sc.slots):
        for k in per_slot:
            out[k].append(out["status_ltime"][s] if wide and k == "status_ltime_u32" else getattr(sim, k)(s))
    if sc.user_events is not None:
        events = range(len(sc.user_events))
        out.update(user_event_records=sim.user_event_records(), user_event_stats=sim.user_event_stats(), event_time=sim.event_time(),
                   user_event_ltime=[sim.user_event_ltime(e) for e in events], user_event_seen=[sim.user_event_seen(e) for e in events])
    if sc.byzantine is not None:
        out.update(byzantine_stats=sim.byzantine_stats(), anomaly_flags=sim.anomaly_flags())
    return out


def merge_ranks(per_rank):
    """The outputs of a sharded run as one unsharded run reports them.  Per-node arrays are concatenated in rank order; every
    other output is global, and every rank must hold the same value."""
    out = {}
    for k, v in per_rank[0].items():
        vals = [r[k] for r in per_rank]
        if k in PER_NODE:
            out[k] = [np.concatenate(x) for x in zip(*vals)] if isinstance(v, list) else np.concatenate(vals)
            continue
        # Global on every rank: the convergence verdict, the trace rows and injector counters (all-reduced), the state hash (a sum
        # over every node) and the event times.  user_event_stats: event_time is the largest event clock a node of the shard holds,
        # so the global one is the maximum over the ranks.
        local = SHARD_STATS if k == "stats" else ("event_time",) if k == "user_event_stats" else ()
        glob = (lambda x: {s: y for s, y in x.items() if s not in local}) if local else (lambda x: x)
        for r, x in enumerate(vals):
            _same(k, glob(x), glob(v), True, f"rank {r} against rank 0")
        out[k] = dict(v, event_time=max(x["event_time"] for x in vals)) if k == "user_event_stats" else glob(v)
    return out


def _arrays(name, at, got, ref, what):
    assert got.shape == ref.shape, f"{what}: {name} has shape {got.shape}, oracle {ref.shape}"
    bad = np.nonzero(got != ref)[0]
    assert bad.size == 0, f"{what}: {name} first differs at {at} {bad[0]}: got {got[bad[0]]} oracle {ref[bad[0]]}"


def _same(k, got, ref, with_hash, what):
    if k == "trace":
        assert got.size == ref.size, f"{what}: {got.size} trace rows, oracle {ref.size}"
        for f in ref.dtype.names:
            if f != "hash" or with_hash:
                _arrays(f"trace field {f}", "tick", got[f], ref[f], what)
    elif k == "stats" and got.keys() != ref.keys():
        # a merged sharded run (merge_ranks) has no agreement summary
        assert set(ref) - set(got) == set(SHARD_STATS), (what, sorted(got), sorted(ref))
        assert got == {s: ref[s] for s in got}, (what, k, got, ref)
    elif isinstance(ref, list):
        assert len(got) == len(ref), (what, k, len(got), len(ref))
        for i, (g, r) in enumerate(zip(got, ref)):
            _same(f"{k}[{i}]", g, r, with_hash, what)
    elif isinstance(ref, np.ndarray):
        _arrays(k, "node", got, ref, what)
    else:
        assert got == ref, f"{what}: {k} differs: got {got} oracle {ref}"


def assert_same(got, ref, *, with_hash, what=""):
    """got equals ref (outputs() dicts) in every output.  The per-tick hash is compared only when the run had trace = 1."""
    assert got.keys() == ref.keys(), f"{what}: outputs on one side only: {sorted(got.keys() ^ ref.keys())}"
    for k in ref:
        _same(k, got[k], ref[k], with_hash, what)


def run_against_oracle(make_sim, sc, traces=(1, 0), world=1, **cfg):
    """Runs sc on the oracle (trace = 1) and with make_sim in each trace mode of `traces`; every run must equal the oracle's.
    world > 1 runs the host build sharded over that many ranks (run_ranks).  Returns the outputs of the last run."""
    assert world == 1 or make_sim is emu_sim
    o = sc.build(oracle_sim, trace=1, **cfg)
    ref = outputs(o, sc, o.run_until_converged(sc.max_ticks))
    got = None
    for trace in traces:
        if world > 1:
            got = run_ranks(sc, world, trace, **cfg)
        else:
            g = sc.build(make_sim, trace=trace, **cfg)
            got = outputs(g, sc, g.run_until_converged(sc.max_ticks))
            g.close()
        assert_same(got, ref, with_hash=bool(trace), what=f"{sc.name} world {world} trace={trace}")
    return got


# ---- ranks as threads of this process ----------------------------------------------------------------------------
class ThreadComm:
    """The host collectives of `world` ranks that are threads of this process (the hooks GossipSim.connect takes)."""

    def __init__(self, world):
        self.world = world
        self.bar = threading.Barrier(world)
        self.blobs = [None] * world
        self.acc = None
        self.lock = threading.Lock()

    def hooks(self, rank):
        def all_gather_bytes(b):
            self.blobs[rank] = b
            self.bar.wait()
            out = list(self.blobs)
            self.bar.wait()
            return out

        def barrier():
            self.bar.wait()

        def allreduce_u64(arr):
            with self.lock:
                if self.acc is None:
                    self.acc = arr.copy()
                else:
                    self.acc = self.acc + arr                       # u64 wrap-around sum
            self.bar.wait()
            arr[:] = self.acc
            self.bar.wait()
            if rank == 0:
                self.acc = None
            self.bar.wait()
        return all_gather_bytes, barrier, allreduce_u64


def run_ranks(sc, world, trace, **cfg):
    """Runs sc on the host build sharded over `world` ranks, each a thread of this process with its own handle (the "NVLink
    windows" are shared memory); returns the merged outputs.  The first error of any rank is raised here."""
    comm = ThreadComm(world)
    per_rank, errs = [None] * world, []

    def rank(r):
        try:
            g = sc.build(emu_sim, rank=r, world_size=world, trace=trace, **cfg)
            g.connect(*comm.hooks(r))
            per_rank[r] = outputs(g, sc, g.run_until_converged(sc.max_ticks))
            comm.bar.wait()                                         # no handle goes away while another rank still uses the windows
        except BaseException as e:                                  # noqa: BLE001 — surface it in the main thread
            errs.append(e)
            comm.bar.abort()
    th = [threading.Thread(target=rank, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(600)
    if errs:
        raise errs[0]
    return merge_ranks(per_rank)
