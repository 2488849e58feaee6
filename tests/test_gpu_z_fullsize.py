"""Full-size parity against the (threaded) CPU oracle — BASELINE.json configs[2] and configs[4] at their stated sizes.

* configs[2] (SURVEY §8d item 3): 1 M-node Watts–Strogatz small world (k = 16, β = 0.1), 50 000 nodes fail / rejoin at random
  ticks in [0, 200), R = 8 tracked subjects sampled from the churn set, memberlist LAN timers, one GPU.
* configs[4] (SURVEY §8d item 5): 10 M-node random graph, 100 000 stale-record injectors (Δ = 2), anomaly-flag output; sharded
  over every GPU of the box (8 on the scaling box; the same test runs unsharded on a one-GPU box).
Production mode (trace = 0: tile skipping, compaction, no per-tick hash).  Compared: everything parity_lib.outputs reports, the per-tick
hash excepted; configs[4] leaves the raw records out (the final state hash changes with any differing byte of any record or clock)."""
import os
import pickle
import sys

import pytest
import torch

import parity_lib as P
from oracle_lib import oracle_sim_threaded
from serf_b200 import GossipSim, scenarios

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_config2_small_world_1m_r8():
    sc = scenarios.small_world_churn(1_000_000, 16, 0.1, 0.05, slots=8, window=200, seed=1, fanout=3)
    assert sc.n == 1_000_000 and sc.slots == 8 and sum(1 for op in sc.ops if op[1] == 4) == 50_000
    o = sc.build(oracle_sim_threaded, trace=0)
    to = o.run_until_converged(sc.max_ticks)
    assert to[1], to
    g = sc.build(GossipSim, trace=0)
    P.assert_same(P.outputs(g, sc, g.run_until_converged(sc.max_ticks)), P.outputs(o, sc, to), with_hash=False)


CONFIG4 = dict(n=10_000_000, degree=16, fanout=4, frac=0.01, delta=2, seed=1)


def _worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from serf_b200 import GossipSim, scenarios
    from serf_b200 import dist as sdist
    sc = scenarios.byzantine_injectors(**CONFIG4)
    g = sc.build(GossipSim, device=rank, rank=rank, world_size=world, trace=0)
    sdist.connect(g, dist, torch.device("cuda", rank))
    out = P.outputs(g, sc, g.run_until_converged(sc.max_ticks), records=False)
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump(out, f)
    dist.barrier()
    dist.destroy_process_group()


def test_config4_byzantine_10m_sharded(tmp_path):
    ngpu = torch.cuda.device_count()
    world = int(os.environ.get("SERFSIM_CONFIG4_WORLD", "0")) or (8 if ngpu >= 8 else 4 if ngpu >= 4 else 2 if ngpu >= 2 else 1)
    sc = scenarios.byzantine_injectors(**CONFIG4)
    assert sc.n == 10_000_000 and 99_000 <= len(sc.byzantine) <= 100_000
    o = sc.build(oracle_sim_threaded, trace=0)
    to = o.run_until_converged(sc.max_ticks)
    assert to[1]
    ref = P.outputs(o, sc, to, records=False)
    fo = ref["anomaly_flags"]
    assert fo[sc.byzantine].mean() > 0.95 and fo.sum() == fo[sc.byzantine].sum()        # injectors are flagged, nobody else is
    if world == 1:
        g = sc.build(GossipSim, trace=0)
        P.assert_same(P.outputs(g, sc, g.run_until_converged(sc.max_ticks), records=False), ref, with_hash=False)
        return
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    port = 29500 + os.getpid() % 1000
    procs = [ctx.Process(target=_worker, args=(r, world, port, str(tmp_path))) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(900)
        assert p.exitcode == 0
    per_rank = []
    for r in range(world):
        with open(os.path.join(str(tmp_path), f"r{r}.pkl"), "rb") as f:
            per_rank.append(pickle.load(f))
    P.assert_same(P.merge_ranks(per_rank), ref, with_hash=False, what=f"world {world}")
