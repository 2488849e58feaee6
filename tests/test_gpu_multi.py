"""Multi-GPU parity (needs ≥ 2 GPUs; run with `python -m pytest tests/test_gpu_multi.py -m gpu` on a machine with them).
The id range is sharded over 2 (or 4) ranks, cross-shard gossip goes through the NVLink windows, and the
concatenated records / summed trace must equal the CPU oracle's — i.e. the result is independent of the sharding."""
import os
import pickle
import sys

import pytest
import torch

import parity_lib as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, scen_args, outdir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from serf_b200 import GossipSim, scenarios
    from serf_b200 import dist as sdist
    name, kwargs, cfg = scen_args
    sc = getattr(scenarios, name)(**kwargs)
    g = sc.build(GossipSim, device=rank, rank=rank, world_size=world, trace=1, **cfg)
    sdist.connect(g, dist, torch.device("cuda", rank))
    out = P.outputs(g, sc, g.run_until_converged(sc.max_ticks))
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump(out, f)
    dist.barrier()
    dist.destroy_process_group()


def _run(world, scen_args, tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    port = 29500 + os.getpid() % 1000
    procs = [ctx.Process(target=_worker, args=(r, world, port, scen_args, str(tmp_path))) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(600)
        assert p.exitcode == 0
    res = []
    for r in range(world):
        with open(os.path.join(str(tmp_path), f"r{r}.pkl"), "rb") as f:
            res.append(pickle.load(f))
    return res


WORLDS = [int(x) for x in os.environ.get("SERFSIM_TEST_WORLDS", "2,4").split(",")]


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("scen", [
    ("random_graph_leave", dict(n=50_000, degree=16, fanout=3, seed=2, slots=1), {}),
    ("random_graph_leave", dict(n=30_001, degree=12, fanout=4, seed=3, slots=3), {}),
    ("random_graph_fail", dict(n=20_000, degree=16, fanout=3, seed=2), dict(suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)),
    ("fuzz", dict(seed=7, n=3000, slots=4), dict(push_pull_interval_ticks=0)),
    # cross-shard traffic added after the last multi-GPU run (checked with the host-compiled kernels, tests/test_emu_multi.py)
    ("user_event_storm", dict(n=40_000, degree=16, fanout=3, seed=3, n_events=5, spacing=2, churn=100, with_leave=True), {}),
    ("byzantine_injectors", dict(n=40_000, degree=16, fanout=4, frac=0.02, seed=1), {}),
    ("fuzz", dict(seed=11, n=3000, slots=3), {}),                                   # push-pull rounds across shards (fuzz 11 has them on)
    ("fuzz_features", dict(seed=6, n=3000, slots=3), {}),
    ("user_event_storm", dict(n=20_000, degree=8, fanout=2, seed=6, n_events=5, spacing=2, churn=100, with_leave=True), dict(push_pull_interval_ticks=5, retransmit_mult=1)),
    ("byzantine_injectors", dict(n=20_000, degree=12, fanout=3, frac=0.05, seed=5), dict(push_pull_interval_ticks=6)),
])
def test_sharded_equals_oracle(world, scen, tmp_path):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    from oracle_lib import oracle_sim
    from serf_b200 import scenarios
    name, kwargs, cfg = scen
    sc = getattr(scenarios, name)(**kwargs)
    o = sc.build(oracle_sim, trace=1, **cfg)
    ref = P.outputs(o, sc, o.run_until_converged(sc.max_ticks))
    P.assert_same(P.merge_ranks(_run(world, scen, tmp_path)), ref, with_hash=True, what=f"world {world}")
