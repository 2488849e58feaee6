#!/usr/bin/env python
"""Sharded parity on real GPUs in ONE process group per world size (launch under torchrun): every scenario of
tests/test_gpu_multi.py — membership, failure detection, fuzz, user events, injectors, push-pull rounds across shards — plus,
with --full, BASELINE configs[4] at its stated size (10 M nodes, 100 000 injectors).  Rank 0 runs the (threaded) oracle and
compares every output of tests/parity_lib.py (the raw records only below 500 K nodes: the state hash covers them above).  One line
per scenario; exit code 1 if anything differs.  The same comparisons as the pytest file, without paying the NCCL start-up once per
case (GPU minutes on a multi-GPU box are charged per GPU).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29511 tools/multi_parity.py [--full]
"""
import os
import sys
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from serf_b200 import GossipSim, scenarios  # noqa: E402
from serf_b200 import dist as sdist  # noqa: E402
import parity_lib as P  # noqa: E402

rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lr)
dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
full = "--full" in sys.argv

CASES = [
    ("random_graph_leave", dict(n=50_000, degree=16, fanout=3, seed=2, slots=1), {}),
    ("random_graph_leave", dict(n=30_001, degree=12, fanout=4, seed=3, slots=3), {}),
    ("random_graph_fail", dict(n=20_000, degree=16, fanout=3, seed=2), dict(suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)),
    ("dissemination_storm", dict(n=200_000, degree=16, fanout=4, slots=2, seed=3, with_fail=True), {}),           # LAN timers: the ranks sleep through the timer wait
    ("fuzz", dict(seed=7, n=3000, slots=4), dict(push_pull_interval_ticks=0)),
    ("user_event_storm", dict(n=40_000, degree=16, fanout=3, seed=3, n_events=5, spacing=2, churn=100, with_leave=True), {}),
    ("byzantine_injectors", dict(n=40_000, degree=16, fanout=4, frac=0.02, seed=1), {}),
    ("fuzz", dict(seed=11, n=3000, slots=3), {}),
    ("fuzz_features", dict(seed=6, n=3000, slots=3), {}),
    ("fuzz_prune", dict(seed=4, n=3000, slots=3), {}),
    ("user_event_storm", dict(n=20_000, degree=8, fanout=2, seed=6, n_events=5, spacing=2, churn=100, with_leave=True), dict(push_pull_interval_ticks=5, retransmit_mult=1)),
    ("byzantine_injectors", dict(n=20_000, degree=12, fanout=3, frac=0.05, seed=5), dict(push_pull_interval_ticks=6)),
]
if full:
    CASES = [("byzantine_injectors", dict(n=10_000_000, degree=16, fanout=4, frac=0.01, delta=2, seed=1), {}),
             ("small_world_churn", dict(n=1_000_000, k=16, beta=0.1, churn_frac=0.05, slots=8, window=200, seed=1, fanout=3), {})]

failed = 0
for name, kwargs, cfg in CASES:
    t0 = time.time()
    sc = getattr(scenarios, name)(**kwargs)
    big = sc.n > 500_000
    trace = 0 if big else 1
    g = sc.build(GossipSim, device=lr, rank=rank, world_size=world, trace=trace, **cfg)
    sdist.connect(g, dist, torch.device("cuda", lr))
    out = P.outputs(g, sc, g.run_until_converged(sc.max_ticks), records=not big)
    parts = [None] * world
    dist.gather_object(out, parts if rank == 0 else None, dst=0)
    msg = "ok"
    if rank == 0:
        from oracle_lib import oracle_sim, oracle_sim_threaded
        o = sc.build(oracle_sim_threaded if big else oracle_sim, trace=trace, **cfg)
        to = o.run_until_converged(sc.max_ticks)
        try:
            P.assert_same(P.merge_ranks(parts), P.outputs(o, sc, to, records=not big), with_hash=bool(trace))
        except AssertionError as e:
            failed += 1
            msg = f"FAILED: {e}"[:400]
        print(f"world {world}  {sc.name:38s} {cfg if cfg else ''}  ticks {to}  {time.time() - t0:5.1f} s  {msg}", flush=True)
    g.close()
    dist.barrier()
flag = torch.tensor([failed], device="cuda")
dist.broadcast(flag, 0)
dist.destroy_process_group()
sys.exit(1 if int(flag.item()) else 0)
