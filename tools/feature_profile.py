#!/usr/bin/env python
"""Device time of the user-event and byzantine-injector scenarios at BASELINE scale (10 M nodes by default):
per-run kernel time, ticks to quiescence, deliveries per second and the algorithmic bytes behind them.

  python tools/feature_profile.py --what events    --out events.json
  python tools/feature_profile.py --what byzantine --out byzantine.json     # BASELINE configs[4] shape, one GPU
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from serf_b200 import GossipSim, scenarios  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--what", choices=["events", "byzantine"], required=True)
ap.add_argument("--nodes", type=int, default=10_000_000)
ap.add_argument("--fanout", type=int, default=4)
ap.add_argument("--degree", type=int, default=16)
ap.add_argument("--events", type=int, default=4)
ap.add_argument("--frac", type=float, default=0.01)
ap.add_argument("--runs", type=int, default=3)
ap.add_argument("--out", default=None)
a = ap.parse_args()

if a.what == "events":
    sc = scenarios.user_event_storm(a.nodes, a.degree, a.fanout, seed=1, n_events=a.events, spacing=3)
else:
    sc = scenarios.byzantine_injectors(a.nodes, a.degree, a.fanout, a.frac, seed=1)
g = sc.build(lambda n, s, **kw: GossipSim(n, s, **kw))
res = []
for run in range(a.runs):
    g.reset(sc.cfg["seed"])
    sc.schedule(g)
    g.set_tick_timing(run == a.runs - 1)
    ticks, ok = g.run_until_converged(sc.max_ticks)
    ms, launches = g.last_step_device_ms()
    res.append({"ticks": ticks, "converged": ok, "kernel_ms": ms, "launches": launches})
st = g.stats()
out = {"scenario": sc.name, "runs": res, "stats": st}
if a.what == "events":
    ue = g.user_event_stats()
    p_dirty = ue["delivered"] / max(1, ue["edge_updates"])
    b = 4 + 16 / a.fanout + 4 + 16 + 16 * p_dirty            # DESIGN §8.3: neighbour index + sender record / f + inbox word + destination record (+ write-back)
    out.update(user_events=ue, bytes_per_event_edge_update=b,
               event_edge_updates_per_s=ue["edge_updates"] / (res[-1]["kernel_ms"] * 1e-3),
               algorithmic_GBps=ue["edge_updates"] * b / (res[-1]["kernel_ms"] * 1e-3) / 1e9)
else:
    bz = g.byzantine_stats()
    out.update(byzantine=bz, injectors=int(len(sc.byzantine)), flagged_fraction=bz["flagged"] / max(1, len(sc.byzantine)),
               edge_updates_per_s=st["edge_updates"] / (res[-1]["kernel_ms"] * 1e-3))
tr, tms = g.tick_trace(), g.tick_times_ms()
out["ticks"] = [{"tick": t, "ms": float(tms[t]), "edge_updates": int(tr["edge_updates"][t]), "pending": int(tr["pending"][t])} for t in range(len(tms))]
print(json.dumps({k: v for k, v in out.items() if k != "ticks"}))
if a.out:
    json.dump(out, open(a.out, "w"), indent=1)
