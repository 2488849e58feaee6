#!/usr/bin/env python
"""Per-tick device time of the bench workload: edge-updates, ms and algorithmic GB/s of every tick launch.

Multi-slot runs also print the messages each view sent (leave / join / memberlist, counted by the per-view passes; ticks that ran the
general kernel show none) and what that means for the passes of the NEXT tick, which choose their loads from their own view's counts:
`compact` = passes that walk their view compacted although the whole tick was saturated, `skip` = inbox planes of a kind in flight in
another view that a pass leaves unread (both counted for the views that sent in the tick before: a lower bound).  --busy trims the table to ticks that sent or took longer than that many microseconds."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from serf_b200 import GossipSim, scenarios  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--nodes", type=int, default=10_000_000)
ap.add_argument("--fanout", type=int, default=4)
ap.add_argument("--slots", type=int, default=1)
ap.add_argument("--degree", type=int, default=16)
ap.add_argument("--waves", type=int, default=1)
ap.add_argument("--runs", type=int, default=2)
ap.add_argument("--out", default=None)
ap.add_argument("--scenario", default="storm", choices=["storm", "storm_fail", "churn"])
ap.add_argument("--busy", type=float, default=0.0, help="print only ticks that sent messages or took at least this many microseconds")
a = ap.parse_args()
if a.scenario == "churn":      # BASELINE configs[2]: small-world graph, 5 % of the nodes fail / rejoin, 8 tracked subjects
    sc = scenarios.small_world_churn(a.nodes, a.degree, 0.1, 0.05, slots=a.slots, window=200, seed=1, fanout=a.fanout)
    extra = dict(suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)
elif a.scenario == "storm_fail":   # bench.py's default workload (SURVEY §8d item 4): one subject leaves, one crashes
    sc = scenarios.dissemination_storm(a.nodes, a.degree, a.fanout, slots=max(2, a.slots), seed=1, waves=a.waves, with_fail=True)
    extra = {}
else:
    sc = scenarios.dissemination_storm(a.nodes, a.degree, a.fanout, slots=a.slots, seed=1, waves=a.waves)
    extra = {}
g = sc.build(lambda n, s, **kw: GossipSim(n, s, **kw), **extra)
st_n = sc.n
for run in range(a.runs):
    g.reset(1); sc.schedule(g)
    g.set_tick_timing(run == a.runs - 1)
    ticks, ok = g.run_until_converged(sc.max_ticks)
tr, ms = g.tick_trace(), g.tick_times_ms()
st = g.stats()
p_dirty = st["changed"] / max(1, st["edge_updates"])
R = sc.slots
vk = g.tick_view_kinds() if R > 1 and hasattr(g._lib, "serfsim_tick_view_kinds") else None   # (a library older than the counters: none)
rows = []
n_compact = n_skip = 0
for t in range(len(ms)):
    eu, ch = int(tr["edge_updates"][t]), int(tr["changed"][t])
    be = 4 + 32 / a.fanout + 32 + 32 * (ch / eu if eu else 0)
    rows.append({"tick": t, "edge_updates": eu, "changed": ch, "pending": int(tr["pending"][t]), "messages": int(tr["messages"][t]), "ms": float(ms[t]),
                 "alg_GBps": float(eu * be / (ms[t] * 1e-3) / 1e9) if ms[t] > 0 else 0.0})
    extra = ""
    if vk is not None:
        rows[-1]["view_kinds"] = vk[t].tolist()
        extra = "  " + " ".join("v%d %s" % (s, "/".join(str(int(x)) for x in vk[t, s])) for s in range(R))
        # the passes of tick t use their own view's counts of tick t-1 when every message of t-1 was a pass's
        prev = vk[t - 1] if t > 0 else None
        if prev is not None and prev.sum() > 0 and prev.sum() == int(tr["messages"][t - 1]):
            whole_sat = prev.sum() >= st_n // 2
            cmp_ = sum(1 for s in range(R) if whole_sat and prev[s].sum() < st_n // 2 and prev[s].sum() > 0)
            skp = sum(1 for s in range(R) for k in range(3) if prev[s].sum() > 0 and prev[s, k] == 0 and prev[:, k].sum() > 0)
            rows[-1]["passes_compacted"], rows[-1]["planes_skipped"] = cmp_, skp
            n_compact += cmp_; n_skip += skp
            extra += f"  compact {cmp_} skip {skp}"
    if int(tr["messages"][t]) or ms[t] * 1e3 >= a.busy:
        print(f"tick {t:3d}  eu {eu:10d}  changed {ch:9d}  pending {int(tr['pending'][t]):9d}  {ms[t]*1e3:9.1f} us  {rows[-1]['alg_GBps']:8.1f} GB/s(alg){extra}")
if vk is not None:
    print(f"passes of a view that sent in the tick before and walk compacted in a tick the whole-tick rule calls saturated: {n_compact}; inbox planes left unread: {n_skip}")
tot = float(ms.sum())
print(f"total {tot:.3f} ms kernel time, {st['edge_updates']} edge-updates, {st['edge_updates'] / tot / 1e6:.2f} G edge-updates/s (kernel time only), p_dirty {p_dirty:.4f}")
if a.out:
    json.dump({"scenario": sc.name, "rows": rows, "kernel_ms": tot, "edge_updates": st["edge_updates"], "p_dirty": p_dirty}, open(a.out, "w"), indent=1)
