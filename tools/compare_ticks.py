#!/usr/bin/env python
"""Side-by-side per-tick device times of two (or more) tools/tick_profile.py outputs, with the phase sums that matter:
ramp-up, plateau, second wave, tail.

  python tools/compare_ticks.py ticks_main.json ticks_nocompact.json [...]
"""
import json
import sys

runs = [(p, json.load(open(p))) for p in sys.argv[1:]]
if not runs:
    sys.exit(__doc__)
n = max(len(r["rows"]) for _, r in runs)
print("tick  edge_updates " + " ".join(f"{p.split('/')[-1][:22]:>22s}" for p, _ in runs))
for t in range(n):
    eu = next((r["rows"][t]["edge_updates"] for _, r in runs if t < len(r["rows"])), 0)
    print(f"{t:4d} {eu:12d}  " + " ".join(f"{(r['rows'][t]['ms'] * 1e3 if t < len(r['rows']) else float('nan')):19.1f} µs" for _, r in runs))
print()
base = runs[0][1]["rows"]
peak = max(r["edge_updates"] for r in base) or 1
phases = {"unsaturated (< 25 % of peak edge-updates)": lambda r: r["edge_updates"] < 0.25 * peak,
          "saturated (>= 25 % of peak)": lambda r: r["edge_updates"] >= 0.25 * peak}
for name, f in phases.items():
    idx = [t for t, r in enumerate(base) if f(r)]
    print(f"{name:45s}" + " ".join(f"{sum(r['rows'][t]['ms'] for t in idx if t < len(r['rows'])):19.3f} ms" for _, r in runs))
print(f"{'whole run (kernel time)':45s}" + " ".join(f"{r['kernel_ms']:19.3f} ms" for _, r in runs))
