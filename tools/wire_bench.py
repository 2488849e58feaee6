"""Times serfsim_wire_local_state_range — SerfDelegate::local_state of every node, encoded on the device — with and without a
user-event content table, alternated in one process, at 1 M and 10 M nodes.

The workload: user_event_storm with 8 tracked events of ~500 B each (name + payload = 496 B), stepped until every node holds
all 8, so a node's push-pull message carries its whole ring (~4 KB).  The shard is encoded in chunks of --chunk nodes (the
full batch of 10 M nodes would be ~40 GB).  Per arm and size it reports the wall time of the range calls (length kernel,
scan, emit kernel, device→host copy of the bytes) and, from torch.profiler, the device time of the emit kernel with the
bytes it wrote per second and their share of HBM bandwidth (3.35 TB/s, H100 SXM data sheet: the emit kernel is bound by
its writes).  Card name and power limit are read in the same run.

    python tools/wire_bench.py [--sizes 1000000 10000000] [--chunk 500000] [--reps 3] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time


sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from serf_b200 import GossipSim, scenarios  # noqa: E402

HBM_BPS = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def encode_all(g, chunk):
    total = 0
    for first in range(0, g.count, chunk):
        buf, off = g.wire_local_state_range(first, min(chunk, g.count - first))
        total += int(off[-1])
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 10_000_000])
    ap.add_argument("--chunk", type=int, default=500_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", help="also write the results as JSON to this file")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("wire_bench: no GPU — nothing to measure")
    torch.cuda.init()
    res = dict(card=card(), chunk=a.chunk, runs=[])
    names = [f"release-{e:04d}-x".encode() for e in range(8)]                     # 16 B
    pays = [bytes((e * 29 + k) & 0xFF for k in range(480)) for e in range(8)]     # 480 B
    for n in a.sizes:
        sc = scenarios.user_event_storm(n, 16, 4, seed=1, n_events=8, spacing=1)
        arms = {}
        for arm in ("no_content", "content"):
            g = sc.build(lambda nn, s, **kw: GossipSim(nn, s, **kw), trace=0)
            if arm == "content":
                g.set_user_event_content(names, pays)
            g.run_until_converged(400)
            seen = g.user_event_records()["seen"]
            arms[arm] = dict(sim=g, full_ring=float((seen == 0xFF).mean()))
        for arm in arms.values():
            encode_all(arm["sim"], a.chunk)                                         # warm-up: modules, allocations
        for name in ("no_content", "content"):
            arms[name]["wall_s"] = []
        for r in range(a.reps):                                                     # alternate the two arms
            for name in ("no_content", "content"):
                t0 = time.perf_counter()
                arms[name]["bytes"] = encode_all(arms[name]["sim"], a.chunk)
                arms[name]["wall_s"].append(time.perf_counter() - t0)
        for name in ("no_content", "content"):                                      # device time, in a profiled pass of its own
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                encode_all(arms[name]["sim"], a.chunk)
                torch.cuda.synchronize()
            dev = {}
            for ev in prof.key_averages():
                for k in ("pp_len_kernel", "pp_scan_kernel", "pp_emit_kernel"):
                    if k in ev.key:
                        us = getattr(ev, "device_time_total", None)
                        dev[k] = dev.get(k, 0.0) + (us if us is not None else ev.cuda_time_total) / 1e6
            arms[name]["device_s"] = dev
        for name in ("no_content", "content"):
            x = arms[name]
            run = dict(n=n, arm=name, bytes=x["bytes"], full_ring_share=x["full_ring"], wall_s=x["wall_s"],
                       wall_bytes_per_s=x["bytes"] / min(x["wall_s"]), device_s=x["device_s"])
            emit = x["device_s"].get("pp_emit_kernel")
            if emit:
                run["emit_bytes_per_s"] = x["bytes"] / emit
                run["emit_share_of_hbm"] = x["bytes"] / emit / HBM_BPS
            res["runs"].append(run)
            print(json.dumps(run), flush=True)
            x["sim"].close()
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(dict(card=res["card"], card_after=res["card_after"])))


if __name__ == "__main__":
    main()
