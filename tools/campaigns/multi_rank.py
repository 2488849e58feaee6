"""Randomized campaign of fuzz / fuzz_features scenarios beyond the committed seeds: host-compiled kernels (tests/emu) vs oracle.
Run from the repo root; prints the failing seeds (none expected).  Takes 10-20 minutes."""
import sys, time
import os; ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import parity_lib as P
from emu_lib import emu_sim
from serf_b200 import scenarios
bad=[]; t0=time.time(); n_done=0
for seed in range(100, 400):
    sc = scenarios.fuzz_features(seed, n=300 + 13 * (seed % 40), slots=1 + seed % 4)
    sc.max_ticks = 300
    world = 2 + seed % 3
    try:
        P.run_against_oracle(emu_sim, sc, traces=(0,), world=world)
        n_done+=1
    except Exception as e:
        bad.append((seed, repr(e)[:200])); print('FAIL', seed, world, repr(e)[:300], flush=True)
    if time.time()-t0 > 1200: break
print('multi-rank campaign:', n_done, 'ok, last seed', seed, round(time.time()-t0), 's, bad:', bad, flush=True)
