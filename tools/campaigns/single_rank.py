"""Randomized campaign of fuzz / fuzz_features scenarios beyond the committed seeds: host-compiled kernels (tests/emu) vs oracle.
Run from the repo root; prints the failing seeds (none expected).  Takes 10-20 minutes."""
import sys, time
import os; ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
from emu_lib import emu_sim
from serf_b200 import scenarios
import parity_lib as P
bad=[]
t0=time.time()
def one(sc, tag):
    sc.max_ticks=min(sc.max_ticks,1500)
    try:
        P.run_against_oracle(emu_sim, sc, traces=(0, 1))
    except Exception as e:
        bad.append((tag, repr(e)[:200])); print('FAIL', tag, repr(e)[:200], flush=True)
for s in range(40, 400):
    one(scenarios.fuzz(s), f'fuzz{s}')
    if time.time()-t0 > 900: break
print('fuzz done up to', s, round(time.time()-t0), flush=True)
t1=time.time()
for s in range(30, 330):
    one(scenarios.fuzz_features(s), f'feat{s}')
    if time.time()-t1 > 900: break
print('features done up to', s, round(time.time()-t1), 'bad:', bad, flush=True)
