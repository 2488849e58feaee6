"""Campaign aimed at the convergence loop (launch chunks, probe tick, jump over sleeping stretches, gate): fuzz scenarios with a few more
host operations — many of them no-ops — scattered over the 300 ticks AFTER the busy part, where the cluster sleeps between timers, reaper and
anti-entropy rounds.  Host-compiled kernels (tests/emu) against the oracle, production mode and trace mode, default launch chunks and a random
fixed chunk; single rank and two ranks.  Prints the failing seeds (none expected)."""
import sys, time, os
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import parity_lib as P
from emu_lib import emu_sim
from oracle_lib import oracle_sim
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from late_ops_gen import late

bad = []; t_start = time.time()
for seed in range(1000, 1400):
    sc = late(seed)
    try:
        o = sc.build(oracle_sim, trace=1); ref = P.outputs(o, sc, o.run_until_converged(sc.max_ticks))
        for trace, chunk in ((0, None), (1, None), (0, str(2 + seed % 11))):
            if chunk: os.environ["SERFSIM_CHUNK"] = chunk
            else: os.environ.pop("SERFSIM_CHUNK", None)
            g = sc.build(emu_sim, trace=trace)
            P.assert_same(P.outputs(g, sc, g.run_until_converged(sc.max_ticks)), ref, with_hash=bool(trace), what=f"trace={trace} chunk={chunk}")
        os.environ.pop("SERFSIM_CHUNK", None)
        if seed % 3 == 0:                                   # two ranks, production mode
            P.assert_same(P.run_ranks(sc, 2, 0), ref, with_hash=False, what="2 ranks")
    except Exception as e:
        bad.append((seed, repr(e)[:160])); print("FAIL", seed, repr(e)[:160], flush=True)
    if time.time() - t_start > 1500: break
print("late-ops campaign done up to seed", seed, round(time.time() - t_start), "s, bad:", bad, flush=True)
