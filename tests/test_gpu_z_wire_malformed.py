"""The malformed-bytes corpus of tests/wire_malformed_lib.py through both batch decode kernels on the device
(pp_decode_kernel and pp_events_decode_kernel of serf_b200/csrc/wire_codec.cu): every input alone and at index k of a batch
of valid messages must fail the call at the first bad index with the host decoder's class, or decode as the host decoders
do; and a batch of 1 M valid messages with about 1 % replaced by corpus inputs must report the lowest bad index and, with
the bad ones removed, decode to the getters' state.  Every batch passes the offsets rule; the rejections of bad offsets are
tested on the host build only (tests/test_wire_malformed.py), as is the agreement of the three host decoders."""
import numpy as np
import pytest

import wire_events_lib as WE
import wire_lib as W
import wire_malformed_lib as ML
from serf_b200 import GossipSim, scenarios
from serf_b200.sim import load_library
from test_wire_events import canonical
from test_wire_malformed import batch_sim

pytestmark = pytest.mark.gpu


def _gpu(n, s, **kw):
    return GossipSim(n, s, **kw)


@pytest.fixture(scope="module")
def P():
    return WE.bind(load_library())               # the host decoders of the product library give the expected outcomes


def test_device_batch_kernels_on_the_corpus(P):
    g, table, valid = batch_sim(_gpu)
    cases = ML.corpus()
    assert len(cases) > 3000
    for i, c in enumerate(cases):
        ML.check_in_batches(P, g, table, 3, c.data, valid[:4], i % 5)
    # the neighbour whose bytes would complete a truncated message is not read
    msgs = [valid[0], valid[1][:-3], valid[1][-3:] + valid[2]]
    assert ML.run_decode_batch(P, g, msgs, 3) == ("err", 1, "truncated")
    assert ML.run_events_batch(g, msgs) == ("err", 1, "truncated")
    g.close()


def test_device_one_million_messages_with_one_percent_from_the_corpus(P):
    sc = scenarios.user_event_storm(1_000_000, 16, 4, seed=2, n_events=4, spacing=1, churn=2000)
    g = sc.build(_gpu, trace=0)
    names, pays = [f"ev-{e}".encode() for e in range(4)], [bytes([e]) * (3 + e) for e in range(4)]
    g.set_user_event_content(names, pays)
    g.step(40)
    n, slots = sc.n, sc.slots
    table = (names, pays, [g.user_event_ltime(e) for e in range(4)])
    buf, off = g.wire_local_state_range()
    raw = buf.tobytes()
    msgs = [raw[int(off[i]):int(off[i + 1])] for i in range(n)]
    cases = ML.corpus()
    rng = np.random.default_rng(11)
    at = np.sort(rng.choice(n, n // 100, replace=False))
    for i in at:
        msgs[i] = cases[int(rng.integers(len(cases)))].data
    want_m = {int(i): ML.expect_decode_batch(P, msgs[i], slots) for i in at}
    want_e = {int(i): ML.expect_events_batch(P, msgs[i], table) for i in at}
    bad_m = sorted(i for i, w in want_m.items() if w[0] == "err")
    bad_e = sorted(i for i, w in want_e.items() if w[0] == "err")
    assert len(bad_m) > 3000 and len(bad_e) > 3000 and len(bad_m) < len(at)
    b, o = ML.pack(msgs)
    rc, _ = W.decode_batch(P, g, b, o, slots, check=False)
    assert rc != 0 and ML.batch_error(P.serfsim_last_error()) == (bad_m[0], want_m[bad_m[0]][1])
    assert ML.run_events_batch(g, msgs) == ("err", bad_e[0], want_e[bad_e[0]][1])
    del b, o

    replaced = np.zeros(n, bool)
    replaced[at] = True
    lamport, ev_all = g.lamport_time(), g.event_time()
    status = np.stack([g.member_status(s) for s in range(slots)], axis=1)
    ltime = np.stack([g.status_ltime(s) for s in range(slots)], axis=1)
    mask = np.zeros(n, np.uint32)
    for e in range(4):
        mask |= g.user_event_seen(e).astype(np.uint32) << e

    # the membership kernel without its bad messages: the originals decode to the getters' state, the corpus inputs as the host decodes them
    keep = np.ones(n, bool)
    keep[bad_m] = False
    idx = np.flatnonzero(keep)
    b, o = ML.pack([msgs[i] for i in idx])
    lt, ids, sts, ns = W.decode_batch(P, g, b, o, slots)
    del b, o
    orig = ~replaced[idx]
    assert (lt[orig] == lamport[idx[orig]]).all()
    known = status[idx[orig]] != 0                                 # entries in slot order, known slots only
    assert (ns[orig] == known.sum(axis=1)).all() and known.mean() > 0.5
    r, s = np.nonzero(known)
    pos = (np.cumsum(known, axis=1) - 1)[r, s]
    assert (ids[orig][r, pos] == sc.subjects.astype(np.uint64)[s]).all() and (sts[orig][r, pos] == ltime[idx[orig]][r, s]).all()
    for j in np.flatnonzero(~orig):
        assert ("ok", (int(lt[j]), [(int(ids[j, k]), int(sts[j, k])) for k in range(ns[j])])) == want_m[int(idx[j])]

    # the events kernel without its bad messages
    keep = np.ones(n, bool)
    keep[bad_e] = False
    idx = np.flatnonzero(keep)
    ev, seen, um = g.wire_decode_events(*ML.pack([msgs[i] for i in idx]))
    orig = ~replaced[idx]
    assert (ev[orig] == ev_all[idx[orig]]).all() and (um[orig] == 0).all()
    assert (canonical(seen[orig], sc.user_events, table[2]) == canonical(mask[idx[orig]], sc.user_events, table[2])).all()
    assert (mask[idx[orig]] != 0).mean() > 0.5
    for j in np.flatnonzero(~orig):
        assert ("ok", (int(ev[j]), int(seen[j]), int(um[j]))) == want_e[int(idx[j])]
    g.close()
