"""User events on the wire, on the device: SerfDelegate::local_state with every node's event ring, encoded by the batch
kernels of serf_b200/csrc/wire_codec.cu, against rings taken from the oracle's run byte for byte, the range API against the
full batch, and back through the decode kernel to user_event_seen / event_time.  The host-side codec and the same checks at
small sizes on the host build are in tests/test_wire_events.py; tests/test_gpu_z_wire.py covers output without a content
table."""
import numpy as np
import pytest

from oracle_lib import oracle_sim
from serf_b200 import GossipSim, scenarios
from test_wire_events import canonical, check_batches, set_content

pytestmark = pytest.mark.gpu


def _gpu(n, s, **kw):
    return GossipSim(n, s, **kw)


@pytest.mark.parametrize("case", ["alias_churn", "push_pull_rounds"])
def test_device_rings_equal_oracle_rings_100k(case):
    if case == "alias_churn":
        sc = scenarios.user_event_storm(100_000, 16, 3, seed=5, n_events=6, spacing=2, alias=True, churn=400)
        cfg = {}
    else:
        sc = scenarios.user_event_storm(100_000, 8, 2, seed=6, n_events=5, spacing=2, churn=300, with_leave=True)
        cfg = dict(push_pull_interval_ticks=9, retransmit_mult=1)
    o = sc.build(oracle_sim, trace=0, **cfg)
    g = sc.build(_gpu, trace=0, **cfg)
    set_content(g, sc.user_events)
    check_batches(g, o, sc, (0, 4, 12, 50), sample=211)


def test_round_trip_1m_nodes_8_events_in_chunks():
    sc = scenarios.user_event_storm(1_000_000, 16, 4, seed=2, n_events=8, spacing=1, churn=2000)
    g = sc.build(_gpu, trace=0)
    names = [f"deploy-{e:02d}".encode() for e in range(8)]
    pays = [bytes((e * 13 + k) & 0xFF for k in range(400 + 10 * e)) for e in range(8)]
    g.set_user_event_content(names, pays)
    g.step(40)
    E, n = 8, sc.n
    ev_all, lt = g.event_time(), [g.user_event_ltime(e) for e in range(E)]
    mask = np.zeros(n, np.uint32)
    for e in range(E):
        mask |= g.user_event_seen(e).astype(np.uint32) << e
    assert (mask == 0xFF).mean() > 0.5                                # most nodes carry the full 8-event ring (~3.4 KB)
    total = 0
    for first in range(0, n, 300_000):
        count = min(300_000, n - first)
        buf, off = g.wire_local_state_range(first, count)
        ev, seen, um = g.wire_decode_events(buf, off)
        assert (ev == ev_all[first:first + count]).all() and (um == 0).all()
        assert (canonical(seen, sc.user_events, lt) == canonical(mask[first:first + count], sc.user_events, lt)).all()
        total += int(off[-1])
    assert total > 1_000_000 * 1000
