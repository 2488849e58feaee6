"""Feature-rich random scenarios at multi-tile scale, shared by tests/test_emu_scaled_fuzz.py and tests/test_gpu_z_scaled_fuzz.py —
test infrastructure only.

scenarios.fuzz and its descendants draw at most 400 nodes: one or two tiles, one or two CTAs.  The large studies reach many tiles but
carry one operation each.  scaled_fuzz puts every feature at once — all operation kinds, the reaper erasing members mid-run, push-pull
rounds, user events with aliased contents, byzantine injectors — on 20 K – 200 K nodes, with operations timed so that the production
tick regimes all occur: saturated and compacted ticks, sparse ticks (fewer than tiles / 2 messages), per-view passes in which one view
saturates and another does not, sleeping stretches the scheduler skips or jumps over, and host operations at launch-chunk boundaries.

- scaled_fuzz(seed, n=None): the scenario.  Every draw comes from Philox streams of the seed, so a seed gives the same scenario on every
  machine; `n` replaces the drawn node count (the ragged last tile is still drawn, so n is rounded to a multiple of 256 plus 1 – 255).
- reach: which production paths a trace = 0 run of the product took, derived from its getters alone (no probes on the device).
"""
import math

import numpy as np

import envelope_lib as E
from serf_b200.scenarios import Scenario
from serf_b200.sim import Op, random_regular_graph, small_world_graph

TILE = E.TILE
KINDS = (Op.JOIN, Op.LEAVE, Op.FORCE_LEAVE, Op.FAIL, Op.REJOIN, Op.FORCE_LEAVE_PRUNE)


def _rng(seed, stream):
    return np.random.Generator(np.random.Philox(seed + 61_000_037 * (stream + 1)))


def _size(rng, n):
    """n tiles' worth of nodes with a ragged last tile of 1, 255 or 2–254 nodes (never a multiple of 256)."""
    tiles = int(rng.integers(80, 782))                               # 20 225 – 199 935 nodes
    last = (1, 255, int(rng.integers(2, 255)))[int(rng.integers(0, 3))]
    if n is not None:
        tiles = max(3, n // TILE + 1)
    return (tiles - 1) * TILE + last


def _node(rng, n):
    """A node id: a tile boundary (256k − 1 or 256k), one of the ragged last tile, or uniform (hot tiles spread over many CTAs)."""
    tiles = (n + TILE - 1) // TILE
    r = rng.random()
    if r < 0.25:
        return min(n - 1, int(rng.integers(1, tiles)) * TILE - int(rng.integers(0, 2)))
    if r < 0.35:
        return (tiles - 1) * TILE + int(rng.integers(0, n - (tiles - 1) * TILE))
    return int(rng.integers(0, n))


def scaled_fuzz(seed, n=None):
    shape, ops_rng, sub = _rng(seed, 0), _rng(seed, 1), _rng(seed, 2)

    # ---- size and shape ----
    n = _size(shape, n)
    slots = int(shape.choice(np.arange(1, 17), p=[0.08] + [0.72 / 7] * 7 + [0.2 / 8] * 8))
    fanout = int(shape.integers(1, 9))
    degree = int(shape.integers(4, 17))
    topology = E.TOPOLOGIES[int(shape.choice(3, p=[0.4, 0.3, 0.3]))]
    if topology == "regular":
        topo = random_regular_graph(n, degree, seed + 17)
    elif topology == "small_world":
        topo = small_world_graph(n, max(2, degree // 2 * 2), 0.2, seed + 17)
    else:
        topo = E.irregular_graph(n, seed + 17, mean_degree=degree, hubs=int(shape.integers(0, 3)), hub_degree=(1000, 3000))
    subjects = []
    while len(subjects) < slots:
        v = _node(shape, n)
        if v not in subjects:
            subjects.append(v)

    # ---- subsystems and timers ----
    lan = sub.random() < 0.4                   # memberlist LAN defaults: long suspicion sleeps, timer-wheel wake-ups
    cfg = dict(fanout=fanout, seed=int(sub.integers(1, 2**40)), init_status_ltime=int(sub.integers(0, 3)), init_clock=int(sub.integers(1, 5)),
               retransmit_mult=1 if sub.random() < 0.35 else int(sub.integers(2, 5)))
    if not lan:
        cfg.update(suspicion_mult=int(sub.integers(2, 5)), suspicion_max_timeout_mult=int(sub.integers(2, 4)),
                   probe_interval_ticks=int(sub.integers(1, 4)))
    reap = int(sub.choice([0, 3, 7, 9, 13]))
    cfg.update(reap_interval_ticks=reap, tombstone_timeout_ticks=int(sub.integers(5, 40)), reconnect_timeout_ticks=int(sub.integers(5, 40)),
               recent_intent_timeout_ticks=int(sub.integers(5, 40)))
    pp = int(sub.choice([0, 4, 5, 6, 11, 17, 23]))
    if pp and reap and math.gcd(pp, reap) != 1:
        pp += 1 if math.gcd(pp + 1, reap) == 1 else 2            # co-prime: some rounds land on reaper ticks, most do not
    cfg["push_pull_interval_ticks"] = pp
    byzantine, delta = None, 2
    if sub.random() < 0.35:                    # injectors switch the per-view passes off: a minority of the scenarios
        k = max(1, int(n * sub.uniform(0.001, 0.02)))
        byzantine = sub.choice(n, size=k, replace=False).astype(np.uint32)
        delta = int(sub.integers(0, 4))
        cfg["init_clock"] = int(sub.integers(4, 13))
    user_events = None
    if sub.random() < 0.6:
        user_events = sub.integers(1, 4, size=int(sub.integers(1, 9))).astype(np.uint32)      # few distinct contents → aliases

    # ---- operations ----
    ops, used = [], set()

    def add(t, kind, node, s):
        if t >= 0 and (t, node) not in used:
            used.add((t, node))
            ops.append((int(t), int(kind), int(node), int(s)))

    def subject_op(t, s, kinds=(Op.LEAVE, Op.FAIL, Op.FORCE_LEAVE, Op.FORCE_LEAVE_PRUNE), p=(0.4, 0.3, 0.15, 0.15)):
        kind = Op(int(ops_rng.choice(kinds, p=p)))
        if kind in (Op.FORCE_LEAVE, Op.FORCE_LEAVE_PRUNE):
            add(t, kind, _node(ops_rng, n), s)                  # the operation's origin; the slot names the subject
        else:
            add(t, kind, subjects[s], s)
        return kind

    def single(t):
        kind = Op(int(ops_rng.choice(KINDS)))
        s = int(ops_rng.integers(0, slots))
        if kind in (Op.JOIN, Op.LEAVE) or (kind in (Op.FAIL, Op.REJOIN) and ops_rng.random() < 0.5):
            add(t, kind, subjects[s], s)
        else:
            add(t, kind, _node(ops_rng, n), s)

    horizon = int(ops_rng.integers(30, 90))
    for _ in range(int(ops_rng.integers(1, 4))):
        # a wave: several subjects leave or crash in one tick, the other views follow a few ticks later
        t0 = int(ops_rng.integers(0, horizon))
        order = ops_rng.permutation(slots)
        first = order[:max(1, (len(order) + 1) // 2)]
        for s in first:
            if subject_op(t0, int(s)) == Op.FAIL and ops_rng.random() < 0.5:
                add(t0 + int(ops_rng.integers(15, 80)), Op.REJOIN, subjects[int(s)], int(s))   # after the reaper may have erased it
        for s in order[len(first):]:
            subject_op(t0 + int(ops_rng.integers(1, 6)), int(s))
        for _ in range(int(ops_rng.integers(1, 4))):
            single(t0 + int(ops_rng.integers(1, 4)))                  # ramp-up: sparse ticks
        for _ in range(int(ops_rng.integers(1, 4))):
            single(t0 + int(ops_rng.integers(8, 40)))                 # tail
    for _ in range(int(ops_rng.integers(2, 6))):
        # launch-chunk boundaries (chunks of 8 / 16 / 32, restarting at 8 after a jump) and ticks deep inside a sleep
        k = int(ops_rng.integers(1, (horizon + 120) // 8))
        single(8 * k + int(ops_rng.choice([0, 1, 7])))
    for _ in range(int(ops_rng.integers(0, 3))):
        single(horizon + int(ops_rng.integers(40, 160)))
    # JOIN / REJOIN after the reaper's timeouts: the new-member branch
    for _ in range(int(ops_rng.integers(1, 4))):
        s = int(ops_rng.integers(0, slots))
        add(horizon + int(ops_rng.integers(20, 60)), Op.JOIN if ops_rng.random() < 0.5 else Op.REJOIN, subjects[s], s)
    if user_events is not None:
        for e in range(len(user_events)):
            for _ in range(8):
                t = int(ops_rng.integers(0, horizon + 40))
                v = _node(ops_rng, n)
                if (t, v) not in used:
                    add(t, Op.USER_EVENT, v, e)
                    break
    ops.sort(key=lambda x: x[0])

    # Irregular graphs: isolated nodes that received mail never go quiet (envelope_lib) — such runs stop at the cap on both sides.
    max_ticks = 160 if topology == "irregular" else 420
    sc = Scenario(f"scaled_fuzz_{seed}_n{n}_{topology}_f{fanout}_r{slots}" + ("_lan" if lan else ""), n, slots, topo, subjects, ops, cfg,
                  max_ticks=max_ticks, user_events=user_events, byzantine=byzantine, delta=delta)
    sc.topology, sc.lan = topology, lan
    return sc


# ---- which production paths a trace = 0 run took, from the product's getters ----------------------------------------
def reach(got, sc):
    """got: an envelope_lib.product_run of sc.  Counts of the ticks of a trace = 0 run that exercised each path, from the trace rows and the per-view kind counters.
    pass_ticks: ticks that ran as per-view passes.  compacted_under_other: pass ticks after a pass tick in which the whole tick sent
    at least n / 2 messages but some view fewer (that view's pass takes the compacted walk).  unread_plane: pass ticks after a pass
    tick in which a kind was in flight in one view and absent in another.  sparse / dense: ticks below / at or above tiles / 2 messages."""
    n = sc.n
    tiles = (n + TILE - 1) // TILE
    msgs = got["out"]["trace"]["messages"].astype(np.int64)
    vk = got["view_kinds"].astype(np.int64)
    ran = vk.reshape(len(vk), -1).sum(axis=1) > 0
    follow = ran[1:] & ran[:-1]                                    # tick t + 1 ran as passes on the counts of pass tick t
    per_view = vk.sum(axis=2)
    other = (msgs[:-1] >= n >> 1) & (per_view[:-1] < n >> 1).any(axis=1)
    in_some = (vk > 0).any(axis=1)                                 # [t, kind]
    in_all = (vk > 0).all(axis=1)
    unread = (in_some & ~in_all).any(axis=1)[:-1]
    return dict(pass_ticks=int(ran.sum()), compacted_under_other=int((follow & other).sum()), unread_plane=int((follow & unread).sum()),
                sparse=int(((msgs > 0) & (msgs < tiles / 2)).sum()), dense=int((msgs >= tiles / 2).sum()))
