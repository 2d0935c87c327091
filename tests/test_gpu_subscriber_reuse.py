"""Subscriber id reuse (cpbus_release_many, cpbus_subscribe_list; Bus.release_many / subscribe_list and the GroupBus twins)
on the GPU, against the oracle extended with release and a lowest-free subscribe (tests/reuse_oracle.py).  Random traces
mix subscribes, subscribe_list with and without cases, unsubscribes, releases (repeats, live, never-issued and released
ids), sends, publishes, timers (cancels with stale ids of a slot's previous occupant), clock jumps, drains and (lossless)
takes and acks, on dense, sparse and drop-missed-ticks buses, K = 1, 2, 4, 8, in both modes; each trace ends with every
mailbox, the stats but the launch-shaped ones, publish counts, lagging and blockers compared.  Also: churn past capacity,
stale timer ids, lossless held records and room, CPBUS_EAGAIN with nothing applied, the one-launch cost, a stream shard
with outstanding followers, the group against one bus, a fleet of 2^20, and the C++ mirror."""
import ctypes as C
import os
import subprocess
from collections import Counter

import numpy as np
import pytest

import drop_oracle
import lag_oracle
import reuse_oracle as ro
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from containerpilot_b200.group import GroupBus

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAUNCH_SHAPED = ("batches", "kernel_launches", "admit_passes", "admit_skipped", "admit_partial", "device_splits")
MODES = {"dense": {}, "sparse_ticks": {"sparse_ticks": True}, "sparse_records": {"sparse_records": True},
         "drop_missed": {"drop_missed_ticks": True}}


class DropReuseOracle(ro.ReuseOracle):
    def advance(self, now_ns):
        return drop_oracle.lib().orc_advance_drop_missed(self.h, now_ns)


def _st(fn, *args):
    """(status, result) of a Bus method, whether it returns a status or raises"""
    try:
        r = fn(*args)
    except nat.CpbusError as e:
        return e.status, None
    if fn.__name__ in ("publish", "send", "advance", "flush"):
        return int(r), None
    return nat.OK, r


def _trace(seed, n0=12, n_ops=900, n_max=40):
    rng = np.random.default_rng(seed)
    ops, now = [], 0

    def masks(k):
        return [nat.MASK_ALL if rng.random() < 0.4 else int(rng.integers(0, 1 << 17)) for _ in range(k)]

    def cases():
        return [(int(rng.integers(0, 17)), int(rng.integers(0, 8))) for _ in range(int(rng.integers(1, 5)))]

    ops.append(("list", masks(n0), None))
    for _ in range(n_ops):
        r = rng.random()
        if r < 0.05:
            k = int(rng.integers(1, 5))
            ops.append(("list", masks(k), [cases() if rng.random() < 0.4 else [] for _ in range(k)] if rng.random() < 0.5 else None))
        elif r < 0.06:
            ops.append(("sub", masks(1)[0], cases() if rng.random() < 0.3 else None))
        elif r < 0.11:
            ops.append(("unsub", [int(rng.integers(0, n_max)) for _ in range(int(rng.integers(1, 4)))]))
        elif r < 0.16:
            ids = [int(rng.integers(0, n_max + 3)) for _ in range(int(rng.integers(1, 6)))]
            ops.append(("release", ids + ids[:int(rng.integers(0, 2))]))
        elif r < 0.24:
            ops.append(("tadd", int(rng.integers(0, n_max)), int(rng.integers(2000, 20000)), int(rng.integers(0, 8)),
                        bool(rng.random() < 0.35)))
        elif r < 0.28:
            ops.append(("tcancel", int(rng.integers(0, 1 << 30))))   # an index into every timer id handed out so far
        elif r < 0.32:
            ops.append(("send", int(rng.integers(0, n_max)), int(rng.integers(0, 17)), int(rng.integers(0, 8))))
        elif r < 0.55:
            now += int(rng.integers(1, 3000)) * (40 if rng.random() < 0.03 else 1)
            ops.append(("adv", now))
        elif r < 0.60:
            ops.append(("drain", int(rng.integers(0, n_max)), int(rng.integers(1, 40))))
        elif r < 0.63:
            ids = [int(rng.integers(0, n_max + 3)) for _ in range(int(rng.integers(1, 6)))]
            ids += ids[:int(rng.integers(0, 2))]
            ops.append(("ack", ids, [int(rng.integers(0, 6)) for _ in ids]))
        else:
            ops.append(("pub", int(rng.integers(0, 17)), int(rng.integers(0, 8))))
    return ops


class _Model:
    """What the test knows beyond the oracle: publish counts by {code, source} (Metric excluded), publishes and sends, the
    records each mailbox holds taken and not acked, and the stats a fresh bus starts with (no string is interned here)"""

    def __init__(self, bus):
        self.pairs, self.publishes, self.held, self.fresh = Counter(), 0, {}, bus.stats()


def _expected_stats(bus, orc, m, lossless):
    hw, R = orc.high_water(), bus.ring_cap
    backlog = [0 if orc.released(s) else lag_oracle.backlog(orc, s) for s in range(hw)]
    exp = {k: v for k, v in m.fresh.items() if k not in LAUNCH_SHAPED}
    exp.update(publishes=m.publishes, deliveries=orc.total_deliveries(), ticks=orc.total_ticks(),
               overwritten=0 if lossless else sum(max(0, b - R) for b in backlog),
               published_by_code=[orc.published_by_code(c) for c in range(17)],
               n_subs=sum(orc.active(s) for s in range(hw)), n_timers=orc.n_timers(), now_ns=orc.now())
    return exp, backlog


def _compare(bus, orc, m, lossless, where):
    """every mailbox's count, digest and window, the stats but the launch-shaped ones, debug events, publish counts,
    lagging entries and summary, and (lossless) blockers, against the oracle and the model"""
    hw, R = orc.high_water(), bus.ring_cap
    got = bus.digests(0, hw)
    for s in range(hw):
        assert (int(got["count"][s]), int(got["digest"][s])) == (orc.count(s), orc.digest(s)), f"{where}: subscriber {s}"
        w = orc.mailbox(s)[-R:]
        rc, win = _st(bus.peek_window, s)
        if orc.released(s):
            assert rc == nat.ENOENT and len(w) == 0, f"{where}: released {s}"
        else:
            assert win.tobytes() == w[len(w) - len(win):].tobytes() and len(win) == min(len(w), R), where
    exp, backlog = _expected_stats(bus, orc, m, lossless)
    assert {k: v for k, v in bus.stats().items() if k not in LAUNCH_SHAPED} == exp, where
    assert [tuple(r) for r in bus.debug_events()[["code", "source_id"]]] == \
        [tuple(r) for r in orc.debug_events()[["code", "source_id"]]], where
    assert bus.publish_counts() == dict(m.pairs), where
    ent, _, summary = bus.lagging(0, hw, 0, min_backlog=0)
    want = [(s, min(backlog[s], R), max(0, backlog[s] - R)) for s in range(hw) if orc.active(s)]
    assert [(int(e["sub_id"]), int(e["backlog"]), int(e["lost"])) for e in ent] == want, where
    assert summary["active"] == len(want) and summary["backlog_total"] == sum(b for _, b, _ in want), where
    if lossless:   # the next flush's unit: one staged record, with the ticks due by the clock
        assert bus.publish(3, 1) == nat.OK and orc.publish(3, 1) == 0
        m.pairs[(3, 1)] += 1; m.publishes += 1
        assert list(bus.blockers()) == list(lag_oracle.blockers(orc, orc.now())), where


def _run(bus, orc, ops, lossless, rng, m):
    tids = []

    def drained(sub, n):   # a drain reads from head, held records first
        m.held[sub] = max(0, m.held.get(sub, 0) - n)

    for i, op in enumerate(ops):
        k, where = op[0], f"op {i} {op}"
        if k == "list":
            rc, ids = _st(bus.subscribe_list, op[1], op[2])
            orc_rc, orc_ids = orc.subscribe_list(op[1], op[2])
            assert rc == orc_rc and (ids is None or list(ids) == orc_ids), where
            for sid in orc_ids:
                m.held[sid] = 0
        elif k == "sub":
            fn = (lambda: bus.subscribe_pairs(op[1], op[2])) if op[2] else (lambda: bus.subscribe(op[1]))
            rc, sid = _st(fn)
            if orc.high_water() < orc.n_max:
                assert sid == orc.subscribe(op[1], op[2]), where
            else:
                assert rc == nat.ENOSPC, where
        elif k == "unsub":
            assert list(bus.unsubscribe_many(op[1])) == [orc.unsubscribe(s) for s in op[1]], where
        elif k == "release":
            if lossless and rng.random() < 0.5:   # records taken and never acked go with the mailbox
                _take(bus, orc, m)
            assert list(bus.release_many(op[1])) == orc.release_many(op[1]), where
        elif k == "ack":
            if not lossless:
                continue
            _take(bus, orc, m)
            want = []
            for sid, cnt in zip(op[1], op[2]):
                if sid >= orc.high_water() or orc.released(sid):
                    want.append(nat.ENOENT)
                elif cnt > m.held.get(sid, 0):
                    want.append(nat.EINVAL)
                else:   # ack(id, k) leaves the state drain(id, cap = k) would
                    want.append(nat.OK)
                    m.held[sid] -= cnt
                    orc.consume(sid, cnt)
            assert list(bus.ack_many(op[1], op[2])) == want, where
        elif k == "tadd":
            rc, tid = _st(bus.timer_add, op[1], op[2], op[3], op[4])
            orc_rc, orc_tid = orc.timer_add(op[1], op[2], op[3], op[4])
            assert (rc, tid) == (orc_rc, orc_tid), where
            if tid is not None:
                tids.append(tid)
        elif k == "tcancel" and tids:
            tid = tids[op[1] % len(tids)]
            assert _st(bus.timer_cancel, tid)[0] == orc.timer_cancel(tid), where
        elif k == "send":
            rc = bus.send(op[1], op[2], op[3])
            assert rc == orc.receive(op[1], op[2], op[3]), where
            m.publishes += rc == nat.OK
        elif k == "adv":
            assert bus.advance(op[1]) == nat.OK and orc.advance(op[1]) == 0, where
        elif k == "drain":
            assert bus.flush() == nat.OK, where   # (the oracle delivers at once; the bus at its flush)
            rc, recs = _st(bus.drain, op[1], op[2])
            if orc.released(op[1]) or op[1] >= orc.high_water():
                assert rc == nat.ENOENT, where
            else:
                assert rc == nat.OK, where
                assert recs.tobytes() == orc.consume(op[1], op[2]).tobytes(), where
                drained(op[1], len(recs))
        elif k == "pub":
            assert bus.publish(op[1], op[2]) == nat.OK and orc.publish(op[1], op[2]) == 0, where
            m.publishes += 1
            if op[1] != 13:   # Metric is not counted
                m.pairs[(op[1], op[2])] += 1
        if lossless and i % 50 == 49:   # consumers keep up: the lossless trace never stalls
            assert bus.flush() == nat.OK, where
            for s in range(orc.high_water()):
                if not orc.released(s):
                    orc.consume(s, 1 << 20)
            bus.consume_all()
            m.held = {}
    assert bus.flush() == nat.OK
    bus.sync()


def _take(bus, orc, m):
    """take every mailbox's records (the caps hold them all): each one's backlog is now held"""
    hw = orc.high_water()
    if not hw:
        return
    assert bus.flush() == nat.OK
    bus.take_ready(0, hw, 0, hw * bus.ring_cap, hw)
    for s in range(hw):
        m.held[s] = 0 if orc.released(s) else lag_oracle.backlog(orc, s)


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("mode", list(MODES))
def test_reuse_against_oracle(mode, K, lossless):
    seed = 500 + 10 * K + 2 * list(MODES).index(mode) + lossless
    n_max, R = 40, 1024
    # throughput: the oracle keeps a ring of R, so that its consume skips what the bus overwrote; lossless: its mailboxes
    # hold R, so that the lag extension finds the same blockers
    orc = (DropReuseOracle if mode == "drop_missed" else ro.ReuseOracle)(
        n_max, timers_per_sub=K, keep_window=0 if lossless else R, mailbox_cap=R if lossless else 0)
    orc.n_max = n_max
    with Bus(n_max, ring_cap=R, batch_cap=32, timers_per_sub=K, lossless=lossless, device=0, **MODES[mode]) as bus:
        m = _Model(bus)
        _run(bus, orc, _trace(seed, n_max=n_max), lossless, np.random.default_rng(seed), m)
        _compare(bus, orc, m, lossless, f"{mode} K={K}")
        if lossless:   # what the oracle consumed the bus drained; what is left is each mailbox's backlog
            assert bus.flush() == nat.OK
            for s in range(orc.high_water()):
                if not orc.released(s):
                    assert bus.drain(s, R).tobytes() == orc.consume(s, R).tobytes(), s


def test_churn_past_capacity():
    """100 rounds of releasing and re-subscribing about half of a 4,096-subscriber fleet: no CPBUS_ENOSPC, the ids stay
    below 4,096, and every delivery matches the oracle"""
    N, R = 4096, 64
    rng = np.random.default_rng(7)
    orc = ro.ReuseOracle(N, timers_per_sub=1, keep_window=R)
    with Bus(N, ring_cap=R, batch_cap=32, timers_per_sub=1, device=0) as bus:
        model = _Model(bus)
        masks = [int(x) for x in rng.integers(0, 1 << 17, N)]
        assert list(bus.subscribe_list(masks)) == orc.subscribe_list(masks)[1] == list(range(N))
        for rnd in range(100):
            gone = [int(x) for x in rng.choice(N, int(rng.integers(N // 3, 2 * N // 3)), replace=False)]
            assert (bus.unsubscribe_many(gone) == nat.OK).all() and (bus.release_many(gone) == nat.OK).all()
            for s in gone:
                assert orc.unsubscribe(s) == 0 and orc.release_many([s]) == [0]
            m = [int(x) for x in rng.integers(0, 1 << 17, len(gone))]
            ids = bus.subscribe_list(m)
            assert list(ids) == orc.subscribe_list(m)[1] == sorted(gone), rnd
            for _ in range(3):
                c, s = int(rng.integers(0, 17)), int(rng.integers(0, 8))
                assert bus.publish(c, s) == nat.OK and orc.publish(c, s) == 0
                model.publishes += 1
                if c != 13:
                    model.pairs[(c, s)] += 1
            t = int(rng.integers(0, N))
            rc, tid = _st(bus.timer_add, t, 1000, 5, True)
            assert (rc, tid) == orc.timer_add(t, 1000, 5, True)
            now = 2000 * (rnd + 1)
            assert bus.advance(now) == nat.OK and orc.advance(now) == 0
            assert orc.high_water() == N
            assert _st(bus.subscribe_list, [0])[0] == nat.ENOSPC
        assert bus.flush() == nat.OK
        bus.sync()
        _compare(bus, orc, model, False, "churn")


def test_stream_shard_with_outstanding_followers():
    """A shard that follows a stream (cpbus_stream_fanout_next) without being told the batches' shapes, with followers still
    queued when release_many and subscribe_list are called: each call resolves them first, so every batch followed before
    it is delivered before it, and the batches after it reach the new occupants of the released slots as the oracle says"""
    N, spare, B, dt, period = 48, 8, 64, 40_000, 90_000
    rng = np.random.default_rng(21)
    masks = [nat.MASK_ALL if rng.random() < 0.5 else int(x) for x in rng.integers(0, 1 << 17, N)]
    orc = ro.ReuseOracle(N + spare, timers_per_sub=1, keep_window=1024)
    bus = Bus(N + spare, ring_cap=1024, batch_cap=B, timers_per_sub=1, device=0)
    st, _ = bus.stream_create(8, 1)
    try:
        assert list(bus.subscribe_list(masks)) == orc.subscribe_list(masks)[1]
        for i in range(0, N, 2):
            assert _st(bus.timer_add, i, period, 7000 + i) == orc.timer_add(i, period, 7000 + i)
        j = 0

        def follow(k):   # put k batches and queue a follower for each; the oracle delivers them at once
            nonlocal j
            for _ in range(k):
                n = int(rng.integers(1, B + 1))
                ev = np.zeros(n, dtype=EVENT_DTYPE)
                ev["code"], ev["source_id"] = rng.integers(0, 17, n), rng.integers(0, 8, n)
                w = (j + 1) * dt
                nat.check(bus.stream_put(st, ev, w, nowait=True), "cpbus_stream_put")
                nat.check(bus.stream_fanout_next(st), "cpbus_stream_fanout_next")
                assert orc.advance(w) == 0
                for c, s_ in zip(ev["code"], ev["source_id"]):
                    assert orc.publish(int(c), int(s_)) == 0
                j += 1

        gone = [int(x) for x in np.sort(rng.choice(N, 12, replace=False))]
        follow(2)
        assert list(bus.unsubscribe_many(gone)) == [orc.unsubscribe(s) for s in gone] == [nat.OK] * 12
        follow(3)
        follow(2)
        assert list(bus.release_many(gone + gone[:2])) == orc.release_many(gone + gone[:2])
        follow(3)
        new_masks = [nat.MASK_ALL] * 6 + [1 << 3] * 6 + [0, nat.MASK_ALL]
        pairs = [[] if i % 3 else [(5, 2), (6, 1)] for i in range(len(new_masks))]
        ids = bus.subscribe_list(new_masks, pairs)
        assert list(ids) == orc.subscribe_list(new_masks, pairs)[1] == gone + [N, N + 1]
        follow(2)
        assert _st(bus.timer_add, int(ids[0]), period, 42) == orc.timer_add(int(ids[0]), period, 42)
        follow(4)
        assert bus.stream_status(st) == nat.OK
        hw = orc.high_water()
        got = bus.digests(0, hw)
        for s in range(hw):
            assert (int(got["count"][s]), int(got["digest"][s])) == (orc.count(s), orc.digest(s)), s
            assert bus.peek_window(s).tobytes() == orc.mailbox(s)[-1024:].tobytes(), s
        sts = bus.stats()
        assert (sts["deliveries"], sts["ticks"], sts["now_ns"]) == (orc.total_deliveries(), orc.total_ticks(), j * dt)
        assert sts["n_subs"] == N + 2 and bus.stream_poll(st) is None
    finally:
        bus.stream_close(st)
        bus.close()


def test_stale_timer_id_of_previous_occupant():
    with Bus(4, ring_cap=64, batch_cap=32, timers_per_sub=2, device=0) as bus:
        a, b = bus.subscribe_list([nat.MASK_ALL, nat.MASK_ALL])
        old = bus.timer_add(int(a), 1000, 7)
        bus.unsubscribe(int(a))
        assert list(bus.release_many([a, a, b, 9])) == [nat.OK, nat.ENOENT, nat.EINVAL, nat.ENOENT]
        (c,) = bus.subscribe_list([0])
        assert c == a
        new = bus.timer_add(int(c), 1000, 8)
        assert new & ((1 << 26) - 1) == old & ((1 << 26) - 1) and new != old   # same slot, next generation
        assert _st(bus.timer_cancel, old)[0] == nat.ENOENT
        assert list(bus.timer_cancel_many([old])) == [nat.ENOENT]
        assert bus.stats()["n_timers"] == 1
        assert bus.advance(1500) == nat.OK and bus.flush() == nat.OK
        recs = bus.drain(int(c))
        assert len(recs) == 1 and recs[0]["source_id"] == 8
        assert _st(bus.timer_cancel, new)[0] == nat.OK


def test_lossless_held_records_and_room():
    """Records taken and not acked in a released mailbox are gone and ack_many of its id is refused; a subscriber that reuses
    a slot whose old mailbox was full starts with ring_cap slots of room, and admission and blockers agree"""
    R = 64
    with Bus(4, ring_cap=R, batch_cap=32, timers_per_sub=1, lossless=True, device=0) as bus:
        ids = bus.subscribe_list([nat.MASK_ALL] * 3)
        ev = np.zeros(R, dtype=EVENT_DTYPE)
        ev["code"] = 3
        assert bus.publish_many(ev) == nat.OK and bus.flush() == nat.OK                 # every mailbox full
        bus.take_ready(0, 3, 0, 4 * R, 4)                                               # taken, not acked
        bus.unsubscribe(int(ids[1]))
        assert list(bus.release_many([ids[1]])) == [nat.OK]
        assert list(bus.ack_many([ids[1], ids[0]], [1, 1])) == [nat.ENOENT, nat.OK]
        (x,) = bus.subscribe_list([nat.MASK_ALL])
        assert x == ids[1] and len(bus.peek_window(int(x))) == 0
        assert bus.digests(int(x), 1)["count"][0] == 0
        bus.consume_all()
        assert bus.publish_many(ev) == nat.OK and bus.flush() == nat.OK                 # the new occupant takes R records
        assert bus.digests(int(x), 1)["count"][0] == R and len(bus.blockers()) == 0
        assert bus.publish(3, 1) == nat.OK and bus.flush() == nat.EAGAIN
        assert list(bus.blockers()) == [0, int(x), 2]
        ent, _, _ = bus.lagging(0, 3, 0, min_backlog=R)
        assert [int(e["sub_id"]) for e in ent] == [0, int(x), 2]


def test_lossless_eagain_applies_nothing():
    R = 64
    with Bus(8, ring_cap=R, batch_cap=32, timers_per_sub=1, lossless=True, device=0) as bus:
        bus.subscribe_list([nat.MASK_ALL] * 4)
        bus.unsubscribe_many([1, 2])
        ev = np.zeros(R, dtype=EVENT_DTYPE)
        ev["code"] = 3
        assert bus.publish_many(ev) == nat.OK and bus.flush() == nat.OK
        assert bus.publish_many(ev[:3]) == nat.OK                                       # staged behind full mailboxes
        ids = np.array([1, 2, 0, 9], dtype=np.uint32)
        status, applied = np.full(4, 99, dtype=np.int32), C.c_uint32(77)
        assert bus._lib.cpbus_release_many(bus._h, ids.ctypes.data, 4, status.ctypes.data, C.byref(applied)) == nat.EAGAIN
        assert (status == 99).all() and applied.value == 77
        out = np.full(2, 5, dtype=np.uint32)
        masks = np.zeros(2, dtype=np.uint32)
        assert bus._lib.cpbus_subscribe_list(bus._h, masks.ctypes.data, None, None, 2, out.ctypes.data) == nat.EAGAIN
        assert (out == 5).all() and bus.stats()["n_subs"] == 2
        assert list(bus.release_many([0, 9])) == [nat.EINVAL, nat.ENOENT]               # every element refused: no flush
        bus.consume_all()
        assert list(bus.release_many(ids)) == [nat.OK, nat.OK, nat.EINVAL, nat.ENOENT]
        assert list(bus.subscribe_list([0, 0, 0])) == [1, 2, 4]


def test_one_launch_per_applied_call():
    with Bus(64, ring_cap=64, batch_cap=32, timers_per_sub=2, device=0) as bus:
        bus.subscribe_list([nat.MASK_ALL] * 32)
        bus.unsubscribe_many(list(range(0, 32, 2)))

        def launches():
            return bus.stats()["kernel_launches"]

        for call, n in ((lambda: bus.release_many([1, 3, 40]), 0),                    # refused: no launch
                        (lambda: bus.release_many([]), 0),
                        (lambda: bus.release_many(list(range(0, 32, 2)) + [0]), 1),
                        (lambda: bus.subscribe_list([0] * 20), 1),
                        (lambda: _st(bus.subscribe_list, [0] * 40), 0)):               # ENOSPC
            before = launches()
            call()
            assert launches() - before == n


def _group_trace(seed):
    return [op for op in _trace(seed, n_max=40) if op[0] != "sub"]


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("G", [1, 2, 3, 4])
def test_group_equals_one_bus(G, lossless):
    ops = _group_trace(900 + G)
    kw = dict(ring_cap=128, batch_cap=32, timers_per_sub=2, lossless=lossless)
    tids = {0: [], 1: []}
    with Bus(40, device=0, **kw) as one, GroupBus(40, [0] * G, **kw) as grp:
        for i, op in enumerate(ops):
            res = []
            for j, bus in enumerate((one, grp)):
                k = op[0]
                if k == "list":
                    r = _st(bus.subscribe_list, op[1], op[2])
                elif k == "unsub":
                    r = _st(bus.unsubscribe_many, op[1])
                elif k == "release":
                    r = _st(bus.release_many, op[1])
                elif k == "tadd":
                    r = _st(bus.timer_add, op[1], op[2], op[3], op[4])
                    if r[1] is not None:
                        tids[j].append(r[1])
                elif k == "tcancel":
                    r = _st(bus.timer_cancel, tids[j][op[1] % len(tids[j])]) if tids[j] else None
                elif k == "send":
                    r = _st(bus.send, op[1], op[2], op[3])
                elif k == "adv":
                    r = _st(bus.advance, op[1])
                elif k == "drain":
                    r = _st(bus.drain, op[1], op[2])
                elif k == "ack":   # (throughput mode refuses it, lossless statuses: nothing was taken)
                    r = _st(bus.ack_many, op[1], op[2])
                else:
                    r = _st(bus.publish, op[1], op[2])
                if lossless and i % 40 == 39:
                    bus.consume_all()
                res.append(r)
            a, b = res
            assert (a is None) == (b is None), f"op {i} {op}"
            if a is not None:
                assert a[0] == b[0] and (a[1] is None) == (b[1] is None), f"op {i} {op}: {a} vs {b}"
                if a[1] is not None:
                    assert np.asarray(a[1]).tobytes() == np.asarray(b[1]).tobytes(), f"op {i} {op}"
        for bus in (one, grp):
            assert bus.flush() == nat.OK
        assert one.digests(0, 40).tobytes() == grp.digests(0, 40).tobytes()
        sa, sb = one.stats(), grp.stats()
        assert {k: v for k, v in sa.items() if k not in LAUNCH_SHAPED} == {k: v for k, v in sb.items() if k not in LAUNCH_SHAPED}
        ra, rb = one.drain_ready(0, 40, 0, 64 * 128, 40), grp.drain_ready(0, 40, 0, 64 * 128, 40)
        assert ra[0].tobytes() == rb[0].tobytes() and ra[1].tobytes() == rb[1].tobytes()


def test_scale_fleet_of_2_20():
    """A 2^20 fleet releases and re-subscribes 10^5 scattered ids: the same ids as the oracle, and the same deliveries on
    sampled ids and in the digest fold"""
    N, R = 1 << 20, 64
    rng = np.random.default_rng(12)
    masks = rng.integers(0, 1 << 17, N).astype(np.uint32)
    orc = ro.ReuseOracle(N, keep_window=1)
    with Bus(N, ring_cap=R, batch_cap=32, device=0) as bus:
        bus.subscribe_many(masks)
        assert orc.subscribe_list([int(m) for m in masks])[0] == 0
        for c in (1, 5, 9):
            assert bus.publish(c, 2) == nat.OK and orc.publish(c, 2) == 0
        gone = np.sort(rng.choice(N, 100_000, replace=False)).astype(np.uint32)
        assert (bus.unsubscribe_many(gone) == nat.OK).all() and (bus.release_many(gone) == nat.OK).all()
        for s in gone:
            orc.unsubscribe(int(s))
        assert orc.release_many(gone) == [0] * len(gone)
        new_masks = rng.integers(0, 1 << 17, len(gone)).astype(np.uint32)
        ids = bus.subscribe_list(new_masks)
        assert (ids == gone).all() and orc.subscribe_list([int(m) for m in new_masks])[1] == [int(x) for x in gone]
        for c in (5, 11):
            assert bus.publish(c, 3) == nat.OK and orc.publish(c, 3) == 0
        assert bus.flush() == nat.OK
        bus.sync()
        got = bus.digests(0, N)
        sample = np.concatenate([gone[::50], rng.choice(N, 2000, replace=False)])
        for s in sample:
            assert (int(got["count"][s]), int(got["digest"][s])) == (orc.count(int(s)), orc.digest(int(s))), int(s)
        fold = bus.digest_fold(0, N)
        assert fold[0] == int(got["count"].sum()) == sum(orc.count(s) for s in range(N))
        assert fold[1] == sum(orc.digest(s) for s in range(N)) % (1 << 64)
        assert bus.stats()["n_subs"] == N


def test_cpp_mirror_reuse_ids():
    """csrc/host/events_reuse_test: EventBus::ReuseIds, 10^5 Subscribe / Unsubscribe cycles on a 4,096-subscriber bus"""
    exe = os.path.join(ROOT, "containerpilot_b200", "csrc", "host", "events_reuse_test")
    assert os.path.exists(exe), "built by the host Makefile"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout + r.stderr
