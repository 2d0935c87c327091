"""The bulk membership calls (cpbus_unsubscribe_many, cpbus_set_mask_many, cpbus_timer_cancel_many; Bus.*_many and
GroupBus.*_many) on the GPU.  The contract is loop equivalence: a bus that makes the bulk call and a twin that calls the
single entry point for each id in order give the same statuses and the same results afterwards, on everything but the
launch-shaped stats.  Random traces interleave publishes, sends, timers, clock steps, drains and bulk calls whose id lists
hold duplicates, closed, unknown, fired and stale ids, in throughput and lossless mode, dense and sparse, with and without
dropped missed ticks.  Also: the oracle, lossless CPBUS_EAGAIN with nothing applied, sparse record delivery after
membership changes, the group against one bus, the one-launch cost, and a fleet of 2^20."""
import ctypes as C

import numpy as np
import pytest

import oracle_binding as ob
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from containerpilot_b200.group import GroupBus

pytestmark = pytest.mark.gpu
LAUNCH_SHAPED = ("batches", "kernel_launches", "admit_passes", "admit_skipped", "admit_partial", "device_splits")
REFUSED = (nat.ENOENT, nat.ECLOSED)
MODES = {"dense": {}, "sparse_ticks": {"sparse_ticks": True}, "sparse_records": {"sparse_records": True},
         "drop_missed": {"drop_missed_ticks": True}}


def _call(fn, *args):
    """(status, result) of a Bus method, whether it returns a status or raises"""
    try:
        r = fn(*args)
    except nat.CpbusError as e:
        return e.status, None
    if isinstance(r, (int, np.integer)) and fn.__name__ in ("publish", "send", "advance", "flush"):
        return int(r), None
    return nat.OK, r


def _eq(a, b, where):
    if isinstance(a, np.ndarray):
        assert a.tobytes() == b.tobytes(), where
    elif isinstance(a, (tuple, list)):
        assert len(a) == len(b), where
        for x, y in zip(a, b):
            _eq(x, y, where)
    else:
        assert a == b, where


def _trace(seed, K, n0=24, n_ops=700, max_subs=64, n_unknown=3):
    """Publishes, sends, timers (periodic and one-shot), clock steps (some long), drains, single calls and bulk calls.
    Bulk id lists draw from every id ever handed out plus a few never handed out, with repeats; timer lists draw from
    every timer handle (live, fired, cancelled, or stale after its slot was re-armed) plus raw ids."""
    rng = np.random.default_rng(seed)
    ops, n_total, n_handles, now = [], 0, 0, 0

    def sub():
        m = nat.MASK_ALL if rng.random() < 0.4 else int(rng.integers(0, 1 << 17))
        if rng.random() < 0.3:   # pair-filtered: exact {code, source} cases on a narrower mask
            pairs = [(int(rng.integers(0, 17)), int(rng.integers(0, 16))) for _ in range(int(rng.integers(1, 6)))]
            return ("sub", m & int(rng.integers(0, 1 << 17)), pairs)
        return ("sub", m)

    def ids(k):
        return [int(rng.integers(0, n_total + n_unknown)) for _ in range(k)]

    for _ in range(n0):
        ops.append(sub()); n_total += 1
    for _ in range(n_ops):
        r = rng.random()
        if r < 0.04 and n_total < max_subs:
            ops.append(sub()); n_total += 1
        elif r < 0.11:
            ops.append(("tadd", int(rng.integers(0, n_total)), int(rng.integers(500, 20000)), 1000 + n_handles,
                        bool(rng.random() < 0.35)))
            n_handles += 1
        elif r < 0.13 and n_handles:
            ops.append(("tcancel", int(rng.integers(0, n_handles))))
        elif r < 0.14:
            ops.append(("unsub", int(rng.integers(0, n_total))))
        elif r < 0.155:
            k = int(rng.integers(1, 7))
            ops.append(("unsub_many", ids(k) + ids(1) * int(rng.random() < 0.5)))   # (a repeat now and then)
        elif r < 0.18:
            k = int(rng.integers(1, 10))
            lst = ids(k)
            lst += lst[:int(rng.integers(0, 3))]
            ops.append(("mask_many", lst, [int(rng.integers(0, 1 << 17)) for _ in lst]))
        elif r < 0.20 and n_handles:
            lst = [("h", int(rng.integers(0, n_handles))) for _ in range(int(rng.integers(1, 10)))]
            lst += lst[:int(rng.integers(0, 3))]
            lst += [("raw", int(rng.integers(0, 1 << 32))) for _ in range(int(rng.integers(0, 2)))]
            ops.append(("cancel_many", lst))
        elif r < 0.24:
            ops.append(("send", int(rng.integers(0, n_total)), int(rng.integers(0, 17)), int(rng.integers(0, 16))))
        elif r < 0.50:
            now += int(rng.integers(1, 3000)) * (40 if rng.random() < 0.03 else 1)
            ops.append(("adv", now))
        elif r < 0.53:
            ops.append(("flush",))
        elif r < 0.58:
            first = int(rng.integers(0, n_total))
            ops.append(("drain", first, int(rng.integers(1, 80))) if rng.random() < 0.5 else
                       ("ready", first, n_total - first, first, int(rng.integers(32, 200)), int(rng.integers(1, 6))))
        else:
            ops.append(("pub", int(rng.integers(0, 17)), int(rng.integers(0, 16))))
    return ops, max_subs


def _timer_ids(lst, handles):
    return [(handles[x] if x < len(handles) and handles[x] is not None else 0xFFFFFFFF) if kind == "h" else x
            for kind, x in lst]


def _bulk(bus, op, handles):
    """the op with one bulk call: ('status', statuses) or ('rc', refusal)"""
    k = op[0]
    try:
        if k == "unsub_many":
            st = bus.unsubscribe_many(op[1])
        elif k == "mask_many":
            st = bus.set_mask_many(op[1], op[2])
        else:
            st = bus.timer_cancel_many(_timer_ids(op[1], handles))
    except nat.CpbusError as e:
        return ("rc", e.status)
    return ("status", [int(x) for x in st])


def _loop(bus, op, handles):
    """the op as the loop of single calls, stopping at CPBUS_EAGAIN, as a caller would"""
    k = op[0]
    if k == "unsub_many":
        calls = [(bus.unsubscribe, (i,)) for i in op[1]]
    elif k == "mask_many":
        calls = [(bus.set_mask, (i, m)) for i, m in zip(op[1], op[2])]
    else:
        calls = [(bus.timer_cancel, (t,)) for t in _timer_ids(op[1], handles)]
    out = []
    for fn, args in calls:
        rc, _ = _call(fn, *args)
        if rc not in (nat.OK,) + REFUSED:
            return ("rc", rc, out)
        out.append(rc)
    return ("status", out)


def _apply(bus, op, handles, loop=False):
    k = op[0]
    if k in ("unsub_many", "mask_many", "cancel_many"):
        return _loop(bus, op, handles) if loop else _bulk(bus, op, handles)
    if k == "sub":
        return _call(bus.subscribe_pairs, op[1], op[2]) if len(op) > 2 else _call(bus.subscribe, op[1])
    if k == "unsub":
        return _call(bus.unsubscribe, op[1])
    if k == "pub":
        return _call(bus.publish, op[1], op[2])
    if k == "send":
        return _call(bus.send, op[1], op[2], op[3])
    if k == "adv":
        return _call(bus.advance, op[1])
    if k == "flush":
        return _call(bus.flush)
    if k == "tadd":
        rc, tid = _call(bus.timer_add, op[1], op[2], op[3], op[4])
        handles.append(tid)
        return rc, tid
    if k == "tcancel":
        tid = handles[op[1]] if op[1] < len(handles) else None
        return _call(bus.timer_cancel, tid) if tid is not None else (nat.OK, None)
    if k == "drain":
        return _call(bus.drain, op[1], op[2])
    if k == "ready":
        return _call(bus.drain_ready, *op[1:])
    raise ValueError(op)


def _same_outcome(bulk, loop, where):
    """the bulk call's outcome is the loop's: the same statuses, or CPBUS_EAGAIN where the loop's first element that got
    past its refusals stalled"""
    if bulk[0] == "rc":
        assert loop[0] == "rc" and loop[1] == bulk[1], where
        assert all(s in REFUSED for s in loop[2]), where
    else:
        assert loop[0] == "status" and loop[1] == bulk[1], where


def _state(bus, n, lossless):
    res = [_call(bus.flush), _call(bus.sync), _call(bus.digests, 0, n), _call(bus.digest_fold, 0, n)]
    res += [_call(bus.peek_window, s) for s in range(n)]
    res += [_call(bus.debug_events), _call(bus.publish_counts), _call(bus.lagging, 0, n, n // 2, 1)]
    if lossless:
        res.append(_call(bus.blockers))
    st = bus.stats()
    res.append({k: v for k, v in st.items() if k not in LAUNCH_SHAPED})
    res.append(_call(bus.drain_ready, 0, n, n // 3, 4 * bus.ring_cap, 5))
    return res


def _drains(rng, n):
    first = int(rng.integers(0, n))
    return [("ready", first, n - first, first, 400, 8), ("drain", int(rng.integers(0, n)), 64)]


def _run_twins(a, b, ops, n_max, lossless, loop_b, seed):
    """the same trace on a (bulk calls) and b (the loop of single calls, or bulk calls too), compared op by op"""
    ha, hb = [], []
    rng = np.random.default_rng(seed)
    n_subs = n_bulk = n_eagain = 0
    for i, op in enumerate(ops):
        ra, rb = _apply(a, op, ha), _apply(b, op, hb, loop=loop_b)
        where = f"op {i} {op}: {ra} vs {rb}"
        if op[0] in ("unsub_many", "mask_many", "cancel_many"):
            (_same_outcome if loop_b else _eq)(ra, rb, where)
            n_bulk += 1
            n_eagain += ra[0] == "rc"
        else:
            _eq(ra, rb, where)
        n_subs += op[0] == "sub"
        if ra[0] == nat.EAGAIN or ra[0] == "rc":   # a stall: the consumers run
            for d in _drains(rng, n_subs):
                _eq(_apply(a, d, ha), _apply(b, d, hb), f"op {i} drain {d}")
        if i % 97 == 0:
            _eq(a.stats()["n_subs"], b.stats()["n_subs"], f"op {i} n_subs")
    for j, (x, y) in enumerate(zip(_state(a, n_subs, lossless), _state(b, n_subs, lossless))):
        _eq(x, y, f"final item {j}")
    return n_bulk, n_eagain


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("mode", list(MODES))
def test_bulk_equals_loop_of_single_calls(mode, K, lossless):
    seed = 1000 + 10 * K + 2 * list(MODES).index(mode) + lossless
    ops, n_max = _trace(seed, K)
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=K, lossless=lossless, device=0, **MODES[mode])
    with Bus(n_max, **kw) as a, Bus(n_max, **kw) as b:
        n_bulk, n_eagain = _run_twins(a, b, ops, n_max, lossless, True, seed)
    assert n_bulk > 20


def _oracle_trace(seed, K):
    """tr.random_ops, with each unsubscribe turned into a bulk call of the id, repeats, closed ids and unknown ids, and each
    cancel into a bulk call of the handle and its repeats.  No other timer handle: a cancelled or fired timer's slot can be
    armed again, and the oracle's timer ids carry no generation, so a stale handle would cancel the new timer there and
    nothing on the bus.  The loop-equivalence tests cancel stale handles against the single calls."""
    ops, n_total = tr.random_ops(seed, 20, 1500, timers_per_sub=K, p_member=0.03, p_timer=0.05, p_pairs=0.3,
                                 p_send=0.05, period_min=2000)
    rng = np.random.default_rng(seed ^ 0xB01C)
    out, gone = [], []
    for op in ops:
        if op[0] == "unsub":
            lst = [op[1]] + [op[1]] * int(rng.random() < 0.3) + [n_total + 2] * int(rng.random() < 0.3)
            lst += [int(rng.choice(gone)) for _ in range(int(rng.integers(0, 3)))] if gone else []
            gone.append(op[1])
            out.append(("unsub_many", [int(x) for x in rng.permutation(lst)]))
        elif op[0] == "tcancel":
            out.append(("cancel_many", [op[1]] * int(rng.integers(1, 4))))
        else:
            out.append(op)
    return out, n_total


@pytest.mark.parametrize("mode", ["dense", "sparse_ticks", "sparse_records"])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
def test_bulk_against_oracle(K, mode):
    ops, n_total = _oracle_trace(70 + K, K)
    R = 1024
    orc = ob.Oracle(n_total + 4, timers_per_sub=K, keep_window=R)
    oh, bh = [], []
    with Bus(n_total + 4, ring_cap=R, batch_cap=256, timers_per_sub=K, device=0, **MODES[mode]) as bus:
        for op in ops:
            k = op[0]
            if k == "unsub_many":
                for s in op[1]:
                    orc.unsubscribe(s)
                assert all(x in (nat.OK,) + REFUSED for x in bus.unsubscribe_many(op[1]))
            elif k == "cancel_many":
                for h in op[1]:
                    assert orc.timer_cancel(oh[h]) in (0, ob.ENOENT)
                assert all(x in (nat.OK, nat.ENOENT) for x in bus.timer_cancel_many([bh[h] for h in op[1]]))
            elif k == "tadd":
                oh.append(orc.timer_add(op[1], op[2], op[3], op[4]))
                bh.append(bus.timer_add(op[1], op[2], op[3], op[4]))
            else:
                if k == "sub":
                    orc.subscribe(op[1], op[2] if len(op) > 2 else None)
                    bus.subscribe_pairs(op[1], op[2]) if len(op) > 2 else bus.subscribe(op[1])
                elif k == "pub":
                    assert orc.publish(op[1], op[2]) == 0
                    nat.check(bus.publish(op[1], op[2]), "publish")
                elif k == "send":
                    assert orc.receive(op[1], op[2], op[3]) == 0
                    nat.check(bus.send(op[1], op[2], op[3]), "send")
                elif k == "adv":
                    assert orc.advance(op[1]) == 0
                    nat.check(bus.advance(op[1]), "advance")
                elif k == "flush":
                    nat.check(bus.flush(), "flush")
        nat.check(bus.flush(), "flush")
        bus.sync()
        tr.compare(bus, orc, n_total, window=R)


def _raw(bus, name, arrays, status, applied):
    return getattr(bus._lib, name)(bus._h, *[a.ctypes.data for a in arrays], arrays[0].size, status.ctypes.data,
                                   C.byref(applied))


@pytest.mark.parametrize("mode", ["dense", "sparse_records"])
def test_lossless_eagain_applies_nothing(mode):
    """A full mailbox stalls the flush that a bulk call runs first: CPBUS_EAGAIN, statuses and `applied` untouched, every
    id still subscribed and every timer armed.  After a drain the same call gives the loop's results."""
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=2, lossless=True, device=0, **MODES[mode])
    with Bus(8, **kw) as a, Bus(8, **kw) as b:
        handles = {}
        for bus in (a, b):
            bus.subscribe_many(np.full(8, nat.MASK_ALL, dtype=np.uint32))
            handles[id(bus)] = [bus.timer_add(s, 10**9, 1000 + s) for s in range(8)]
            ev = np.zeros(64, dtype=EVENT_DTYPE)
            ev["code"] = 3
            assert bus.publish_many(ev) == nat.OK
            assert bus.flush() == nat.OK                           # every mailbox holds 64 of 64
            assert bus.publish_many(ev[:5]) == nat.OK              # staged behind the full mailboxes
        ids = np.array([1, 5, 5, 40, 2], dtype=np.uint32)
        masks = np.array([0, 6, 7, 1, 8], dtype=np.uint32)
        tids = np.array(handles[id(a)][:3] + [handles[id(a)][0]], dtype=np.uint32)
        status = np.full(5, 99, dtype=np.int32)
        applied = C.c_uint32(77)
        for name, arrays in (("cpbus_unsubscribe_many", [ids]), ("cpbus_set_mask_many", [ids, masks]),
                             ("cpbus_timer_cancel_many", [tids])):
            assert _raw(a, name, arrays, status[:arrays[0].size], applied) == nat.EAGAIN, name
            assert (status == 99).all() and applied.value == 77
        assert a.stats()["n_subs"] == 8 and a.stats()["n_timers"] == 8
        for bus in (a, b):
            bus.consume_all()
        b_st = [_call(b.set_mask, int(i), int(m))[0] for i, m in zip(ids, masks)]
        assert _raw(a, "cpbus_set_mask_many", [ids, masks], status, applied) == nat.OK
        assert list(status) == b_st and applied.value == b_st.count(nat.OK)
        b_st = [_call(b.timer_cancel, int(t))[0] for t in np.array(handles[id(b)][:3] + [handles[id(b)][0]], dtype=np.uint32)]
        assert list(a.timer_cancel_many(tids)) == b_st == [nat.OK, nat.OK, nat.OK, nat.ENOENT]
        b_st = [_call(b.unsubscribe, int(i))[0] for i in ids]
        assert list(a.unsubscribe_many(ids)) == b_st == [nat.OK, nat.OK, nat.ECLOSED, nat.ENOENT, nat.OK]
        for x, y in zip(_state(a, 8, True), _state(b, 8, True)):
            _eq(x, y, "final")


def test_sparse_records_after_membership_changes():
    """CPBUS_CFG_SPARSE_RECORDS keeps a per-code list while a code has at most `keep` = 64 subscribers (4,096 subscribers).
    Bulk unsubscribes and re-masks move code 5 across that threshold both ways; after each change a publish of code 5 reaches
    exactly the mailboxes that a looping twin's publish and a dense bus's reach, and takes the sparse path (one launch over
    a plan) once at most 32 subscribers are left."""
    N = 4096
    rng = np.random.default_rng(5)
    masks = np.zeros(N, dtype=np.uint32)
    takers = rng.choice(N, 100, replace=False)
    masks[takers] = 1 << 5
    others = np.setdiff1d(np.arange(N), takers)
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=1, device=0)
    with Bus(N, sparse_records=True, **kw) as a, Bus(N, sparse_records=True, **kw) as b, Bus(N, **kw) as c:
        for bus in (a, b, c):
            bus.subscribe_many(masks)
        steps = [("unsub_many", [int(x) for x in takers[:75]]),                                      # 100 -> 25: list rebuilt
                 ("mask_many", [int(x) for x in others[:60]], [1 << 5] * 60),                         # 25 -> 85: past keep
                 ("mask_many", [int(x) for x in others[:60]] + [int(takers[80])], [0] * 61),           # 85 -> 24
                 ("unsub_many", [int(x) for x in takers[75:79]] + [int(takers[0])])]                  # 24 -> 20
        expect = [25, 85, 24, 20]   # subscribers with code 5 after each step
        for i, op in enumerate(steps):
            ra = _apply(a, op, [])
            _same_outcome(ra, _apply(b, op, [], loop=True), f"step {i}")
            _same_outcome(ra, _apply(c, op, [], loop=True), f"step {i}")
            launches, before = a.stats()["kernel_launches"], a.digests(0, N)["count"].copy()
            for bus in (a, b, c):
                assert bus.publish(5, 9) == nat.OK and bus.flush() == nat.OK
            assert int(np.count_nonzero(a.digests(0, N)["count"] - before)) == expect[i], f"step {i}"
            if expect[i] <= 32:
                assert a.stats()["kernel_launches"] == launches + 1, f"step {i}"
            da, db, dc = a.digests(0, N), b.digests(0, N), c.digests(0, N)
            assert da.tobytes() == db.tobytes() == dc.tobytes(), f"step {i}"
        for x, y in zip(_state(a, N, False)[:4], _state(b, N, False)[:4]):
            _eq(x, y, "final")


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("G", [1, 2, 3, 4])
def test_group_equals_one_bus(G, lossless):
    seed = 300 + 10 * G + lossless
    ops, n_max = _trace(seed, 4)
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=4, lossless=lossless)
    with Bus(n_max, device=0, **kw) as one, GroupBus(n_max, [0] * G, **kw) as grp:
        n_bulk, _ = _run_twins(grp, one, ops, n_max, lossless, False, seed)
    assert n_bulk > 20


@pytest.mark.parametrize("mode", ["dense", "sparse_records"])
def test_one_launch_per_bulk_call(mode):
    """A bulk call over m distinct mailboxes adds exactly one launch beyond its flush, and none when every element is
    refused; staged records cost the flush the twin's explicit flush costs."""
    N = 1000
    kw = dict(ring_cap=128, batch_cap=64, timers_per_sub=2, device=0, **MODES[mode])
    rng = np.random.default_rng(11)
    with Bus(N, **kw) as a, Bus(N, **kw) as b:
        tids = {}
        for bus in (a, b):
            bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
            bus.timer_add_many(0, N, 10**9, source_id0=100)
            tids[id(bus)] = [bus.timer_add(s, 10**9, 7) for s in range(0, N, 3)]
            assert bus.flush() == nat.OK
        ids = [int(x) for x in rng.choice(N, 300, replace=False)]

        def launches(bus):
            return bus.stats()["kernel_launches"]

        # (call, whether some element gets past the single call's up-front checks and so the call flushes)
        calls = [(lambda bus: bus.set_mask_many(ids, [1 << 4] * len(ids)), True),
                 (lambda bus: bus.timer_cancel_many(tids[id(bus)][:200] + tids[id(bus)][:5]), True),
                 (lambda bus: bus.unsubscribe_many(ids + ids[:10]), True),
                 (lambda bus: bus.unsubscribe_many(ids), True),                   # every element ECLOSED, after the flush
                 (lambda bus: bus.unsubscribe_many([N + 5, N + 9]), False),       # every element ENOENT, no flush
                 (lambda bus: bus.timer_cancel_many(tids[id(bus)][:200]), True)]  # every element ENOENT, after the flush
        for j, (call, flushes) in enumerate(calls):
            for bus in (a, b):
                assert bus.publish(4, 1) == nat.OK                               # staged: the call flushes it first
            x0, y0 = launches(a), launches(b)
            if flushes:
                assert b.flush() == nat.OK
            y1 = launches(b)
            sa, sb = call(a), call(b)
            assert list(sa) == list(sb)
            all_refused = not any(s == nat.OK for s in sa)
            assert launches(b) - y1 == (0 if all_refused else 1), j
            assert launches(a) - x0 == (y1 - y0) + (0 if all_refused else 1), j
        assert a.digests(0, N).tobytes() == b.digests(0, N).tobytes()


def test_scale_fleet_of_2_20():
    """Unsubscribe 2^20 - 1 of 2^20 subscribers and cancel every timer, against a twin that loops the single calls"""
    N = 1 << 20
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=1, device=0)
    keep = 123457
    ids = np.array([i for i in np.random.default_rng(3).permutation(N) if i != keep], dtype=np.uint32)
    with Bus(N, **kw) as a, Bus(N, **kw) as b:
        for bus in (a, b):
            bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
            bus.timer_add_many(0, N, 5000, source_id0=10)
            assert bus.advance(12000) == nat.OK and bus.publish(2, 1) == nat.OK
        st = a.unsubscribe_many(ids)
        assert (st == nat.OK).all()
        for i in ids:
            b.unsubscribe(int(i))
        all_tids = np.arange(N, dtype=np.uint32)             # K = 1 and cpbus_timer_add_many: timer id = subscriber
        st = a.timer_cancel_many(all_tids)
        assert int(np.count_nonzero(st == nat.OK)) == 1 and st[keep] == nat.OK
        assert [_call(b.timer_cancel, int(t))[0] for t in all_tids] == [int(x) for x in st]
        for bus in (a, b):
            assert bus.advance(40000) == nat.OK and bus.publish(3, 2) == nat.OK and bus.flush() == nat.OK
            bus.sync()
        sa, sb = a.stats(), b.stats()
        assert sa["n_subs"] == sb["n_subs"] == 1 and sa["n_timers"] == sb["n_timers"] == 0
        assert {k: v for k, v in sa.items() if k not in LAUNCH_SHAPED} == {k: v for k, v in sb.items() if k not in LAUNCH_SHAPED}
        assert a.digest_fold(0, N) == b.digest_fold(0, N)
        assert a.peek_window(keep).tobytes() == b.peek_window(keep).tobytes()
        ra, rb = a.drain_ready(0, N, 0, 4096, 16), b.drain_ready(0, N, 0, 4096, 16)
        assert ra[1].tobytes() == rb[1].tobytes() and ra[0].tobytes() == rb[0].tobytes()


def test_cpp_mirror_unsubscribe_many():
    """csrc/host/events_bulk_test: EventBus::UnsubscribeMany of events.hpp on one bus and on a group of three shards"""
    import os
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "containerpilot_b200", "csrc", "host",
                       "events_bulk_test")
    assert os.path.exists(exe), "built by the host Makefile"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
