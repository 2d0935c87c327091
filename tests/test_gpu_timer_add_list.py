"""Bulk timer arming (cpbus_timer_add_list, cpbus_group_timer_add_list; Bus.timer_add_list and GroupBus.timer_add_list) on
the GPU.  The contract is loop equivalence: a bus that arms a list in one call and a twin that calls cpbus_timer_add for
each element in order give the same statuses and ids and the same results afterwards, on everything but the launch-shaped
stats.  Random traces interleave publishes, sends, single timer adds and cancels, clock steps (some long), drains,
unsubscribes and list calls whose elements hold unknown ids, closed owners, period 0, one owner repeated past K, owners
whose one-shot has just fired, periodic and one-shot timers; in throughput and lossless mode, dense and sparse, with and
without dropped missed ticks.  Then every id handed out, stale ones included, is cancelled on both buses.  Also: the
oracle, lossless CPBUS_EAGAIN with nothing applied, the one-launch cost, the group against one bus, and a fleet of 2^20."""
import ctypes as C

import numpy as np
import pytest

import oracle_binding as ob
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from containerpilot_b200.group import GroupBus
from test_gpu_bulk_membership import LAUNCH_SHAPED, MODES, _call, _drains, _eq, _state

pytestmark = pytest.mark.gpu
REFUSED = (nat.EINVAL, nat.ENOSPC, nat.ENOENT, nat.ECLOSED)


def _trace(seed, K, n0=24, n_ops=700, max_subs=64, n_unknown=3):
    """Publishes, sends, single timer adds and cancels, clock steps, drains, unsubscribes, bulk cancels and list calls.
    A list element is (owner, period, source, oneshot); owners include ids never handed out, and some periods are 0."""
    rng = np.random.default_rng(seed)
    ops, n_total, n_handles, now = [], 0, 0, 0

    def sub():
        m = nat.MASK_ALL if rng.random() < 0.4 else int(rng.integers(0, 1 << 17))
        if rng.random() < 0.3:
            pairs = [(int(rng.integers(0, 17)), int(rng.integers(0, 16))) for _ in range(int(rng.integers(1, 6)))]
            return ("sub", m & int(rng.integers(0, 1 << 17)), pairs)
        return ("sub", m)

    def spec(owner=None):
        s = int(rng.integers(0, n_total + n_unknown)) if owner is None else owner
        period = 0 if rng.random() < 0.05 else int(rng.integers(500, 20000))
        return (s, period, int(rng.integers(1000, 1100)), bool(rng.random() < 0.35))

    for _ in range(n0):
        ops.append(sub()); n_total += 1
    for _ in range(n_ops):
        r = rng.random()
        if r < 0.04 and n_total < max_subs:
            ops.append(sub()); n_total += 1
        elif r < 0.09:
            ops.append(("tadd",) + spec(int(rng.integers(0, n_total))))
            n_handles += 1
        elif r < 0.11 and n_handles:
            ops.append(("tcancel", int(rng.integers(0, n_handles))))
        elif r < 0.12:
            ops.append(("unsub", int(rng.integers(0, n_total))))
        elif r < 0.17:
            lst = [spec() for _ in range(int(rng.integers(1, 10)))]
            if rng.random() < 0.3:   # one owner past K
                s = int(rng.integers(0, n_total))
                lst += [spec(s) for _ in range(K + 1)]
            lst = [lst[i] for i in rng.permutation(len(lst))]
            ops.append(("tlist", lst)); n_handles += len(lst)
        elif r < 0.185:
            # a one-shot that fires, then a list that arms its owner again before any other call retires it
            s, p = int(rng.integers(0, n_total)), int(rng.integers(100, 2000))
            ops.append(("tadd", s, p, 999, True)); n_handles += 1
            now += p + int(rng.integers(1, 50))
            ops.append(("adv", now))
            lst = [spec(s)] + [spec() for _ in range(int(rng.integers(0, 4)))]
            ops.append(("tlist", lst)); n_handles += len(lst)
        elif r < 0.20 and n_handles:
            lst = [("h", int(rng.integers(0, n_handles))) for _ in range(int(rng.integers(1, 8)))]
            lst += [("raw", int(rng.integers(0, 1 << 32))) for _ in range(int(rng.integers(0, 2)))]
            ops.append(("cancel_many", lst))
        elif r < 0.24:
            ops.append(("send", int(rng.integers(0, n_total)), int(rng.integers(0, 17)), int(rng.integers(0, 16))))
        elif r < 0.49:
            now += int(rng.integers(1, 3000)) * (40 if rng.random() < 0.03 else 1)
            ops.append(("adv", now))
        elif r < 0.52:
            ops.append(("flush",))
        elif r < 0.57:
            first = int(rng.integers(0, n_total))
            ops.append(("drain", first, int(rng.integers(1, 80))) if rng.random() < 0.5 else
                       ("ready", first, n_total - first, first, int(rng.integers(32, 200)), int(rng.integers(1, 6))))
        else:
            ops.append(("pub", int(rng.integers(0, 17)), int(rng.integers(0, 16))))
    return ops, max_subs


def _list(bus, lst, handles):
    """the list in one call: ('status', statuses, ids) or ('rc', refusal); each element's id (None: refused) joins handles"""
    s, p, src, one = (list(x) for x in zip(*lst))
    try:
        ids, st = bus.timer_add_list(s, p, src, one)
    except nat.CpbusError as e:
        handles.extend([None] * len(lst))
        return ("rc", e.status)
    st, ids = [int(x) for x in st], [int(x) for x in ids]
    handles.extend(t if rc == nat.OK else None for rc, t in zip(st, ids))
    return ("status", st, [t if rc == nat.OK else None for rc, t in zip(st, ids)])


def _loop(bus, lst, handles):
    """the list as the loop of cpbus_timer_add, stopping at CPBUS_EAGAIN as a caller would"""
    st, ids = [], []
    for s, p, src, one in lst:
        rc, tid = _call(bus.timer_add, s, p, src, one)
        if rc not in (nat.OK,) + REFUSED:
            handles.extend([None] * len(lst))
            return ("rc", rc, st)
        st.append(rc); ids.append(tid)
    handles.extend(ids)
    return ("status", st, ids)


def _same_outcome(one_call, loop, where):
    """the list call's outcome is the loop's: the same statuses and ids, or CPBUS_EAGAIN where the loop's first element
    that got past its up-front refusals stalled"""
    if one_call[0] == "rc":
        assert loop[0] == "rc" and loop[1] == one_call[1], where
        assert all(s in REFUSED for s in loop[2]), where
    else:
        assert loop == one_call, where


def _timer_ids(lst, handles):
    return [(handles[x] if x < len(handles) and handles[x] is not None else 0xFFFFFFFF) if kind == "h" else x
            for kind, x in lst]


def _apply(bus, op, handles, loop=False):
    k = op[0]
    if k == "tlist":
        return (_loop if loop else _list)(bus, op[1], handles)
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
        rc, tid = _call(bus.timer_add, *op[1:])
        handles.append(tid)
        return rc, tid
    if k == "tcancel":
        tid = handles[op[1]] if op[1] < len(handles) else None
        return _call(bus.timer_cancel, tid) if tid is not None else (nat.OK, None)
    if k == "cancel_many":
        return _call(bus.timer_cancel_many, _timer_ids(op[1], handles))
    if k == "drain":
        return _call(bus.drain, op[1], op[2])
    if k == "ready":
        return _call(bus.drain_ready, *op[1:])
    raise ValueError(op)


def _cancel_everything(bus, handles):
    """every id handed out, stale ones included: the first half singly, the rest (with repeats) in one bulk cancel"""
    tids = [t for t in handles if t is not None]
    half = len(tids) // 2
    single = [_call(bus.timer_cancel, t)[0] for t in tids[:half]]
    return single, _call(bus.timer_cancel_many, tids[half:] + tids[:3])


def _run_twins(a, b, ops, lossless, loop_b, seed):
    """the same trace on a (list calls) and b (the loop of cpbus_timer_add, or list calls too), compared op by op, then
    every handed-out id cancelled on both and the final state compared"""
    ha, hb = [], []
    rng = np.random.default_rng(seed)
    n_subs = n_lists = n_applied = 0
    for i, op in enumerate(ops):
        ra, rb = _apply(a, op, ha), _apply(b, op, hb, loop=loop_b)
        where = f"op {i} {op}: {ra} vs {rb}"
        if op[0] == "tlist":
            (_same_outcome if loop_b else _eq)(ra, rb, where)
            n_lists += 1
            n_applied += ra[0] == "status" and nat.OK in ra[1]
        else:
            _eq(ra, rb, where)
        assert len(ha) == len(hb)
        n_subs += op[0] == "sub"
        if ra[0] == nat.EAGAIN or ra[0] == "rc":   # a stall: the consumers run
            for d in _drains(rng, n_subs):
                _eq(_apply(a, d, ha), _apply(b, d, hb), f"op {i} drain {d}")
    for j, (x, y) in enumerate(zip(_state(a, n_subs, lossless), _state(b, n_subs, lossless))):
        _eq(x, y, f"after the trace, item {j}")
    for bus in (a, b):
        bus.consume_all()
    _eq(_cancel_everything(a, ha), _cancel_everything(b, hb), "cancelling every id")
    n_timers = a.stats()["n_timers"]
    assert n_timers == b.stats()["n_timers"] and (lossless or n_timers == 0)   # (a lossless cancel can stall)
    for bus in (a, b):
        _eq(_call(bus.publish, 1, 1), (nat.OK, None), "publish after the cancels")
        bus.advance(bus.stats()["now_ns"] + 50_000)
    for j, (x, y) in enumerate(zip(_state(a, n_subs, lossless), _state(b, n_subs, lossless))):
        _eq(x, y, f"after the cancels, item {j}")
    return n_lists, n_applied


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("mode", list(MODES))
def test_list_equals_loop_of_timer_add(mode, K, lossless):
    seed = 2000 + 10 * K + 2 * list(MODES).index(mode) + lossless
    ops, n_max = _trace(seed, K)
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=K, lossless=lossless, device=0, **MODES[mode])
    with Bus(n_max, **kw) as a, Bus(n_max, **kw) as b:
        n_lists, n_applied = _run_twins(a, b, ops, lossless, True, seed)
    assert n_lists > 20 and n_applied > 3


def _oracle_trace(seed, K):
    """tr.random_ops with its timer adds gathered into list calls: the adds up to the next cancel or unsubscribe become one
    list call placed just before it, behind the publishes, sends and clock steps between them (the oracle gets the same
    order, and every owner is still subscribed when its timer is armed)"""
    ops, n_total = tr.random_ops(seed, 20, 1500, timers_per_sub=K, p_member=0.02, p_timer=0.08, p_pairs=0.3,
                                 p_send=0.05, period_min=2000)
    out, pending = [], []
    for op in ops:
        if op[0] == "tadd":
            pending.append(op[1:])
            continue
        if pending and op[0] in ("tcancel", "unsub"):
            out.append(("tlist", pending)); pending = []
        out.append(op)
    if pending:
        out.append(("tlist", pending))
    return out, n_total


@pytest.mark.parametrize("mode", ["dense", "sparse_records"])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
def test_list_against_oracle(K, mode):
    ops, n_total = _oracle_trace(90 + K, K)
    assert sum(len(op[1]) > 1 for op in ops if op[0] == "tlist") > 3
    R = 1024
    orc = ob.Oracle(n_total + 4, timers_per_sub=K, keep_window=R)
    oh, bh = [], []
    with Bus(n_total + 4, ring_cap=R, batch_cap=256, timers_per_sub=K, device=0, **MODES[mode]) as bus:
        for op in ops:
            k = op[0]
            if k == "tlist":
                for s, p, src, one in op[1]:
                    oh.append(orc.timer_add(s, p, src, one))
                s, p, src, one = (list(x) for x in zip(*op[1]))
                ids, st = bus.timer_add_list(s, p, src, one)
                assert (st == nat.OK).all()
                bh.extend(int(t) for t in ids)
            elif k == "tcancel":
                assert orc.timer_cancel(oh[op[1]]) in (0, ob.ENOENT)
                rc, _ = _call(bus.timer_cancel, bh[op[1]])
                assert rc in (nat.OK, nat.ENOENT)
            elif k == "sub":
                orc.subscribe(op[1], op[2] if len(op) > 2 else None)
                bus.subscribe_pairs(op[1], op[2]) if len(op) > 2 else bus.subscribe(op[1])
            elif k == "unsub":
                assert orc.unsubscribe(op[1]) == 0
                bus.unsubscribe(op[1])
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


def _specs(lst):
    specs = np.zeros(len(lst), dtype=nat.TIMER_SPEC_DTYPE)
    for i, (s, p, src, one) in enumerate(lst):
        specs[i] = (p, s, src, int(one), 0)
    return specs


@pytest.mark.parametrize("mode", ["dense", "sparse_records"])
def test_lossless_eagain_applies_nothing(mode):
    """A full mailbox stalls the flush that a list call runs first: CPBUS_EAGAIN, and ids, statuses and `applied` untouched,
    and both buses still alike.  After a drain the same call gives the loop's statuses and ids."""
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=2, lossless=True, device=0, **MODES[mode])
    lst = [(1, 10**9, 7, False), (5, 2 * 10**9, 8, True), (5, 3 * 10**9, 9, False), (5, 10**9, 10, False),
           (40, 10**9, 11, False), (2, 0, 12, False), (3, 5 * 10**8, 13, True)]
    with Bus(8, **kw) as a, Bus(8, **kw) as b:
        for bus in (a, b):
            bus.subscribe_many(np.full(8, nat.MASK_ALL, dtype=np.uint32))
            for s in range(8):
                bus.timer_add(s, 10**9, 1000 + s)
            ev = np.zeros(64, dtype=EVENT_DTYPE)
            ev["code"] = 3
            assert bus.publish_many(ev) == nat.OK
            assert bus.flush() == nat.OK                           # every mailbox holds 64 of 64
            assert bus.publish_many(ev[:5]) == nat.OK              # staged behind the full mailboxes
        specs = _specs(lst)
        ids = np.full(len(lst), 0xABCD, dtype=np.uint32)
        status = np.full(len(lst), 99, dtype=np.int32)
        applied = C.c_uint32(77)
        rc = a._lib.cpbus_timer_add_list(a._h, specs.ctypes.data, len(lst), ids.ctypes.data, status.ctypes.data,
                                         C.byref(applied))
        assert rc == nat.EAGAIN
        assert (status == 99).all() and (ids == 0xABCD).all() and applied.value == 77
        assert a.stats()["n_timers"] == 8
        for x, y in zip(_state(a, 8, True), _state(b, 8, True)):
            _eq(x, y, "after the refused call")
        for bus in (a, b):
            bus.consume_all()
        hb = []
        loop = _loop(b, lst, hb)
        rc = a._lib.cpbus_timer_add_list(a._h, specs.ctypes.data, len(lst), ids.ctypes.data, status.ctypes.data,
                                         C.byref(applied))
        assert rc == nat.OK and list(status) == loop[1] and applied.value == loop[1].count(nat.OK)
        assert loop[1] == [nat.OK, nat.OK, nat.ENOSPC, nat.ENOSPC, nat.ENOENT, nat.EINVAL, nat.OK]
        assert [int(t) for t, s in zip(ids, status) if s == nat.OK] == [t for t in loop[2] if t is not None]
        assert [int(t) for t, s in zip(ids, status) if s != nat.OK] == [0xABCD] * 4
        for x, y in zip(_state(a, 8, True), _state(b, 8, True)):
            _eq(x, y, "final")


@pytest.mark.parametrize("mode", ["dense", "sparse_records"])
def test_one_launch_per_list_call(mode):
    """A list call that arms anything adds exactly one launch beyond its flush; one whose elements are all refused, and
    n == 0, add none.  Staged records cost the flush the twin's explicit flush costs."""
    N, K = 1000, 2
    kw = dict(ring_cap=128, batch_cap=64, timers_per_sub=K, device=0, **MODES[mode])
    rng = np.random.default_rng(12)
    owners = [int(x) for x in rng.choice(N, 300, replace=False)]
    with Bus(N, **kw) as a, Bus(N, **kw) as b:
        for bus in (a, b):
            bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
            bus.timer_add_many(0, N, 10**9, source_id0=100)
            assert bus.flush() == nat.OK

        def launches(bus):
            return bus.stats()["kernel_launches"]

        def arm(owners, period=5 * 10**8, oneshot=False):
            return lambda bus: bus.timer_add_list(owners, [period] * len(owners), [7] * len(owners), oneshot)

        # (call, whether some element gets past the up-front checks and so the call flushes)
        calls = [(arm(owners, oneshot=rng.random(300) < 0.5), True),
                 (arm(owners), True),                                     # every owner full: ENOSPC after the flush
                 (arm([N + 5, N + 9]), False),                            # every element ENOENT, no flush
                 (arm(owners[:10], period=0), False),                     # every element EINVAL, no flush
                 (arm([]), False),
                 (arm(owners[:5] + [N + 1]), True)]                       # still full: ENOSPC and ENOENT
        for j, (call, flushes) in enumerate(calls):
            for bus in (a, b):
                assert bus.publish(4, 1) == nat.OK                       # staged: the call flushes it first
            x0, y0 = launches(a), launches(b)
            if flushes:
                assert b.flush() == nat.OK
            y1 = launches(b)
            (ia, sa), (ib, sb) = call(a), call(b)
            assert sa.tobytes() == sb.tobytes() and ia.tobytes() == ib.tobytes(), j
            none_applied = not (sa == nat.OK).any()
            assert launches(b) - y1 == (0 if none_applied else 1), j
            assert launches(a) - x0 == (y1 - y0) + (0 if none_applied else 1), j
        for bus in (a, b):
            assert bus.advance(3 * 10**9) == nat.OK and bus.flush() == nat.OK
        assert a.digests(0, N).tobytes() == b.digests(0, N).tobytes()


def _group_cases():
    import torch
    cases = [[0, 0], [0, 0, 0]]
    if torch.cuda.device_count() > 1:
        cases.append([0, 1])
    return cases


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("devices", [[0, 0], [0, 0, 0], [0, 1]], ids=["2x_dev0", "3x_dev0", "dev0_dev1"])
def test_group_equals_one_bus(devices, lossless):
    if devices not in _group_cases():
        pytest.skip("needs a second GPU")
    seed = 400 + 10 * len(devices) + 5 * devices[-1] + lossless
    ops, n_max = _trace(seed, 4)
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=4, lossless=lossless)
    with Bus(n_max, device=0, **kw) as one, GroupBus(n_max, devices, **kw) as grp:
        n_lists, n_applied = _run_twins(grp, one, ops, lossless, False, seed)
    assert n_lists > 20 and n_applied > 3


def test_scale_fleet_of_2_20():
    """Arm one timer per subscriber of 2^20 in shuffled order in one list call: a period of 1-10 s per contiguous chunk of
    4,096 subscribers, every seventh chunk one-shot.  After clock steps the results equal a twin armed chunk by chunk with
    cpbus_timer_add_many."""
    N, chunk = 1 << 20, 1 << 12
    rng = np.random.default_rng(4)
    n_chunks = N // chunk
    period = rng.integers(1, 11, n_chunks).astype(np.uint64) * 10**9
    oneshot = np.arange(n_chunks) % 7 == 0
    src = (10 + np.arange(N)).astype(np.uint32)
    order = rng.permutation(N).astype(np.uint32)
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=1, device=0)
    with Bus(N, **kw) as a, Bus(N, **kw) as b:
        for bus in (a, b):
            bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
            assert bus.advance(123_456) == nat.OK and bus.publish(2, 1) == nat.OK
        ids, st = a.timer_add_list(order, period[order // chunk], src[order], oneshot[order // chunk])
        assert (st == nat.OK).all()
        assert (ids == (order | np.uint32(1 << 26))).all()
        for c in range(n_chunks):
            b.timer_add_many(c * chunk, chunk, int(period[c]), source_ids=src[c * chunk:(c + 1) * chunk],
                             oneshot=bool(oneshot[c]))
        for t in (500_000_000, 3_100_000_000, 7_250_000_000, 12_000_000_000, 25_000_000_001):
            for bus in (a, b):
                assert bus.advance(t) == nat.OK and bus.publish(3, 2) == nat.OK and bus.flush() == nat.OK
        for bus in (a, b):
            bus.sync()
        sa, sb = a.stats(), b.stats()
        assert sa["n_timers"] == sb["n_timers"] == N - int(oneshot.sum()) * chunk
        assert {k: v for k, v in sa.items() if k not in LAUNCH_SHAPED} == {k: v for k, v in sb.items() if k not in LAUNCH_SHAPED}
        assert a.digests(0, N).tobytes() == b.digests(0, N).tobytes()
        assert a.digest_fold(0, N) == b.digest_fold(0, N)
        for s in (0, 1, 4095, 4096, 777_777, N - 1):
            assert a.peek_window(s).tobytes() == b.peek_window(s).tobytes()
