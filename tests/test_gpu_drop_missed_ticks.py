"""Periodic timers that drop missed ticks (CPBUS_CFG_DROP_MISSED_TICKS) on the GPU: a flagged bus against the flagged oracle,
flagged sparse buses against a flagged dense twin, a flagged group against a flagged single bus (return codes, drains, sparse
drains, windows, digests, folds, debug events, publish counts, lagging, blockers and the stats that are not launch-shaped),
the entry points a flagged bus refuses, the 1,000 s heartbeat step, and steps shorter than every period, which launch
exactly what an unflagged twin launches."""
import numpy as np
import pytest

import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus
from containerpilot_b200.group import GroupBus
from drop_oracle import DropOracle
from test_gpu_group import _apply, _consume, _consumers, _eq, _final, _trace

pytestmark = pytest.mark.gpu
TOP = (1 << 64) - 1
SEC = 10 ** 9


def _queries(bus, n_total):
    return [bus.lagging(0, n_total, n_total // 2, 1), bus.blockers()]


def _steps(ops, rng, t0=0, p_long=0.0):
    """the trace's clock from t0 (below 2^64 - 1); some steps land exactly on a grid point of a timer armed at the step's
    start (ties at c + k * period), and with p_long some timers are first due within 2^21 of the top"""
    out, last = [], 0
    for op in ops:
        if op[0] == "adv":
            now = min(op[1] + t0, TOP - 1)
            if rng.random() < 0.1 and out:
                periods = [o[2] for o in out if o[0] == "tadd" and o[2] != "long"]
                if periods:
                    now = min(TOP - 1, max(now, last + int(rng.choice(periods)) * int(rng.integers(2, 50))))
            last = max(last, now)
            op = ("adv", last)
        elif op[0] == "tadd" and p_long and rng.random() < p_long:
            op = ("tadd", op[1], "long", op[3], op[4])
        out.append(op)
    return out


def _resolve(op, bus):
    if op[0] == "tadd" and op[2] == "long":   # first due just short of 2^64 - 1, from the bus's own clock
        return ("tadd", op[1], max(1, TOP - bus.stats()["now_ns"] - 1 - (op[3] * 7919) % (1 << 21)), op[3], op[4])
    return op


def _twins(make_a, make_b, seed, lossless, K, R=64, B=32, n_ops=1500, jump_every=150, p_consume=0.08, t0=0, p_long=0.0):
    """One trace on two buses, every result compared; advances that return CPBUS_EAGAIN are retried after a drain, at the
    same clock or a later one.  Returns the number of CPBUS_EAGAINs from advances."""
    ops, n_total = _trace(seed, 24, n_ops, K, jump_every=jump_every)
    rng = np.random.default_rng(seed + 31)
    ops = _steps(ops, rng, t0, p_long)
    kw = dict(ring_cap=R, batch_cap=B, timers_per_sub=K, lossless=lossless, drop_missed_ticks=True)
    a, b = make_a(n_total + 4, kw), make_b(n_total + 4, kw)
    ha, hb = [], []
    n_adv_eagain = n_ids = 0
    try:
        if t0:
            assert a.advance(t0) == b.advance(t0) == nat.OK
        for i, op in enumerate(ops):
            op = _resolve(op, a)
            x, y = _apply(a, op, ha), _apply(b, op, hb)
            _eq(x, y, f"op {i} {op}: {x} vs {y}")
            n_ids += op[0] == "sub" and x[0] == nat.OK
            retries = 0
            while op[0] == "adv" and x[0] == nat.EAGAIN and retries < 8:
                n_adv_eagain += 1
                retries += 1
                for _ in range(int(rng.integers(1, 4))):
                    c = _consumers(rng, n_ids, R)
                    _eq(_consume(a, c), _consume(b, c), f"op {i} retry consumer {c}")
                if rng.random() < 0.5:   # the same clock, or a later one
                    op = ("adv", min(TOP - 1, op[1] + int(rng.integers(0, 40_000))))
                x, y = _apply(a, op, ha), _apply(b, op, hb)
                _eq(x, y, f"op {i} retry {op}: {x} vs {y}")
            if n_ids and (x[0] == nat.EAGAIN or rng.random() < p_consume):
                for _ in range(int(rng.integers(1, 4))):
                    c = _consumers(rng, n_ids, R)
                    _eq(_consume(a, c), _consume(b, c), f"op {i} consumer {c}")
            if n_ids and rng.random() < 0.02:
                for q, r in zip(_queries(a, n_ids), _queries(b, n_ids)):
                    _eq(q, r, f"op {i} queries")
        for q, r in zip(_final(a, n_ids), _final(b, n_ids)):
            _eq(q, r, "final")
        return n_adv_eagain
    finally:
        a.close(); b.close()


def _dense(n, kw):
    return Bus(n, device=0, **kw)


def _sparse(n, kw):
    return Bus(n, device=0, sparse_ticks=True, **kw)


def _sparse_records(n, kw):
    return Bus(n, device=0, sparse_records=True, **kw)


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
def test_sparse_ticks_twin_equals_dense(K, lossless):
    n = _twins(_dense, _sparse, 300 + 10 * K + lossless, lossless, K)
    if lossless:
        assert n > 0   # mailboxes kept nearly full: advances stall in their first flush or in the window split


@pytest.mark.parametrize("lossless", [False, True])
def test_sparse_records_twin_equals_dense(lossless):
    _twins(_dense, _sparse_records, 400 + lossless, lossless, 2)


@pytest.mark.parametrize("lossless", [False, True])
def test_twins_near_the_top_of_the_clock(lossless):
    _twins(_dense, _sparse, 410 + lossless, lossless, 4, n_ops=1000, t0=TOP - (1 << 22), p_long=0.3)


@pytest.mark.parametrize("env", [("CPBUS_PDL", "0"), ("CPBUS_HINTS", "2")])
@pytest.mark.parametrize("lossless", [False, True])
def test_twins_with_knobs(env, lossless, monkeypatch):
    monkeypatch.setenv(*env)
    _twins(_dense, _sparse, 420 + lossless, lossless, 4, n_ops=800)


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("G", [1, 2, 3, 4])
def test_group_equals_one_bus(G, lossless):
    n = _twins(_dense, lambda n, kw: GroupBus(n, [0] * G, **kw), 500 + 10 * G + lossless, lossless, 4, n_ops=1000)
    if lossless:
        assert n > 0


def _oracle_ops(seed, K, n_ops, jump_every=50):
    """_trace without set_mask (the oracle has no such call): clock jumps of hundreds of the shortest period"""
    ops, n_total = _trace(seed, 20, n_ops, K, jump_every=jump_every, period=(20000, 40000))
    return [op for op in ops if op[0] != "setmask"], n_total


def _oracle_apply(orc, op, handles):
    k = op[0]
    if k == "sub":
        orc.subscribe(op[1], op[2] if len(op) > 2 else None)
    elif k == "unsub":
        assert orc.unsubscribe(op[1]) == 0
    elif k == "pub":
        assert orc.publish(op[1], op[2]) == 0
    elif k == "send":
        assert orc.receive(op[1], op[2], op[3]) == 0
    elif k == "adv":
        assert orc.advance(op[1]) == 0
    elif k == "tadd":
        handles.append(orc.timer_add(op[1], op[2], op[3], op[4]))
    elif k == "tcancel":
        assert orc.timer_cancel(handles[op[1]]) in (0, tr.ob.ENOENT)


def _against_oracle(ops, n_total, K, lossless, t0=0, every=100):
    """the flagged bus and the flagged oracle through the same ops, compared every `every` calls and at the end; returns
    the bus's tick count"""
    R = 1024   # lossless: no mailbox of the oracle ever fills
    orc = DropOracle(n_total + 4, timers_per_sub=K, keep_window=R, mailbox_cap=R if lossless else 0)
    with Bus(n_total + 4, ring_cap=R, batch_cap=256, timers_per_sub=K, lossless=lossless, drop_missed_ticks=True,
             device=0) as bus:
        if t0:
            assert orc.advance(t0) == 0 and bus.advance(t0) == nat.OK
        ho, hb = [], []
        n_ids = 0
        for i, op in enumerate(ops):
            _oracle_apply(orc, op, ho)
            r = _apply(bus, op, hb)
            assert r[0] == nat.OK or (op[0] == "tcancel" and r[0] == nat.ENOENT), (i, op, r)
            n_ids += op[0] == "sub"
            if i % every == every - 1 or i == len(ops) - 1:
                assert bus.flush() == nat.OK
                bus.sync()
                tr.compare(bus, orc, n_ids, window=R)
        assert n_ids == n_total
        return bus.stats()["ticks"]


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
def test_flagged_bus_against_flagged_oracle(K, lossless):
    """every tick of a clock jump but the last is dropped on both sides"""
    ops, n_total = _oracle_ops(600 + 10 * K + lossless, K, 700 if lossless else 1500)
    ticks = _against_oracle(ops, n_total, K, lossless)
    plain = tr.run_oracle(ops, n_total + 4, timers_per_sub=K)
    assert plain.total_ticks() > ticks > 0   # the jumps dropped ticks


@pytest.mark.parametrize("lossless", [False, True])
def test_flagged_bus_against_flagged_oracle_near_the_top(lossless):
    t0 = TOP - (1 << 30)
    ops, n_total = _oracle_ops(650 + lossless, 2, 700)
    ops = [("adv", min(TOP - 1, op[1] + t0)) if op[0] == "adv" else op for op in ops]
    assert _against_oracle(ops, n_total, 2, lossless, t0=t0) > 0


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("sparse", [False, True])
def test_two_firings_coalesce_into_one(sparse, lossless):
    """Armed with period p at clock c, a step to exactly c + 2p (two firings due: the smallest step that coalesces)
    delivers one tick, seq 1 and ts c + 2p, and the next at c + 3p with seq 2; a second timer of period 2p - 1 on the same
    mailbox has one firing in the step and is left alone.  Against the flagged oracle, also near the top of the clock."""
    for c, p in ((0, 1000), (123_456, 7), (TOP - 4000, 1000)):
        N, K = 8, 2
        orc = DropOracle(N, timers_per_sub=K, keep_window=64, mailbox_cap=64 if lossless else 0)
        with Bus(N, ring_cap=64, batch_cap=32, timers_per_sub=K, lossless=lossless, sparse_ticks=sparse,
                 drop_missed_ticks=True, device=0) as bus:
            for x in (bus, orc):
                for i in range(N):
                    x.subscribe(nat.MASK_ALL)
                assert x.advance(c) == 0
                for i in range(N):
                    x.timer_add(i, p, 40 + i, False)
                x.timer_add(3, 2 * p - 1, 99, False)
            assert bus.advance(c + 2 * p) == nat.OK and bus.flush() == nat.OK and orc.advance(c + 2 * p) == 0
            bus.sync()
            tr.compare(bus, orc, N, window=64)
            for i in range(N):
                w = bus.peek_window(i)
                want = [(1, c + 2 * p, 40 + i)] if i != 3 else [(0, c + 2 * p - 1, 99), (1, c + 2 * p, 43)]
                assert [(int(r["seq"]), int(r["ts_ns"]), int(r["source_id"])) for r in w] == want, (c, p, i, w)
            if c + 3 * p < TOP:
                assert bus.advance(c + 3 * p) == nat.OK and bus.flush() == nat.OK and orc.advance(c + 3 * p) == 0
                bus.sync()
                tr.compare(bus, orc, N, window=64)
                w = bus.peek_window(0)
                assert (int(w["seq"][-1]), int(w["ts_ns"][-1])) == (2, c + 3 * p)


def _oracle_rc(orc, op, handles):
    """the oracle's status for one op (publishes, sends and advances can stall in lossless mode)"""
    k = op[0]
    if k == "pub":
        return orc.publish(op[1], op[2])
    if k == "send":
        return orc.receive(op[1], op[2], op[3])
    if k == "adv":
        return orc.advance(op[1])
    _oracle_apply(orc, op, handles)
    return 0


@pytest.mark.parametrize("env", [None, ("CPBUS_PDL", "0"), ("CPBUS_HINTS", "2")])
@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("K", [1, 4])
def test_stalls_against_flagged_oracle(K, sparse, env, monkeypatch):
    """Lossless mailboxes of 64 records kept nearly full, so that advances stall in the flush to the old clock (an advance
    with nothing flushed since the previous one) and in the window split after the catch-up.  Every call that stalls, on
    the bus or on the oracle, is retried with the same arguments after a few records of every mailbox of the side that
    stalled are drained (more on each retry, the whole mailbox at last), so mailboxes stay nearly full; once both have
    completed a call (and the bus has flushed), the delivered sequences, windows, digests and counts must be the oracle's.  (The two stall
    at different calls: the oracle fires timers when the clock moves, the bus at the next flush.)"""
    if env:
        monkeypatch.setenv(*env)
    R = 64
    ops, n_total = _oracle_ops(700 + 10 * K + sparse, K, 1500)
    rng = np.random.default_rng(K * 7 + sparse)
    orc = DropOracle(n_total + 4, timers_per_sub=K, keep_window=R, mailbox_cap=R)
    stalls = {"bus": 0, "first flush": 0, "window split": 0, "oracle": 0}
    with Bus(n_total + 4, ring_cap=R, batch_cap=32, timers_per_sub=K, lossless=True, sparse_ticks=sparse,
             drop_missed_ticks=True, device=0) as bus:
        ho, hb = [], []
        n_ids = 0

        DRAIN = (2, 4, 8, 16, R, R)   # records taken from every mailbox of the side that stalled, before retry j

        def drain_bus(cap):
            for i in range(n_ids):
                try:
                    bus.drain(i, cap)
                except nat.CpbusError:
                    pass   # (unsubscribed)

        def bus_call(fn):
            for cap in DRAIN:
                r = fn()
                if r[0] != nat.EAGAIN:
                    return r
                stalls["bus"] += 1
                drain_bus(cap)
            raise AssertionError("the bus still stalls with every mailbox drained")

        for i, op in enumerate(ops):
            for cap in DRAIN:
                rc = _oracle_rc(orc, op, ho)
                if rc != tr.ob.EAGAIN:
                    break
                stalls["oracle"] += 1
                for j in range(n_ids):
                    orc.consume(j, cap)
            assert rc == 0 or (op[0] == "tcancel" and rc == tr.ob.ENOENT), (i, op, rc)

            def once():
                c = bus.stats()["now_ns"]
                r = _apply(bus, op, hb)
                if r[0] == nat.EAGAIN:
                    if op[0] == "tadd":
                        hb.pop()   # (no timer was armed)
                    if op[0] == "adv":
                        stalls["first flush" if bus.stats()["now_ns"] == c else "window split"] += 1
                return r

            r = bus_call(once)
            assert r[0] == nat.OK or (op[0] == "tcancel" and r[0] == nat.ENOENT), (i, op, r)
            n_ids += op[0] == "sub"
            if op[0] in ("adv", "pub") and rng.random() < 0.4:
                continue   # nothing flushed: the next advance's first flush owes the ticks and records
            bus_call(lambda: (bus.flush(), None))
            if i % 40 == 39:
                bus.sync()
                tr.compare(bus, orc, n_ids, window=R)
        bus_call(lambda: (bus.flush(), None))
        bus.sync()
        tr.compare(bus, orc, n_ids, window=R)
    assert stalls["bus"] > 0 and stalls["oracle"] > 0, stalls   # (advances that stall: test_stalled_advances_against_...)


@pytest.mark.parametrize("env", [None, ("CPBUS_PDL", "0"), ("CPBUS_HINTS", "2")])
@pytest.mark.parametrize("sparse", [False, True])
def test_stalled_advances_against_flagged_oracle(sparse, env, monkeypatch):
    """Full lossless mailboxes and a 1 us heartbeat each.  (a) An advance across one firing with nothing flushed, then a jump:
    the jump's flush to the old clock owes that tick and stalls with the clock unchanged.  (b) A jump whose last firing ends
    a window of the split: the split stalls with the clock moved.  Each stalled call is retried with the same clock after a
    drain; the oracle, which stalls on other calls, is driven the same way, and the two must then agree."""
    if env:
        monkeypatch.setenv(*env)
    N, R, P = 16, 64, 1000
    orc = DropOracle(N, timers_per_sub=1, keep_window=R, mailbox_cap=R)
    with Bus(N, ring_cap=R, batch_cap=32, timers_per_sub=1, lossless=True, sparse_ticks=sparse, drop_missed_ticks=True,
             device=0) as bus:
        for x in (bus, orc):
            for i in range(N):
                x.subscribe(nat.MASK_ALL)
                x.timer_add(i, P, 10 + i, False)

        def both(call):
            """call(x) on the oracle and the bus, each retried after a full drain of its own mailboxes until it completes;
            returns (bus clock after the bus's first attempt, whether the bus stalled)"""
            while call(orc) == tr.ob.EAGAIN:
                for i in range(N):
                    orc.consume(i, R)
            c0 = bus.stats()["now_ns"]
            rc = call(bus)
            c1 = bus.stats()["now_ns"]
            stalled = rc == nat.EAGAIN
            while rc == nat.EAGAIN:
                bus.consume_all()
                rc = call(bus)
            assert rc == nat.OK
            return c0, c1, stalled

        def fill():   # drain both, then exactly R records into every mailbox
            bus.consume_all()
            for i in range(N):
                orc.consume(i, R)
            for _ in range(R):
                both(lambda x: x.publish(5, 1))
                assert bus.flush() == nat.OK

        def check():
            assert bus.flush() == nat.OK
            bus.sync()
            tr.compare(bus, orc, N, window=R)

        t = 100
        both(lambda x: x.advance(t)); check()
        fill()
        both(lambda x: x.advance(t + 950))                 # across the firing at 1,000: the bus owes it, nothing is flushed
        c0, c1, stalled = both(lambda x: x.advance(t + 950 + 50 * P))
        assert stalled and c1 == c0 == t + 950, (c0, c1)  # (a) the flush to the old clock stalled
        check()
        T = (bus.stats()["now_ns"] // P + 1) * P           # a point of every grid
        both(lambda x: x.advance(T)); check()
        fill()
        c0, c1, stalled = both(lambda x: x.advance(T + 3 * 32 * P + P // 2))
        assert stalled and c0 == T and c1 == T + 3 * 32 * P, (c0, c1)   # (b) the split's third window ends on the firing
        check()
        w = bus.peek_window(0)
        assert (int(w["seq"][-1]), int(w["ts_ns"][-1])) == ((T + 96 * P) // P - 1, T + 96 * P)


def test_refusals():
    with Bus(64, ring_cap=64, batch_cap=32, timers_per_sub=1, drop_missed_ticks=True, device=0) as flagged, \
            Bus(64, ring_cap=64, batch_cap=32, timers_per_sub=1, device=0) as plain:
        with pytest.raises(nat.CpbusError) as e:
            flagged.stream_create(8, 2)
        assert e.value.status == nat.EINVAL
        st, handle = plain.stream_create(8, 2)
        try:
            for call in (lambda: flagged.stream_attach(st, 1), lambda: flagged.stream_open(handle, 1)):
                with pytest.raises(nat.CpbusError) as e:
                    call()
                assert e.value.status == nat.EINVAL
        finally:
            plain.stream_close(st)
        assert flagged.publish_device(0, 0, 10) == nat.EINVAL
        assert flagged.publish_device_staged(0, 0, 10) == nat.EINVAL
    # the group's own streams are not refused
    with GroupBus(64, [0, 0], ring_cap=64, batch_cap=32, timers_per_sub=1, drop_missed_ticks=True) as g:
        g.subscribe(nat.MASK_ALL)
        assert g.advance(5) == nat.OK and g.flush() == nat.OK


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("sparse", [False, True])
def test_thousand_second_heartbeat_step(sparse, lossless):
    """1,000 subscribers with one 1 s heartbeat each; the clock jumps 1,000 s: one tick per timer, seq 999, due at 1,000 s,
    where an unflagged twin delivers 1,000.  In lossless mode (64-record mailboxes) the flagged bus needs no drain."""
    N = 1000
    kw = dict(ring_cap=64 if lossless else 1024, batch_cap=32, timers_per_sub=1, lossless=lossless, sparse_ticks=sparse,
              device=0)
    with Bus(N, drop_missed_ticks=True, **kw) as bus, Bus(N, **kw) as plain:
        for b in (bus, plain):
            b.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
            b.timer_add_many(0, N, SEC, source_id0=100)
        assert bus.advance(1000 * SEC) == nat.OK and bus.flush() == nat.OK
        bus.sync()
        d = bus.digests(0, N)
        assert (d["count"] == 1).all()
        for s in (0, 517, N - 1):
            w = bus.peek_window(s)
            assert len(w) == 1 and int(w["seq"][0]) == 999 and int(w["ts_ns"][0]) == 1000 * SEC
            assert int(w["code"][0]) == 8 and int(w["source_id"][0]) == 100 + s and int(w["target"][0]) == s
        assert bus.stats()["ticks"] == N
        assert bus.advance(1001 * SEC) == nat.OK and bus.flush() == nat.OK   # the phase is kept: next due at 1,001 s
        bus.sync()
        assert int(bus.peek_window(5)["seq"][-1]) == 1000 and int(bus.peek_window(5)["ts_ns"][-1]) == 1001 * SEC
        if lossless:
            assert plain.advance(1000 * SEC) == nat.EAGAIN   # 1,000 ticks per 64-record mailbox
        else:
            assert plain.advance(1000 * SEC) == nat.OK and plain.flush() == nat.OK
            plain.sync()
            assert (plain.digests(0, N)["count"] == 1000).all()


@pytest.mark.parametrize("sparse", [False, True])
def test_steady_state_launches_no_catch_up(sparse):
    """1 ms steps under 1 s periods (and a step of exactly one period): the same launches as an unflagged twin, and the
    same results"""
    N = 4096
    kw = dict(ring_cap=1024, batch_cap=256, timers_per_sub=2, lossless=True, sparse_ticks=sparse, device=0)
    with Bus(N, drop_missed_ticks=True, **kw) as bus, Bus(N, **kw) as plain:
        rng = np.random.default_rng(5)
        for b in (bus, plain):
            b.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
            b.timer_add_many(0, N, SEC, source_id0=0)
            b.timer_add(7, 3 * SEC, 1, False)
        now = 0
        for step in range(3000):
            now += 1_000_000 if step != 1500 else SEC
            code = int(rng.integers(1, 17)) if step % 50 == 0 else None
            for b in (bus, plain):
                assert b.advance(now) == nat.OK
                if code is not None:
                    assert b.publish(code, 3) == nat.OK
                assert b.flush() == nat.OK
                if step % 200 == 199:
                    b.consume_all()
        assert bus.stats()["kernel_launches"] == plain.stats()["kernel_launches"]
        for x, y in zip(_final(bus, N), _final(plain, N)):
            _eq(x, y, "final")
