"""Drain tickets (cpbus_drain_ready_begin, cpbus_take_ready_begin, cpbus_drain_ready_end) on the GPU.
Seeded traces of publishes, sends, clock steps, timers (K = 1, 2, 4), subscribes, unsubscribes, re-masks, releases and,
in lossless mode, stalls run on twin buses: one drains with cpbus_drain_ready / cpbus_take_ready, the other with tickets
that are ended right away, one step later, or up to 8 at a time in any order.  Every return code and every drain result
is compared byte for byte, and at the end the drains, windows, digests, folds, lagging, blockers, debug events and every
stats field but kernel_launches.  Also the refusals, destroy with tickets outstanding, the C oracle's mailboxes and the
dense bridge shape (8,192 mailboxes x 512 records)."""
import numpy as np
import pytest

import oracle_binding as ob
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE

pytestmark = pytest.mark.gpu
R, BATCH, MAX_SUBS = 64, 32, 48


def _bus(K, lossless, base=0, **kw):
    return Bus(MAX_SUBS, ring_cap=R, batch_cap=BATCH, timers_per_sub=K, lossless=lossless, sub_id_base=base, device=0, **kw)


def _status(fn, *args):
    try:
        r = fn(*args)
    except nat.CpbusError as e:
        return e.status
    return r.tobytes() if isinstance(r, np.ndarray) else (int(r) if isinstance(r, (int, np.integer)) else nat.OK)


def _trace(seed, n_ops=400, n0=12):
    """Bus-level operations with ("pump", r) where the consumer side runs; ids and timers are drawn by index into what
    has been handed out, so the same trace runs on both twins."""
    rng = np.random.default_rng(seed)
    ops, n_timers, now = [], 0, 0
    for _ in range(n0):
        ops.append(("sub", nat.MASK_ALL if rng.random() < 0.6 else int(rng.integers(1, 1 << 17)), None))
    for _ in range(n_ops):
        r = rng.random()
        if r < 0.03:
            pairs = [(int(rng.integers(0, 17)), int(rng.integers(0, 8)))] if rng.random() < 0.5 else None
            ops.append(("sub", int(rng.integers(0, 1 << 17)), pairs))
        elif r < 0.05:
            ops.append(("unsub", int(rng.integers(0, 1 << 20))))
        elif r < 0.06:
            ops.append(("release", int(rng.integers(0, 1 << 20))))
        elif r < 0.07:
            ops.append(("sublist", rng.integers(0, 1 << 17, int(rng.integers(1, 3))).tolist()))
        elif r < 0.09:
            ops.append(("mask", int(rng.integers(0, 1 << 20)), int(rng.integers(0, 1 << 17))))
        elif r < 0.14:
            ops.append(("tadd", int(rng.integers(0, 1 << 20)), int(rng.integers(700, 9000)), int(rng.integers(0, 8)),
                        bool(rng.random() < 0.3)))
            n_timers += 1
        elif r < 0.16 and n_timers:
            ops.append(("tcancel", int(rng.integers(0, n_timers))))
        elif r < 0.45:
            k = int(rng.integers(1, 6)) if rng.random() < 0.9 else int(rng.integers(R // 2, 2 * R))
            ops.append(("pub", rng.integers(0, 17, k).tolist(), rng.integers(0, 8, k).tolist()))
        elif r < 0.55:
            ops.append(("send", int(rng.integers(0, 1 << 20)), int(rng.integers(0, 17)), int(rng.integers(0, 8))))
        elif r < 0.65:
            now += int(rng.integers(1, 4000)) if rng.random() < 0.9 else int(rng.integers(20_000, 60_000))
            ops.append(("advance", now))
        elif r < 0.72:
            ops.append(("flush",))
        else:
            ops.append(("pump", int(rng.integers(0, 1 << 30))))
    return ops


class _Run:
    """Applies a trace's bus-level operations to one bus; step() returns the operation's result."""

    def __init__(self, bus):
        self.bus, self.ids, self.tids = bus, [], []

    def id(self, i):
        return self.ids[i % len(self.ids)]

    def step(self, op):
        b, kind = self.bus, op[0]
        if not self.ids and kind in ("unsub", "release", "mask", "tadd", "send"):
            return None
        if kind == "sub":
            return _status(lambda: self.ids.append(b.subscribe_pairs(op[1], op[2]) if op[2] else b.subscribe(op[1])))
        if kind == "sublist":
            return _status(lambda: self.ids.extend(int(x) for x in b.subscribe_list(op[1])))
        if kind == "unsub":
            return _status(b.unsubscribe, self.id(op[1]))
        if kind == "release":   # released ids are not used again until subscribe_list hands them out
            sid = self.id(op[1])
            rc = (_status(b.unsubscribe, sid), _status(b.release_many, [sid]))
            self.ids.remove(sid)
            return rc
        if kind == "mask":
            return _status(b.set_mask, self.id(op[1]), op[2])
        if kind == "tadd":
            tid = [0xFFFFFFFF]

            def add():
                tid[0] = b.timer_add(self.id(op[1]), op[2], op[3], op[4])
            rc = _status(add)
            self.tids.append(tid[0])
            return rc
        if kind == "tcancel":
            return _status(b.timer_cancel, self.tids[op[1]])
        if kind == "pub":
            ev = np.zeros(len(op[1]), dtype=EVENT_DTYPE)
            ev["code"], ev["source_id"] = op[1], op[2]
            return b.publish_many(ev)
        if kind == "send":
            return b.send(self.id(op[1]), op[2], op[3])
        if kind == "advance":
            return b.advance(op[1])
        if kind == "flush":
            return b.flush()
        return None


def _state(bus, base, n_ids):
    """Everything a consumer or operator can read without consuming over ids [base, base + n_ids)."""
    out = {"stats": {k: v for k, v in bus.stats().items() if k != "kernel_launches"}, "debug": bus.debug_events().tobytes(),
           "fold": bus.digest_fold(base, n_ids), "digests": bus.digests(base, n_ids).tobytes(), "blockers": bus.blockers().tolist()}
    lag, nxt, summary = bus.lagging(base, n_ids, min_backlog=0)
    out["lagging"] = (lag.tobytes(), nxt, summary)
    out["windows"] = [_status(bus.peek_window, base + i) for i in range(n_ids)]   # released ids: CPBUS_ENOENT
    return out


def _same(a, b, where):
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() and a[2] == b[2], where


def _twins(seed, K, lossless, depth, base=0, take=False, ack_early=False, shuffle=False, chain=True, n_ops=400, **kw):
    """Runs one trace on a synchronous twin `a` and a ticketed twin `b`.  At each pump step `a` drains (or takes and
    acks) at once, and `b` begins a ticket with the same arguments; `b` ends its tickets when `depth` are outstanding
    (shuffle: in random order, several at a time), and each result must equal `a`'s at the begin's place.  chain: the
    next start_sub is the next_sub of the last ticket ended, as a pipelined pump passes it on."""
    rng = np.random.default_rng(seed + 1000)
    a, b = _bus(K, lossless, base, **kw), _bus(K, lossless, base, **kw)
    pending, ended, start = [], 0, base
    try:
        ra, rb = _Run(a), _Run(b)

        def end(k):
            nonlocal ended, start
            t, want, cap, ready_cap, where = pending.pop(k)
            got = b.drain_ready_end(t, cap, ready_cap)
            _same(want, got, where)
            ended += 1
            if chain:
                start = got[2]

        for i, op in enumerate(_trace(seed, n_ops)):
            assert ra.step(op) == rb.step(op), (i, op)
            if op[0] != "pump" or not ra.ids:
                continue
            n_ids = max(ra.ids) + 1 - base
            if not chain or not base <= start < base + n_ids:
                start = base + int(rng.integers(0, n_ids))
            cap = int(rng.choice([R, R + 7, 2 * R, 3 * R + 5, 64 * R]))
            ready_cap = int(rng.choice([1, 2, 3, 5, 64]))
            if take:
                want = a.take_ready(base, n_ids, start, cap, ready_cap)
                assert (a.ack_many(want[1]["sub_id"], want[1]["count"]) == nat.OK).all()
                t = b.take_ready_begin(base, n_ids, start, cap, ready_cap)
                if ack_early:   # acked before the take's _end: stream-ordered behind the take's scan
                    assert (b.ack_many(want[1]["sub_id"], want[1]["count"]) == nat.OK).all()
                    pending.append((t, want, cap, ready_cap, (i, op)))
                else:
                    pending.append((t, want, cap, ready_cap, (i, op)))
                    while pending:
                        end(0)
                    assert (b.ack_many(want[1]["sub_id"], want[1]["count"]) == nat.OK).all()
            else:
                want = a.drain_ready(base, n_ids, start, cap, ready_cap)
                pending.append((b.drain_ready_begin(base, n_ids, start, cap, ready_cap), want, cap, ready_cap, (i, op)))
            if pending and len(pending) >= depth:
                if shuffle:
                    for _ in range(int(rng.integers(1, len(pending) + 1))):
                        end(int(rng.integers(0, len(pending))))
                else:
                    end(0)
        while pending:
            end(int(rng.integers(0, len(pending))) if shuffle else 0)
        n_ids = max(ra.ids) + 1 - base
        assert ended > 30
        assert _state(a, base, n_ids) == _state(b, base, n_ids)
        _same(a.drain_ready(base, n_ids, base, 64 * R, 64), b.drain_ready(base, n_ids, base, 64 * R, 64), "final")
    finally:
        a.close(); b.close()


# ---- equivalence with the synchronous calls ----------------------------------------------------------------------------
@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4])
def test_end_right_after_begin(K, lossless):
    _twins(10 + K, K, lossless, depth=1)


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("seed", [21, 22])
def test_end_after_further_publishes_and_flushes(seed, lossless):
    """each ticket is ended at the next pump step, after the operations in between"""
    _twins(seed, 2, lossless, depth=2)


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("seed", [31, 32])
def test_eight_outstanding_ended_out_of_order(seed, lossless):
    _twins(seed, 4, lossless, depth=8, shuffle=True, chain=True)


def test_eight_outstanding_unchained():
    _twins(33, 1, False, depth=8, shuffle=True, chain=False)


@pytest.mark.parametrize("ack_early", [False, True])
@pytest.mark.parametrize("seed", [41, 42])
def test_take_ready_begin_then_ack(seed, ack_early):
    _twins(seed, 2, True, depth=3 if ack_early else 1, take=True, ack_early=ack_early, shuffle=ack_early)


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("records", [False, True])
def test_sparse_buses(records, lossless):
    """CPBUS_CFG_SPARSE_TICKS, and with CPBUS_CFG_SPARSE_RECORDS"""
    _twins(50 + records, 2, lossless, depth=2, sparse_ticks=True, sparse_records=records)


@pytest.mark.parametrize("lossless", [False, True])
def test_sub_id_base(lossless):
    _twins(61, 1, lossless, depth=3, base=100_000, shuffle=True)


def test_ticket_that_finds_nothing_ready():
    with _bus(1, False, base=7) as bus:
        for _ in range(5):
            bus.subscribe()
        t = bus.drain_ready_begin(7, 5, 9, R, 4)
        rec, ready, nxt = bus.drain_ready_end(t, R, 4)
        assert len(rec) == 0 and len(ready) == 0 and nxt == 9
        bus.publish(3, 1); bus.flush()
        t0 = bus.drain_ready_begin(7, 5, 7, 4 * R, 8)
        t1 = bus.drain_ready_begin(7, 5, 7, 4 * R, 8)   # behind t0, which took everything
        rec, ready, nxt = bus.drain_ready_end(t1, 4 * R, 8)
        assert len(rec) == 0 and len(ready) == 0 and nxt == 7
        rec, ready, nxt = bus.drain_ready_end(t0, 4 * R, 8)
        assert ready["sub_id"].tolist() == [7, 8, 9, 10, 11] and len(rec) == 5 and nxt == 7


# ---- refusals, destroy ------------------------------------------------------------------------------------------------
def _status_of(fn, *args):
    try:
        fn(*args)
    except nat.CpbusError as e:
        return e.status
    return nat.OK


def test_refusals():
    with _bus(1, True) as bus:
        ids = [bus.subscribe() for _ in range(4)]
        for i in range(10):
            bus.publish(2, i)
        assert bus.flush() == nat.OK
        tickets = [bus.drain_ready_begin(0, 4, 0, R, 1) for _ in range(8)]
        assert len(set(tickets)) == 8
        before = bus.stats()
        assert _status_of(bus.drain_ready_begin, 0, 4, 0, R, 1) == nat.ENOSPC
        assert _status_of(bus.take_ready_begin, 0, 4, 0, R, 1) == nat.ENOSPC
        after = bus.stats()
        assert after["kernel_launches"] == before["kernel_launches"], "a refused begin enqueued something"
        # the usual checks of the synchronous call
        assert _status_of(bus.drain_ready_begin, 0, 4, 0, R - 1, 1) == nat.EINVAL
        assert _status_of(bus.drain_ready_begin, 0, 4, 4, R, 1) == nat.EINVAL
        assert _status_of(bus.drain_ready_begin, 0, 5, 0, R, 1) == nat.ENOENT
        assert _status_of(bus.drain_ready_begin, 0, 4, 0, 1 << 32, 1) == nat.EINVAL
        # a short cap or ready_cap at _end: refused, and the ticket stays collectable
        assert _status_of(bus.drain_ready_end, tickets[3], R - 1, 1) == nat.EINVAL
        assert _status_of(bus.drain_ready_end, tickets[3], R, 0) == nat.EINVAL
        got = {}
        for j in (3, 0, 7, 1, 2, 6, 5, 4):
            rec, ready, nxt = bus.drain_ready_end(tickets[j], R, 1)
            got[j] = ready["sub_id"].tolist()
            assert _status_of(bus.drain_ready_end, tickets[j], R, 1) == nat.ENOENT   # ended twice
        assert [got[j] for j in range(8)] == [[ids[0]], [ids[1]], [ids[2]], [ids[3]], [], [], [], []]
        assert _status_of(bus.drain_ready_end, 12345, R, 1) == nat.ENOENT            # never begun
        t = bus.drain_ready_begin(0, 4, 0, R, 1)                                     # slots are free again
        assert t not in tickets
        bus.drain_ready_end(t, R, 1)
    with _bus(1, False) as bus:
        bus.subscribe()
        assert _status_of(bus.take_ready_begin, 0, 1, 0, R, 1) == nat.EINVAL         # throughput mode


def test_destroy_with_tickets_outstanding():
    for lossless in (False, True):
        bus = _bus(2, lossless)
        for _ in range(MAX_SUBS):
            bus.subscribe()
        for k in range(6):
            ev = np.zeros(BATCH, dtype=EVENT_DTYPE)
            ev["code"] = 3; ev["source_id"] = np.arange(BATCH) + k
            bus.publish_many(ev); bus.flush()
            bus.drain_ready_begin(0, MAX_SUBS, 0, 64 * R, 64)
        bus.close()
    with _bus(1, False) as bus:   # the device is still usable
        s = bus.subscribe()
        bus.publish(1, 1); bus.flush()
        t = bus.drain_ready_begin(s, 1, s, R, 1)
        assert bus.drain_ready_end(t, R, 1)[0]["source_id"].tolist() == [1]


# ---- the C oracle's mailboxes -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [1, 2])
def test_lossless_stalls_released_by_tickets_match_the_oracle(seed):
    """Lossless back pressure released by ticketed drains (ended one step later, or at once when the flush is stuck):
    every ticket's runs are the oracle's records of those mailboxes, consumed in order."""
    Rr, B, N = 128, 64, 6
    rng = np.random.default_rng(700 + seed)
    masks = [nat.MASK_ALL, 1 << 2, (1 << 3) | (1 << 2), nat.MASK_ALL, 1 << 5, 0]
    orc = ob.Oracle(N, keep_window=0, mailbox_cap=Rr)
    for m_ in masks:
        orc.subscribe(m_)
    pending, n_again, start = [], 0, 0

    def collect():
        nonlocal start
        t = pending.pop(0)
        rec, rdy, start = bus.drain_ready_end(t, Rr, 2)
        for e in rdy:
            got = rec[int(e["offset"]):int(e["offset"]) + int(e["count"])]
            assert got.tobytes() == orc.consume(int(e["sub_id"]), int(e["count"])).tobytes()
        return len(rdy)

    with Bus(N, ring_cap=Rr, batch_cap=B, lossless=True, device=0) as bus:
        bus.subscribe_many(np.array(masks, dtype=np.uint32))
        for step in range(40):
            ev = np.zeros(B, dtype=EVENT_DTYPE)
            ev["code"] = rng.integers(1, 7, B); ev["source_id"] = step * B + np.arange(B)
            nat.check(bus.publish_many(ev), "publish")
            i = 0
            while True:
                rc = bus.flush()
                while i < B:
                    r = orc.publish(int(ev["code"][i]), int(ev["source_id"][i]))
                    if r == ob.EAGAIN:
                        break
                    assert r == 0
                    i += 1
                if rc == nat.OK:
                    assert i == B
                    break
                assert rc == nat.EAGAIN and i < B
                n_again += 1
                while pending:
                    collect()
                pending.append(bus.drain_ready_begin(0, N, start, Rr, 2))
                assert collect() >= 1
            if rng.random() < 0.5:
                pending.append(bus.drain_ready_begin(0, N, start, Rr, 2))
            if len(pending) > 1:
                collect()
        while pending:
            collect()
        for s in range(N):
            rec, rdy, _ = bus.drain_ready(s, 1, s, Rr, 1)
            assert rec.tobytes() == orc.consume(s, Rr).tobytes()
        assert bus.stats()["overwritten"] == 0
    assert n_again > 5


# ---- the dense bridge shape ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lossless", [False, True])
def test_dense_bridge_shape(lossless):
    """8,192 mailboxes x 512 records: a ticket returns what the synchronous call returns on a twin, whole and in pieces"""
    N, RR, B = 8192, 512, 256
    kw = dict(ring_cap=RR, batch_cap=B, lossless=lossless, device=0)
    with Bus(N, **kw) as a, Bus(N, **kw) as b:
        for bus in (a, b):
            bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
            for k in range(RR // B):
                ev = np.zeros(B, dtype=EVENT_DTYPE)
                ev["code"] = 1 + np.arange(B) % 16; ev["source_id"] = k * B + np.arange(B)
                nat.check(bus.publish_many(ev), "publish")
                nat.check(bus.flush(), "flush")
        cap = N * RR
        want = a.drain_ready(0, N, 0, cap, N)
        got = b.drain_ready_end(b.drain_ready_begin(0, N, 0, cap, N), cap, N)
        assert len(got[0]) == N * RR and len(got[1]) == N
        _same(want, got, "whole")
        for bus in (a, b):
            ev = np.zeros(B, dtype=EVENT_DTYPE)
            ev["code"] = 5; ev["source_id"] = 77 + np.arange(B)
            nat.check(bus.publish_many(ev), "publish"); nat.check(bus.flush(), "flush")
        sa = sb = 4321
        tickets = []
        for _ in range(4):   # a quarter of the fleet's records per call, four tickets in flight
            want = a.drain_ready(0, N, sa, cap // 4 + 3, N)
            sa = want[2]
            tickets.append((b.drain_ready_begin(0, N, sb, cap // 4 + 3, N), want))
            sb = sa
        for t, want in tickets[::-1]:
            _same(want, b.drain_ready_end(t, cap // 4 + 3, N), "pieces")
        assert a.digest_fold(0, N) == b.digest_fold(0, N)


# ---- many short runs: each warp of the gather stores many chunks, most of which cross runs --------------------------------
SHORT_CODES = [1, 2, 2, 3, 3, 3, 4, 4, 4, 4, 4]   # runs of 1, 2, 3 or 5 records: code c reaches the mailboxes of mask bit c


def _short_run_fleet(N, lossless, seed):
    """N mailboxes, each subscribed to one code (most to code 1, a run of one record per round) or to none (empty)"""
    rng = np.random.default_rng(seed)
    code_of = rng.choice([0, 1, 1, 1, 1, 1, 2, 3, 4], N)
    masks = np.where(code_of == 0, 0, 1 << code_of).astype(np.uint32)
    buses = [Bus(N, ring_cap=R, batch_cap=BATCH, lossless=lossless, device=0) for _ in range(2)]
    for bus in buses:
        bus.subscribe_many(masks)
    return buses, code_of


def _publish_round(buses, k):
    ev = np.zeros(len(SHORT_CODES), dtype=EVENT_DTYPE)
    ev["code"] = SHORT_CODES; ev["source_id"] = 1000 * k + np.arange(len(SHORT_CODES))
    for bus in buses:
        nat.check(bus.publish_many(ev), "publish"); nat.check(bus.flush(), "flush")


def _runs_are_the_published_ones(res, code_of, k):
    rec, ready = res[0], res[1]
    codes = code_of[ready["sub_id"]]
    per_code = {c: SHORT_CODES.count(c) for c in (1, 2, 3, 4)}
    assert (ready["count"] == [per_code[int(c)] for c in codes]).all()
    assert (rec["code"] == np.repeat(codes, ready["count"])).all()
    assert (rec["source_id"] // 1000 == k).all()


@pytest.mark.parametrize("mode", ["drain", "lossless", "take"])
def test_many_short_runs_in_one_ticket(mode):
    """262,144 mailboxes with runs of 0 to 5 records, most of one: a ticket that moves ~440,000 records gives every warp of
    the gather several chunks, and most chunks start or end inside a run of one.  Byte-identical with the synchronous call
    on a twin, whole and in pieces with several tickets outstanding, and each run is the mailbox's published records."""
    N = 1 << 18
    buses, code_of = _short_run_fleet(N, mode != "drain", 0x5A07 + len(mode))
    a, b = buses
    sync = a.take_ready if mode == "take" else a.drain_ready
    begin = b.take_ready_begin if mode == "take" else b.drain_ready_begin
    try:
        _publish_round(buses, 1)
        cap = 1 << 20
        want = sync(0, N, 0, cap, N)
        got = b.drain_ready_end(begin(0, N, 0, cap, N), cap, N)
        assert len(got[0]) > 16 * 32 * 132 * 4
        _same(want, got, "whole")
        _runs_are_the_published_ones(got, code_of, 1)
        if mode == "take":
            for bus, res in ((a, want), (b, got)):
                assert (bus.ack_many(res[1]["sub_id"], res[1]["count"]) == nat.OK).all()
        _publish_round(buses, 2)
        sa = sb = 123_457
        tickets = []
        for cap, ready_cap in ((70_001, 50_000), (100_003, 1 << 18), (1 << 16, 30_000), (1 << 20, 1 << 18)):
            want = sync(0, N, sa, cap, ready_cap)
            tickets.append((begin(0, N, sb, cap, ready_cap), want, cap, ready_cap))
            sa = sb = want[2]
        for t, want, cap, ready_cap in tickets[::-1]:
            got = b.drain_ready_end(t, cap, ready_cap)
            _same(want, got, ("pieces", cap, ready_cap))
            _runs_are_the_published_ones(got, code_of, 2)
        assert a.digest_fold(0, N) == b.digest_fold(0, N)
        assert a.lagging(0, N, min_backlog=0)[2] == b.lagging(0, N, min_backlog=0)[2]
    finally:
        a.close(); b.close()
