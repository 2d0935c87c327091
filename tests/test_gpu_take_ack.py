"""Acknowledged drains (cpbus_take_ready, cpbus_ack_many; Bus.take_ready / .ack_many and GroupBus's) on the GPU.
Random lossless traces with small rings, so that publishes stall, interleave broadcasts, unicast sends, exact cases,
periodic and one-shot timers (K = 1 and 4), clock steps, subscribes, unsubscribes, re-masks and pump steps.  Checked
against twins: take + ack of everything taken is cpbus_drain_ready; a take that is never acked is invisible; ack(id, k) is
cpbus_drain(id, cap = k).  Also the statuses, the group of 1-3 shards against one bus, a lossless stream shard's admission,
and the C++ mirror's acknowledging pump (csrc/host/events_ack_test.cc)."""
import os
import subprocess

import numpy as np
import pytest

from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from containerpilot_b200.group import GroupBus
from containerpilot_b200.sharding import LocalShardedBus

pytestmark = pytest.mark.gpu
R, BATCH, MAX_SUBS = 64, 32, 48
NOT_SHARED = ("kernel_launches",)
GROUP_SHAPED = ("batches", "kernel_launches", "admit_passes", "admit_skipped", "admit_partial", "device_splits")


def _bus(K, devices=None, lossless=True, n=MAX_SUBS):
    kw = dict(ring_cap=R, batch_cap=BATCH, timers_per_sub=K, lossless=lossless)
    return Bus(n, device=0, **kw) if devices is None else GroupBus(n, devices, **kw)


def _status(fn, *args):
    """the status of a Bus method, whether it returns one or raises"""
    try:
        r = fn(*args)
    except nat.CpbusError as e:
        return e.status
    return int(r) if isinstance(r, (int, np.integer)) else nat.OK


def _trace(seed, n_ops=500, n0=12):
    """Bus-level operations; ("pump",) marks where the consumer side runs.  Ids and timer handles are drawn by index
    into what has been handed out so far, so the same trace runs on every twin."""
    rng = np.random.default_rng(seed)
    ops, n_subs, n_timers, now = [], 0, 0, 0
    for _ in range(n0):
        ops.append(("sub", nat.MASK_ALL if rng.random() < 0.6 else int(rng.integers(1, 1 << 17)), None)); n_subs += 1
    for _ in range(n_ops):
        r = rng.random()
        if r < 0.03 and n_subs < MAX_SUBS:
            pairs = [(int(rng.integers(0, 17)), int(rng.integers(0, 8)))] if rng.random() < 0.5 else None
            ops.append(("sub", int(rng.integers(0, 1 << 17)), pairs)); n_subs += 1
        elif r < 0.05:
            ops.append(("unsub", int(rng.integers(0, n_subs))))
        elif r < 0.07:
            ops.append(("mask", int(rng.integers(0, n_subs)), int(rng.integers(0, 1 << 17))))
        elif r < 0.12:
            ops.append(("tadd", int(rng.integers(0, n_subs)), int(rng.integers(700, 9000)), int(rng.integers(0, 8)),
                        bool(rng.random() < 0.3)))
            n_timers += 1
        elif r < 0.14 and n_timers:
            ops.append(("tcancel", int(rng.integers(0, n_timers))))
        elif r < 0.45:   # mostly small publishes, and bursts that overrun a mailbox between pump steps
            k = int(rng.integers(1, 6)) if rng.random() < 0.9 else int(rng.integers(R // 2, 2 * R))
            ops.append(("pub", rng.integers(0, 17, k).tolist(), rng.integers(0, 8, k).tolist()))
        elif r < 0.55:
            ops.append(("send", int(rng.integers(0, n_subs)), int(rng.integers(0, 17)), int(rng.integers(0, 8))))
        elif r < 0.65:
            now += int(rng.integers(1, 4000)) if rng.random() < 0.9 else int(rng.integers(20_000, 60_000))
            ops.append(("advance", now))
        elif r < 0.72:
            ops.append(("flush",))
        else:
            ops.append(("pump", int(rng.integers(0, 1 << 30))))
    return ops


class _Run:
    """Applies a trace's bus-level operations to one bus and records every return code."""

    def __init__(self, bus):
        self.bus, self.ids, self.tids, self.codes = bus, [], [], []

    def id(self, i):
        """the i-th id the trace handed out (a subscribe that stalled hands out none)"""
        return self.ids[i % len(self.ids)]

    def step(self, op):
        b, kind = self.bus, op[0]
        if kind == "sub":
            rc = _status(lambda: self.ids.append(b.subscribe_pairs(op[1], op[2]) if op[2] else b.subscribe(op[1])))
        elif kind == "unsub":
            rc = _status(b.unsubscribe, self.id(op[1]))
        elif kind == "mask":
            rc = _status(b.set_mask, self.id(op[1]), op[2])
        elif kind == "tadd":
            tid = [0xFFFFFFFF]

            def add():
                tid[0] = b.timer_add(self.id(op[1]), op[2], op[3], op[4])
            rc = _status(add)
            self.tids.append(tid[0])
        elif kind == "tcancel":
            rc = _status(b.timer_cancel, self.tids[op[1]])
        elif kind == "pub":
            ev = np.zeros(len(op[1]), dtype=EVENT_DTYPE)
            ev["code"], ev["source_id"] = op[1], op[2]
            rc = b.publish_many(ev)
        elif kind == "send":
            rc = b.send(self.id(op[1]), op[2], op[3])
        elif kind == "advance":
            rc = b.advance(op[1])
        elif kind == "flush":
            rc = b.flush()
        else:
            return
        self.codes.append((op, rc))


def _state(bus, n_ids, exclude=NOT_SHARED):
    """Everything a consumer or operator can read without consuming, over ids [0, n_ids): digests, windows, backlog,
    blockers, debug events and the stats but `exclude`."""
    out = {"stats": {k: v for k, v in bus.stats().items() if k not in exclude}, "debug": bus.debug_events().tobytes(),
           "fold": bus.digest_fold(0, n_ids), "digests": bus.digests(0, n_ids).tobytes(), "blockers": bus.blockers().tolist()}
    lag, nxt, summary = bus.lagging(0, n_ids, min_backlog=0)
    out["lagging"] = (lag.tobytes(), nxt, summary)
    out["windows"] = [bus.peek_window(i).tobytes() for i in range(n_ids)]
    return out


def _cut(rng, n_ids):
    cap = int(rng.choice([R, R + 7, 2 * R, 3 * R + 5, 64 * R]))
    ready_cap = int(rng.choice([1, 2, 3, 5, 64]))
    start = int(rng.integers(0, n_ids))
    return cap, ready_cap, start


def _ready_equal(a, b, where):
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() and a[2] == b[2], where


# ---- 1. take + ack of everything taken == drain_ready ----------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_take_then_ack_all_is_drain_ready(K, seed):
    rng = np.random.default_rng(seed + 100)
    a, b = _bus(K), _bus(K)
    try:
        ra, rb = _Run(a), _Run(b)
        pumps = 0
        for op in _trace(seed):
            ra.step(op); rb.step(op)
            if op[0] != "pump" or not ra.ids:
                continue
            n_ids = len(ra.ids)
            cap, ready_cap, start = _cut(rng, n_ids)
            da = a.drain_ready(0, n_ids, start, cap, ready_cap)
            tb = b.take_ready(0, n_ids, start, cap, ready_cap)
            _ready_equal(da, tb, op)
            assert (tb[1]["lost"] == 0).all() and (tb[1]["pad"] == 0).all()
            st = b.ack_many(tb[1]["sub_id"], tb[1]["count"])
            assert (st == nat.OK).all()
            pumps += 1
        assert ra.codes == rb.codes
        assert any(rc == nat.EAGAIN for _, rc in ra.codes), "the trace never stalled"
        assert pumps > 50
        n_ids = len(ra.ids)
        assert _state(a, n_ids) == _state(b, n_ids)
        _ready_equal(a.drain_ready(0, n_ids, 0, 64 * R, 64), b.drain_ready(0, n_ids, 0, 64 * R, 64), "final")
    finally:
        a.close(); b.close()


# ---- 2. take without ack is invisible ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("seed", [4, 5])
def test_take_without_ack_is_invisible(K, seed):
    """A bus that takes and never acks against a twin that never drains: same return codes and EAGAIN points, blockers,
    lagging, windows, digests and stats but kernel_launches, checked after every pump step."""
    rng = np.random.default_rng(seed + 200)
    a, b = _bus(K), _bus(K)
    try:
        ra, rb = _Run(a), _Run(b)
        for op in _trace(seed, n_ops=300):
            ra.step(op); rb.step(op)
            if op[0] != "pump" or not ra.ids:
                continue
            n_ids = len(ra.ids)
            cap, ready_cap, start = _cut(rng, n_ids)
            b.take_ready(0, n_ids, start, cap, ready_cap)
            assert _state(a, n_ids) == _state(b, n_ids), op
        assert ra.codes == rb.codes
        assert any(rc == nat.EAGAIN for _, rc in ra.codes)
    finally:
        a.close(); b.close()


def test_consumer_that_stops_acking_stalls_the_publisher():
    with _bus(1) as bus:
        s0, s1 = bus.subscribe(), bus.subscribe()
        for i in range(R):
            assert bus.publish(3, i) == nat.OK
        assert bus.flush() == nat.OK
        rec, ready, _ = bus.take_ready(0, 2, 0, 4 * R, 8)
        assert ready["count"].tolist() == [R, R] and len(rec) == 2 * R
        assert bus.ack_many([s1], [R]).tolist() == [nat.OK]   # s1's channel took everything; s0's took nothing
        assert bus.publish(3, 99) == nat.OK
        assert bus.flush() == nat.EAGAIN                       # s0's mailbox is full of held records
        assert bus.blockers().tolist() == [s0]
        lag, _, _ = bus.lagging(0, 2)
        assert lag["sub_id"].tolist() == [s0] and lag["backlog"].tolist() == [R]
        assert len(bus.take_ready(0, 2, 0, 4 * R, 8)[1]) == 0  # nothing new for s0, s1 still empty
        assert bus.ack_many([s0], [1]).tolist() == [nat.OK]
        assert bus.flush() == nat.OK and len(bus.blockers()) == 0
        rec, ready, _ = bus.take_ready(0, 2, 0, 4 * R, 8)
        assert ready["sub_id"].tolist() == [s0, s1] and ready["count"].tolist() == [1, 1]
        assert rec["source_id"].tolist() == [99, 99]


# ---- 3. ack(id, k) == drain(id, cap = k) ------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("seed", [6, 7, 8])
def test_partial_ack_is_drain_of_k(K, seed):
    """The taking bus acks arbitrary parts of what it holds; the twin drains exactly that many from the same mailboxes.
    The states agree after every pump step, and per mailbox the records taken over the whole run are the records the twin
    drained, each once."""
    rng = np.random.default_rng(seed + 300)
    a, b = _bus(K), _bus(K)
    got_a, got_b = {}, {}
    try:
        ra, rb = _Run(a), _Run(b)
        held = {}
        for op in _trace(seed):
            ra.step(op); rb.step(op)
            if op[0] != "pump" or not ra.ids:
                continue
            n_ids = len(ra.ids)
            cap, ready_cap, start = _cut(rng, n_ids)
            rec, ready, _ = b.take_ready(0, n_ids, start, cap, ready_cap)
            for e in ready:
                sid = int(e["sub_id"])
                got_b.setdefault(sid, []).append(rec[int(e["offset"]):int(e["offset"]) + int(e["count"])].tobytes())
                held[sid] = held.get(sid, 0) + int(e["count"])
            ids, cnts = [], []
            for sid in sorted(held):
                if held[sid] and rng.random() < 0.7:
                    k = int(rng.integers(0, held[sid] + 1))
                    if k and rng.random() < 0.3:      # the same mailbox twice, in two parts
                        ids += [sid, sid]; cnts += [k // 2, k - k // 2]
                    else:
                        ids.append(sid); cnts.append(k)
            perm = rng.permutation(len(ids))
            ids, cnts = [ids[i] for i in perm], [cnts[i] for i in perm]
            assert (b.ack_many(ids, cnts) == nat.OK).all()
            for sid, k in zip(ids, cnts):
                held[sid] -= k
                if k:
                    got_a.setdefault(sid, []).append(a.drain(sid, cap=k).tobytes())
            assert _state(a, n_ids) == _state(b, n_ids), op
        assert ra.codes == rb.codes
        n_ids = len(ra.ids)
        rest_a = a.drain_ready(0, n_ids, 0, 64 * R, 64)
        rest_b = b.take_ready(0, n_ids, 0, 64 * R, 64)
        for rest, got in ((rest_a, got_a), (rest_b, got_b)):
            for e in rest[1]:
                got.setdefault(int(e["sub_id"]), []).append(rest[0][int(e["offset"]):int(e["offset"]) + int(e["count"])].tobytes())
        for sid in range(n_ids):   # the twin drains each record once: equal runs mean none was taken twice or skipped
            assert b"".join(got_a.get(sid, [])) == b"".join(got_b.get(sid, [])), sid
    finally:
        a.close(); b.close()


# ---- 4. statuses ------------------------------------------------------------------------------------------------------------
def test_ack_statuses():
    with _bus(1) as bus:
        s = [bus.subscribe() for _ in range(3)]
        for i in range(5):
            bus.publish(2, i)
        assert bus.flush() == nat.OK
        assert bus.ack_many([s[0]], [1]).tolist() == [nat.EINVAL]      # nothing taken yet: nothing held
        bus.take_ready(0, 3, 0, 4 * R, 8)
        st = bus.ack_many([s[0], 3, 1000, s[1], s[1], s[1], s[2], s[2], s[0]], [2, 1, 0, 3, 3, 0, 6, 5, 3])
        assert st.tolist() == [nat.OK, nat.ENOENT, nat.ENOENT, nat.OK, nat.EINVAL, nat.OK, nat.EINVAL, nat.OK, nat.OK]
        ids, cnts = np.array([s[0], s[1], 7], dtype=np.uint32), np.array([1, 2, 0], dtype=np.uint32)
        status, applied = np.full(3, 99, dtype=np.int32), np.zeros(1, dtype=np.uint32)
        lib = nat.load()
        assert lib.cpbus_ack_many(bus._h, ids.ctypes.data, cnts.ctypes.data, 3, status.ctypes.data,
                                  applied.ctypes.data_as(nat.C.POINTER(nat.C.c_uint32))) == nat.OK
        assert status.tolist() == [nat.EINVAL, nat.OK, nat.ENOENT] and applied[0] == 1
        assert bus.ack_many([], []).size == 0
        # a plain drain after a take reads from head, held records included, and leaves nothing held
        for i in range(3):
            bus.publish(4, 10 + i)
        assert bus.flush() == nat.OK
        bus.take_ready(0, 3, 0, 4 * R, 8)
        assert bus.drain(s[0]).tolist() == bus.peek_window(s[0])[-3:].tolist()
        assert bus.ack_many([s[0]], [1]).tolist() == [nat.EINVAL]
        bus.consume_all()
        assert bus.ack_many([s[1], s[2]], [1, 1]).tolist() == [nat.EINVAL, nat.EINVAL]
        # unsubscribed mailboxes can be acked: the pump may have taken their records before the unsubscribe
        bus.publish(5, 1)
        assert bus.flush() == nat.OK
        rec, ready, _ = bus.take_ready(0, 3, 0, 4 * R, 8)
        assert len(ready) == 3
        bus.unsubscribe(s[2])
        assert bus.ack_many([s[2], s[2]], [1, 1]).tolist() == [nat.OK, nat.EINVAL]


@pytest.mark.parametrize("group", [False, True])
def test_throughput_bus_refuses_both(group):
    with _bus(1, devices=[0, 0] if group else None, lossless=False, n=4) as bus:
        bus.subscribe_many([nat.MASK_ALL] * 4)
        with pytest.raises(nat.CpbusError) as e:
            bus.take_ready(0, 4, 0, R, 4)
        assert e.value.status == nat.EINVAL
        with pytest.raises(nat.CpbusError) as e:
            bus.ack_many([0], [0])
        assert e.value.status == nat.EINVAL
        assert bus.ack_many([], []).size == 0


def test_one_launch_per_ack():
    with _bus(1) as bus:
        s = [bus.subscribe() for _ in range(4)]
        for i in range(6):
            bus.publish(1, i)
        assert bus.flush() == nat.OK
        k0 = bus.stats()["kernel_launches"]
        bus.ack_many(s, [1, 1, 1, 1])                      # before the first take: refused without a launch
        assert bus.stats()["kernel_launches"] == k0
        bus.take_ready(0, 4, 0, 4 * R, 8)
        k1 = bus.stats()["kernel_launches"]
        assert k1 == k0 + 2                                 # the take scan and the gather
        bus.ack_many([s[0], 99, s[1]], [0, 1, 0])           # nothing for the device
        assert bus.stats()["kernel_launches"] == k1
        assert (bus.ack_many(s + s, [1] * 4 + [2] * 4) == nat.OK).all()
        assert bus.stats()["kernel_launches"] == k1 + 1


# ---- 5. the group against one bus -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("G", [1, 2, 3])
@pytest.mark.parametrize("K", [1, 4])
def test_group_equals_one_bus(G, K):
    """Call for call: the same trace, the same take cuts, partial acks with duplicates and unknown ids, plain drains and
    consume_all on a group of G shards (all on GPU 0) and on one bus."""
    rng_a, rng_b = np.random.default_rng(G * 10 + K), np.random.default_rng(G * 10 + K)
    a, b = _bus(K), _bus(K, devices=[0] * G)
    try:
        ra, rb = _Run(a), _Run(b)
        for op in _trace(900 + G * 10 + K, n_ops=400):
            ra.step(op); rb.step(op)
            if op[0] != "pump" or not ra.ids:
                continue
            n_ids = len(ra.ids)
            results = []
            for bus, rng in ((a, rng_a), (b, rng_b)):
                cap, ready_cap, start = _cut(rng, n_ids)
                r = [bus.take_ready(0, n_ids, start, cap, ready_cap)]
                ids = rng.integers(0, n_ids + 3, 6)
                r.append(bus.ack_many(ids, rng.integers(0, 6, 6)))
                if rng.random() < 0.1:
                    r.append(bus.drain(int(rng.integers(0, n_ids)), cap=int(rng.integers(1, R))))
                if rng.random() < 0.03:
                    bus.consume_all()
                results.append(r)
            _ready_equal(results[0][0], results[1][0], op)
            assert results[0][1].tolist() == results[1][1].tolist(), op
            if len(results[0]) > 2:
                assert results[0][2].tobytes() == results[1][2].tobytes()
        assert ra.codes == rb.codes
        n_ids = len(ra.ids)
        assert _state(a, n_ids, GROUP_SHAPED) == _state(b, n_ids, GROUP_SHAPED)
    finally:
        a.close(); b.close()


# ---- 6. a lossless stream shard ---------------------------------------------------------------------------------------------
def test_held_records_lower_stream_admission():
    """One lossless stream shard: held records lower cpbus_stream_admit's prefix exactly as records never drained do."""
    N = 4
    kw = dict(ring_cap=R, batch_cap=BATCH, stream_slots=8, lossless=True)
    a, b = LocalShardedBus(N, [0], **kw), LocalShardedBus(N, [0], **kw)
    try:
        for sb in (a, b):
            sb.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))

        def batch(n, ts):
            ev = np.zeros(n, dtype=EVENT_DTYPE)
            ev["seq"] = np.arange(n); ev["ts_ns"] = ts; ev["code"] = 1; ev["target"] = nat.TARGET_ALL
            return ev

        def admit(sb, n, w):
            bus, st = sb.shards[0][2], sb._st[0]
            try:
                return bus.stream_admit(st, n, w)
            except nat.CpbusError as e:
                return e.status

        w = 100
        for sb in (a, b):                                    # R - 3 records in every mailbox
            for n in (BATCH, R - 3 - BATCH):
                nat.check(sb.put(batch(n, w), w, raw=True), "put")
                assert sb.fanout(n, w) == nat.OK
        bb = b.shards[0][2]
        assert len(bb.take_ready(0, N, 0, 4 * R, N)[1]) == N  # everything held, nothing acked
        w = 200
        for sb in (a, b):
            nat.check(sb.put(batch(BATCH, w), w, raw=True), "put")
        assert admit(a, BATCH, w) == admit(b, BATCH, w) == 3
        assert len(a.drain(0, cap=5)) == 5
        assert bb.ack_many([0], [5]).tolist() == [nat.OK]
        assert admit(a, BATCH, w) == admit(b, BATCH, w) == 3
        for s in range(1, N):
            assert len(a.drain(s, cap=R)) == R - 3
        assert (bb.ack_many([1, 2, 3], [R - 3] * 3) == nat.OK).all()
        assert admit(a, BATCH, w) == admit(b, BATCH, w) == 5 + 3
        a.drain(0, cap=R)
        assert bb.ack_many([0], [R - 8]).tolist() == [nat.OK]
        assert admit(a, BATCH, w) == admit(b, BATCH, w) == BATCH
        assert a.fanout(BATCH, w) == b.fanout(BATCH, w) == nat.OK
        assert a.digests().tobytes() == b.digests().tobytes()
    finally:
        a.close(); b.close()


# ---- the C++ mirror ---------------------------------------------------------------------------------------------------------
def test_cpp_mirror_acknowledging_pump():
    """csrc/host/events_ack_test: EventBus::AckOnDelivery on one bus and on a group of three shards"""
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "containerpilot_b200", "csrc", "host",
                       "events_ack_test")
    assert os.path.exists(exe), "built by the host Makefile"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
