"""Device batches on the group (`cpbus_group_publish_device`, `_staged`, `GroupBus.publish_device*`): a group of G shards
gives the results of one bus with the same configuration — return codes, drains, sparse drains, windows, digests, folds,
debug events, publish counts and the stats that are not launch-shaped — for traces that mix host publishes, sends, clock
steps, membership changes and timers with device batches, in throughput and lossless mode, and the oracle's mailboxes.

The device batches include batches past batch_cap and past the timer window (cut into slices), records older than the
clock, a watermark behind the clock, unicast records for every shard, codes outside the enum and empty batches."""
import numpy as np
import pytest

import oracle_binding as ob
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from containerpilot_b200.group import GroupBus

pytestmark = pytest.mark.gpu
LAUNCH_SHAPED = ("batches", "kernel_launches", "admit_passes", "admit_skipped", "admit_partial", "device_splits")
OUT = [17, 24, 28, 31, 32, 1000, 0xFFFFFFFF]   # broadcast codes outside the enum: they reach no mailbox


def _n_gpus():
    import torch
    return torch.cuda.device_count()


def _cuda(ev, device=0):
    import torch
    if not len(ev):
        return None
    t = torch.from_numpy(np.ascontiguousarray(ev).view(np.uint8).reshape(-1, 32).copy()).to(f"cuda:{device}")
    torch.cuda.synchronize(device)
    return t


def _batch(rng, now, B, n_targets, seq, older=True, behind=False):
    """(records, watermark): an empty batch, up to batch_cap records or past it; a watermark step within a few timer
    periods or far past the window; records from before the clock (older) and a watermark behind it (behind)"""
    r = rng.random()
    n = 0 if r < 0.1 else int(rng.integers(1, B + 1)) if r < 0.75 else int(rng.integers(B + 1, 3 * B + 6))
    if behind:
        w = now - 1
        lo = max(0, now - 4000)
    else:
        w = now + (int(rng.integers(0, 8000)) if rng.random() < 0.7 else int(rng.integers(20_000, 1_000_000)))
        lo = max(0, now - 3000) if older and rng.random() < 0.3 else now
    ev = np.zeros(n, dtype=EVENT_DTYPE)
    ev["seq"] = seq + np.arange(n)
    ev["ts_ns"] = np.sort(rng.integers(lo, w + 1, n)) if n else []
    ev["code"] = rng.integers(0, 17, n)
    odd = rng.random(n) < 0.15
    ev["code"][odd] = rng.choice(OUT, int(odd.sum()))
    ev["source_id"] = rng.integers(0, 64, n)
    ev["target"] = nat.TARGET_ALL
    ev["flags"] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32) & ~np.uint32(3)
    uni = rng.random(n) < 0.15
    ev["target"][uni] = rng.integers(0, n_targets, int(uni.sum()))   # every shard's ids, and ids not handed out yet
    ev["flags"][uni] = nat.F_UNICAST
    return ev, w


def _trace(seed, n_subs0, n_ops, K, B, jump_every=0, p_dev=0.08, p_staged=0.3, older=True, p_behind=0.03, setmask=True,
           period=(2000, 40000)):
    """the group trace of tests/test_gpu_group.py (random_ops with pairs, unicast, set_mask and clock jumps) with device
    batches in between: ('dev', records, watermark, staged).  A batch moves the clock to its watermark; the advances
    after it move by the same step."""
    ops, n_total = tr.random_ops(seed, n_subs0, n_ops, timers_per_sub=K, p_send=0.05, p_timer=0.04, p_member=0.02,
                                 p_pairs=0.3, p_flush=0.03, period_min=period[0], period_max=period[1])
    rng = np.random.default_rng(seed ^ 0xDE71CE)
    out, shift, now, seq = [], 0, 0, 1 << 40
    for i, op in enumerate(ops):
        if op[0] == "adv":
            if jump_every and i % jump_every == 0:
                shift += int(rng.integers(200, 600)) * period[0]
            op = ("adv", op[1] + shift)
            now = op[1]
        out.append(op)
        if setmask and rng.random() < 0.01:
            out.append(("setmask", int(rng.integers(0, n_total)), int(rng.integers(0, 1 << 17))))
        if rng.random() < p_dev:
            behind = now > 0 and rng.random() < p_behind
            ev, w = _batch(rng, now, B, n_total + 4, seq, older=older, behind=behind)
            seq += len(ev)
            out.append(("dev", ev, w, bool(rng.random() < p_staged)))
            if not behind:
                shift += w - now
                now = w
    return out, n_total


def _call(fn, *args):
    """(status, result) of a Bus method, whether it returns a status or raises"""
    try:
        r = fn(*args)
    except nat.CpbusError as e:
        return e.status, None
    if isinstance(r, int) and fn.__name__ in ("publish", "send", "advance", "flush"):
        return r, None
    return nat.OK, r


class _Dev:
    """device copies of the batches one bus is given, on `device`, kept alive until the bus is closed"""

    def __init__(self, device):
        self.device, self.keep = device, []

    def publish(self, bus, ev, w, staged, hint=None):
        t = _cuda(ev, self.device)
        self.keep.append(t)
        ptr = t.data_ptr() if t is not None else 0
        if not staged:
            return bus.publish_device(ptr, len(ev), w)
        if hint is None:   # the batch names itself as the next one: a valid hint that nothing may take from a cache
            hint = (ptr, len(ev)) if 0 < len(ev) <= bus.batch_cap else (0, 0)
        return bus.publish_device_staged(ptr, len(ev), w, *hint)


def _apply(bus, op, handles, dev):
    k = op[0]
    if k == "dev":
        return dev.publish(bus, op[1], op[2], op[3]), None
    if k == "sub":
        return _call(bus.subscribe_pairs, op[1], op[2]) if len(op) > 2 else _call(bus.subscribe, op[1])
    if k == "unsub":
        return _call(bus.unsubscribe, op[1])
    if k == "setmask":
        return _call(bus.set_mask, op[1], op[2])
    if k == "pub":
        return _call(bus.publish, op[1], op[2])
    if k == "send":
        return _call(bus.send, op[1], op[2], op[3])
    if k == "adv":
        return _call(bus.advance, op[1])
    if k == "tadd":
        rc, tid = _call(bus.timer_add, op[1], op[2], op[3], op[4])
        handles.append(tid)
        return rc, tid
    if k == "tcancel":
        tid = handles[op[1]] if op[1] < len(handles) else None
        return _call(bus.timer_cancel, tid) if tid is not None else (nat.OK, None)
    if k == "flush":
        return _call(bus.flush)
    raise ValueError(op)


def _eq(a, b, where):
    if isinstance(a, np.ndarray):
        assert a.tobytes() == b.tobytes(), where
    elif isinstance(a, (tuple, list)):
        assert len(a) == len(b), where
        for x, y in zip(a, b):
            _eq(x, y, where)
    else:
        assert a == b, where


def _consumers(rng, n_total, R):
    """a random consumer step, the same for both buses: ('drain', sub, cap) or ('ready', first, n, start, cap, ready_cap)"""
    if rng.random() < 0.5:
        return ("drain", int(rng.integers(0, n_total)), int(rng.integers(1, R + 1)))
    first = int(rng.integers(0, n_total))
    n = int(rng.integers(1, n_total - first + 1))
    return ("ready", first, n, first + int(rng.integers(0, n)), R + int(rng.integers(0, 3 * R)), int(rng.integers(1, 6)))


def _consume(bus, c):
    if c[0] == "drain":
        return _call(bus.drain, c[1], c[2])
    return _call(bus.drain_ready, *c[1:])


def _final(bus, n_total):
    res = [_call(bus.flush), _call(bus.sync)]
    res.append(_call(bus.digests, 0, n_total))
    res.append(_call(bus.digest_fold, 0, n_total))
    res.append(_call(bus.digest_fold, n_total // 3, n_total - n_total // 3))
    res += [_call(bus.peek_window, s) for s in range(n_total)]
    res.append(_call(bus.debug_events))
    res.append(_call(bus.publish_counts))
    res.append(_call(bus.lagging, 0, n_total))
    res.append(_call(bus.blockers))
    st = bus.stats()
    res.append({k: v for k, v in st.items() if k not in LAUNCH_SHAPED})
    res.append(_call(bus.drain_ready, 0, n_total, n_total // 2, bus.ring_cap, 3))
    return res


def _twin(seed, devices, lossless, K=4, R=64, B=32, n_subs0=24, n_ops=2500, jump_every=150, p_consume=0.08, src_dev=None,
          **kw_trace):
    """one bus and a group driven by the same trace, compared call by call and at the end; the group's batches live on
    src_dev (default: shard 0's GPU), the single bus's on its own GPU.  Returns (device batches refused with EAGAIN,
    device batches taken)."""
    ops, n_total = _trace(seed, n_subs0, n_ops, K, B, jump_every=jump_every, **kw_trace)
    rng = np.random.default_rng(seed + 77)
    kw = dict(ring_cap=R, batch_cap=B, timers_per_sub=K, lossless=lossless)
    one = Bus(n_total + 4, device=devices[0], **kw)
    grp = GroupBus(n_total + 4, devices, **kw)
    da, db = _Dev(devices[0]), _Dev(devices[0] if src_dev is None else src_dev)
    ha, hb = [], []
    n_eagain = n_dev = n_ids = 0
    try:
        for i, op in enumerate(ops):
            a, b = _apply(one, op, ha, da), _apply(grp, op, hb, db)
            _eq(a, b, f"op {i} {op[0]}: {a} vs {b}")
            n_ids += op[0] == "sub" and a[0] == nat.OK
            retries = 0
            while op[0] == "dev" and a[0] == nat.EAGAIN:
                # every consumer drains some, then the same batch is offered again: the retry delivers what the single
                # bus's retry delivers
                n_eagain += 1
                for _ in range(int(rng.integers(2, 6))):
                    c = _consumers(rng, n_ids, R)
                    _eq(_consume(one, c), _consume(grp, c), f"op {i} consumer {c}")
                a, b = _apply(one, op, ha, da), _apply(grp, op, hb, db)
                _eq(a, b, f"op {i} retry {retries}: {a} vs {b}")
                retries += 1
                if retries > 50:
                    break
            n_dev += op[0] == "dev" and a[0] == nat.OK
            if n_ids and (a[0] == nat.EAGAIN or rng.random() < p_consume):
                for _ in range(int(rng.integers(1, 4))):
                    c = _consumers(rng, n_ids, R)
                    _eq(_consume(one, c), _consume(grp, c), f"op {i} consumer {c}")
        fa, fb = _final(one, n_ids), _final(grp, n_ids)
        for j, (x, y) in enumerate(zip(fa, fb)):
            _eq(x, y, f"final item {j}")
        sa, sb = one.stats(), grp.stats()
        if not lossless:
            assert sa["device_splits"] > 0 and sb["device_splits"] > 0
    finally:
        one.close(); grp.close()
    return n_eagain, n_dev


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("G,K", [(1, 1), (2, 2), (3, 4), (4, 8)])
def test_group_device_equals_one_bus(G, K, lossless):
    """GroupBus.publish_device / _staged against Bus.publish_device / _staged on the same trace"""
    n_eagain, n_dev = _twin(1000 + 10 * G + lossless, [0] * G, lossless, K=K)
    assert n_dev > 15
    if lossless:
        assert n_eagain > 0


def test_group_device_equals_one_bus_empty_shards():
    """capacity for far more subscribers than the trace makes: the last shards stay empty, and unicast records name ids
    that were never handed out"""
    ops, n_total = _trace(31, 6, 600, 2, 32, jump_every=100)
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=2)
    one, grp = Bus(400, device=0, **kw), GroupBus(400, [0, 0, 0, 0], **kw)
    da, db = _Dev(0), _Dev(0)
    ha, hb = [], []
    try:
        for i, op in enumerate(ops):
            _eq(_apply(one, op, ha, da), _apply(grp, op, hb, db), f"op {i} {op[0]}")
        for x, y in zip(_final(one, n_total), _final(grp, n_total)):
            _eq(x, y, "final")
    finally:
        one.close(); grp.close()


@pytest.mark.parametrize("lossless", [False, True])
def test_group_device_on_distinct_gpus(lossless):
    """shards on every GPU of the box (up to 8), the batch in the HBM of a GPU other than shard 0's"""
    G = min(_n_gpus(), 8)
    if G < 2:
        pytest.skip("one GPU")
    _twin(77 + lossless, list(range(G)), lossless, K=4, src_dev=G - 1)


def _stream_of_batches(seed, n, B, count, dt=3000):
    rng = np.random.default_rng(seed)
    out, now, seq = [], 0, 1 << 30
    for q in range(count):
        ev, w = _batch(rng, now, B, n, seq, older=False)
        if len(ev) > B:
            ev = ev[:B]
        out.append((ev, w))
        seq += len(ev); now = w
    return out


def test_group_device_staged_prefetch_chain():
    """publish_device_staged with every batch naming the next one as its hint gives the results of the same calls without
    hints, on the group and on one bus"""
    n, B, R, K = 40, 64, 1024, 2
    batches = _stream_of_batches(5, n, B, 40)
    kw = dict(ring_cap=R, batch_cap=B, timers_per_sub=K)
    buses = [Bus(n, device=0, **kw), GroupBus(n, [0, 0, 0], **kw), GroupBus(n, [0, 0, 0], **kw)]
    try:
        devs = [[_cuda(ev) for ev, _ in batches] for _ in buses]
        for bus in buses:
            bus.subscribe_many(tr.zipf_masks(n, 1.0, 3))
            bus.timer_add_many(0, n, 17_000, source_id0=500)
        for q, (ev, w) in enumerate(batches):
            for j, bus in enumerate(buses):
                d = devs[j][q]
                ptr = d.data_ptr() if d is not None else 0
                if j == 1:
                    nat.check(bus.publish_device(ptr, len(ev), w), "publish_device")
                else:
                    nxt = devs[j][q + 1] if q + 1 < len(batches) else None
                    hint = (nxt.data_ptr(), len(batches[q + 1][0])) if nxt is not None else (0, 0)
                    nat.check(bus.publish_device_staged(ptr, len(ev), w, *hint), "publish_device_staged")
        res = [_final(bus, n) for bus in buses]
        for j in (1, 2):
            for x, y in zip(res[0], res[j]):
                _eq(x, y, f"bus {j}")
    finally:
        for bus in buses:
            bus.close()


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
        assert orc.timer_cancel(handles[op[1]]) in (0, ob.ENOENT)
    elif k == "dev":
        assert orc.publish_records(op[1], op[2]) == 0


@pytest.mark.parametrize("G", [2, 3])
def test_group_device_against_oracle(G):
    """host publishes, sends, timers and device batches (split ones included) against the oracle's mailboxes, publish
    counts by code and debug events"""
    R, B = 1024, 64
    ops, n_total = _trace(60 + G, 20, 900, 2, B, older=False, p_behind=0, setmask=False, p_dev=0.1, period=(20000, 40000))
    orc = ob.Oracle(n_total + 4, timers_per_sub=2, keep_window=R)
    dev, hb, ho = _Dev(0), [], []
    with GroupBus(n_total + 4, [0] * G, ring_cap=R, batch_cap=B, timers_per_sub=2) as grp:
        for i, op in enumerate(ops):
            rc, _ = _apply(grp, op, hb, dev)
            if op[0] == "tcancel":
                assert rc in (nat.OK, nat.ENOENT)
            else:
                assert rc == nat.OK, (i, op[0], rc)
            _oracle_apply(orc, op, ho)
        nat.check(grp.flush(), "flush"); grp.sync()
        st = tr.compare(grp, orc, n_total, window=R)
        assert st["published_by_code"] == [orc.published_by_code(c) for c in range(nat.N_CODES)]
        assert grp.debug_events().tobytes() == orc.debug_events().tobytes()
        assert st["device_splits"] > 0


def _digests_and_deliveries(bus, n):
    bus.sync()
    return bus.digests(0, n).tobytes(), bus.stats()["deliveries"]


@pytest.mark.parametrize("G", [1, 3])
def test_lossless_refusals(G):
    """CPBUS_EAGAIN with nothing delivered on any shard; the retry after the consumers drain delivers what the single bus's
    retry delivers; CPBUS_EINVAL past batch_cap, CPBUS_EORDER past the timer window, CPBUS_EINVAL from _staged"""
    n, R, B = 30, 64, 32
    kw = dict(ring_cap=R, batch_cap=B, timers_per_sub=2, lossless=True)
    one, grp = Bus(n, device=0, **kw), GroupBus(n, [0] * G, **kw)
    rng = np.random.default_rng(9)
    da, db = _Dev(0), _Dev(0)
    try:
        for bus in (one, grp):
            bus.subscribe_many(np.full(n, nat.MASK_ALL, dtype=np.uint32))
            bus.timer_add(n - 1, 10_000, 7)                         # the window: 16 periods at K = 2
        now, seq, stalls = 0, 1 << 20, 0
        for q in range(12):
            ev, w = _batch(rng, now, B, n, seq, older=False)
            ev, w = ev[:B], min(w, now + 5000)
            ev["ts_ns"] = np.minimum(ev["ts_ns"], w)
            seq += len(ev)
            while True:
                before = [_digests_and_deliveries(b, n) for b in (one, grp)]
                a, b = da.publish(one, ev, w, False), db.publish(grp, ev, w, False)
                assert a == b, (q, a, b)
                if a == nat.OK:
                    break
                assert a == nat.EAGAIN
                stalls += 1
                assert [_digests_and_deliveries(x, n) for x in (one, grp)] == before   # nothing delivered anywhere
                for s in range(n):
                    cap = int(rng.integers(4, 20))
                    _eq(one.drain(s, cap), grp.drain(s, cap), f"drain {s}")
            now = w
        assert stalls > 0
        big = np.zeros(B + 1, dtype=EVENT_DTYPE); big["ts_ns"] = now; big["target"] = nat.TARGET_ALL
        for bus, d in ((one, da), (grp, db)):
            assert d.publish(bus, big, now, False) == nat.EINVAL
            assert d.publish(bus, big[:1], now + 10_000 * 17, False) == nat.EORDER
            assert d.publish(bus, big[:1], now, True) == nat.EINVAL
            assert d.publish(bus, big[:1], now - 1, False) == nat.EORDER
        for x, y in zip(_final(one, n), _final(grp, n)):
            _eq(x, y, "final")
    finally:
        one.close(); grp.close()


def test_drop_missed_group_refuses_device_batches():
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=2, drop_missed_ticks=True)
    one, grp = Bus(8, device=0, **kw), GroupBus(8, [0, 0], **kw)
    ev = np.zeros(4, dtype=EVENT_DTYPE); ev["ts_ns"] = 5; ev["target"] = nat.TARGET_ALL
    try:
        for bus in (one, grp):
            bus.subscribe_many(np.full(8, nat.MASK_ALL, dtype=np.uint32))
            d = _Dev(0)
            assert d.publish(bus, ev, 10, False) == nat.EINVAL
            assert d.publish(bus, ev, 10, True) == nat.EINVAL
            assert bus.stats()["publishes"] == 0
    finally:
        one.close(); grp.close()
