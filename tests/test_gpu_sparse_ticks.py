"""Sparse timer delivery (CPBUS_CFG_SPARSE_TICKS): a flagged bus gives the results of an unflagged twin that makes the same
calls — return codes, drains, sparse drains, windows, digests, folds, lagging and blockers, debug events, publish counts
and every stat but the launch-shaped ones — in throughput and lossless mode, with pairs, unicast, set_mask, cancels,
unsubscribes, one-shots, clock jumps, device batches and due times near 2^64; and the oracle's mailboxes.  A flush with
nothing due launches nothing, one with a few due ticks launches one kernel, one with many runs the full fan-out."""
import numpy as np
import pytest
import torch

import oracle_binding as ob  # noqa: F401  (builds the oracle the trace helpers use)
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from test_gpu_group import LAUNCH_SHAPED, _apply, _consume, _consumers, _eq, _final, _trace

pytestmark = pytest.mark.gpu
TOP = (1 << 64) - 1


def _queries(bus, n_total):
    return [bus.lagging(0, n_total, n_total // 2, 1), bus.blockers()]


def _twins(seed, lossless, K, R=64, B=32, n_subs0=24, n_ops=1500, jump_every=150, p_consume=0.08, t0=0, p_long=0.0,
           device_every=0):
    """Run one trace on a flagged and an unflagged bus, comparing every result; returns (EAGAINs, flagged bus stats).
    t0: the trace's clock starts there (and stops at 2^64 - 2); p_long: the share of timers whose first due time lies
    within 2^21 of 2^64 - 1 (some fire, their re-arms saturate)."""
    ops, n_total = _trace(seed, n_subs0, n_ops, K, jump_every=jump_every)
    rng = np.random.default_rng(seed + 91)
    kw = dict(ring_cap=R, batch_cap=B, timers_per_sub=K, lossless=lossless, device=0)
    plain, sparse = Bus(n_total + 4, **kw), Bus(n_total + 4, sparse_ticks=True, **kw)
    ha, hb = [], []
    n_eagain = n_ids = 0
    try:
        if t0:
            assert plain.advance(t0) == sparse.advance(t0) == nat.OK
        for i, op in enumerate(ops):
            if op[0] == "adv":
                op = ("adv", min(op[1] + t0, TOP - 1))
            elif op[0] == "tadd" and p_long and rng.random() < p_long:
                op = ("tadd", op[1], max(1, TOP - plain.stats()["now_ns"] - int(rng.integers(0, 1 << 21))), op[3], op[4])
            a, b = _apply(plain, op, ha), _apply(sparse, op, hb)
            _eq(a, b, f"op {i} {op}: {a} vs {b}")
            n_eagain += a[0] == nat.EAGAIN
            n_ids += op[0] == "sub" and a[0] == nat.OK
            if device_every and i % device_every == device_every - 1 and n_ids:
                _device_batch(plain, sparse, rng, n_ids, lossless)
            if n_ids and (a[0] == nat.EAGAIN or rng.random() < p_consume):
                for _ in range(int(rng.integers(1, 4))):
                    c = _consumers(rng, n_ids, R)
                    _eq(_consume(plain, c), _consume(sparse, c), f"op {i} consumer {c}")
            if n_ids and rng.random() < 0.02:
                for x, y in zip(_queries(plain, n_ids), _queries(sparse, n_ids)):
                    _eq(x, y, f"op {i} queries")
        for x, y in zip(_final(plain, n_ids), _final(sparse, n_ids)):
            _eq(x, y, "final")
        return n_eagain, sparse.stats()
    finally:
        plain.close(); sparse.close()


def _device_batch(plain, sparse, rng, n_ids, lossless):
    """the same complete records through cpbus_publish_device on both buses, at a watermark a little past the clock"""
    now = plain.stats()["now_ns"]
    assert sparse.stats()["now_ns"] == now
    n = int(rng.integers(0, 24))
    w = now + int(rng.integers(0, 3000))
    ev = np.zeros(n, dtype=EVENT_DTYPE)
    ev["seq"] = np.arange(n) + 10_000_000
    ev["ts_ns"] = np.sort(rng.integers(now, w + 1, n)) if n else []
    ev["code"] = rng.integers(0, 17, n)
    ev["source_id"] = rng.integers(0, 8, n)
    uni = rng.random(n) < 0.2
    ev["target"] = np.where(uni, rng.integers(0, n_ids, n), nat.TARGET_ALL)
    ev["flags"] = np.where(uni, nat.F_UNICAST, 0)
    d = torch.from_numpy(ev.view(np.uint8).reshape(-1, 32).copy()).cuda() if n else None
    torch.cuda.synchronize()
    ptr = d.data_ptr() if d is not None else 0
    ra, rb = plain.publish_device(ptr, n, w), sparse.publish_device(ptr, n, w)
    assert ra == rb, (ra, rb)
    plain.sync(); sparse.sync()


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
def test_flagged_bus_equals_unflagged_twin(K, lossless):
    n_eagain, st = _twins(100 * K + lossless, lossless, K)
    if lossless:
        assert n_eagain > 0   # mailboxes kept nearly full: tick flushes that the room bound cannot prove fit fall back


@pytest.mark.parametrize("lossless", [False, True])
def test_twins_with_device_batches(lossless):
    _twins(7 + lossless, lossless, 2, n_ops=1000, device_every=25)


@pytest.mark.parametrize("lossless", [False, True])
def test_twins_near_the_top_of_the_clock(lossless):
    _twins(31 + lossless, lossless, 4, n_ops=1000, t0=TOP - (1 << 22), p_long=0.3)


@pytest.mark.parametrize("env", [("CPBUS_PDL", "0"), ("CPBUS_HINTS", "2")])
@pytest.mark.parametrize("lossless", [False, True])
def test_twins_with_knobs(env, lossless, monkeypatch):
    monkeypatch.setenv(*env)
    _twins(55 + lossless, lossless, 4, n_ops=800)


@pytest.mark.parametrize("lossless", [False, True])
def test_flagged_bus_against_oracle(lossless):
    ops, n_total = tr.random_ops(60 + lossless, 20, 700 if lossless else 1500, timers_per_sub=2, p_pairs=0.3, p_send=0.05,
                                 period_min=20000)            # lossless: no mailbox of the oracle ever fills
    R = 1024
    orc = tr.run_oracle(ops, n_total + 4, timers_per_sub=2, keep_window=R, mailbox_cap=R if lossless else 0)
    with Bus(n_total + 4, ring_cap=R, batch_cap=256, timers_per_sub=2, lossless=lossless, sparse_ticks=True) as bus:
        tr.run_bus(bus, ops)
        tr.compare(bus, orc, n_total, window=R)


def _launches(bus):
    st = bus.stats()
    return st["kernel_launches"], st["batches"]


@pytest.mark.parametrize("lossless", [False, True])
def test_launch_counts_by_path(lossless):
    """N = 4096, so past 32 due slots a flush with no record takes the full fan-out"""
    N, K = 4096, 1
    kw = dict(ring_cap=1024, batch_cap=256, timers_per_sub=K, lossless=lossless, device=0)
    with Bus(N, **kw) as plain, Bus(N, sparse_ticks=True, **kw) as sparse:
        for bus in (plain, sparse):
            bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
            bus.timer_add_many(0, 20, 1000, source_id0=7)           # 20 due every 1,000 ns
            bus.timer_add_many(20, 1000, 7000, source_id0=500)      # 1,000 more due at 7,000 ns
            bus.timer_add_many(1020, N - 1020, 10 ** 9, source_id0=9)

        def step(now):
            before = _launches(sparse)
            for bus in (plain, sparse):
                assert bus.advance(now) == nat.OK and bus.flush() == nat.OK
            res = [bus.step_result_end(bus.step_result_begin()) for bus in (plain, sparse)]
            return before, _launches(sparse), res

        b0, b1, _ = step(500)                  # nothing due
        assert b1 == b0
        r0 = sparse.step_result_end(sparse.step_result_begin())
        b0, b1, (rp, rs) = step(1000)          # 20 due slots: one sparse kernel, not a fan-out batch
        assert b1 == (b0[0] + 1, b0[1])
        assert rs[:3] == rp[:3] and rs[0] == rs[1] == 20 and rs[3] != r0[3]
        b0, b1, _ = step(1500)                 # idle again: the step result stays that of the sparse kernel
        assert b1 == b0 and sparse.step_result_end(sparse.step_result_begin()) == rs
        b0, b1, (rp, rs) = step(7000)          # 20 + 1,000 due: the full fan-out
        assert b1[1] == b0[1] + 1 and rs[:3] == rp[:3] and rs[1] == 20 * 6 + 1000
        b0 = _launches(sparse)
        for bus in (plain, sparse):            # with a record: the full fan-out, whatever is due
            assert bus.advance(8000) == nat.OK and bus.publish(3, 1) == nat.OK and bus.flush() == nat.OK
        assert _launches(sparse)[1] == b0[1] + 1
        for x, y in zip(_final(plain, N), _final(sparse, N)):
            _eq(x, y, "final")


def test_streams_refuse_a_flagged_bus():
    with Bus(64, ring_cap=64, batch_cap=32, timers_per_sub=1, sparse_ticks=True, device=0) as sparse, \
            Bus(64, ring_cap=64, batch_cap=32, timers_per_sub=1, device=0) as plain:
        with pytest.raises(nat.CpbusError) as e:
            sparse.stream_create(8, 2)
        assert e.value.status == nat.EINVAL
        st, handle = plain.stream_create(8, 2)
        try:
            with pytest.raises(nat.CpbusError) as e:
                sparse.stream_attach(st, 1)
            assert e.value.status == nat.EINVAL
            with pytest.raises(nat.CpbusError) as e:
                sparse.stream_open(handle, 1)
            assert e.value.status == nat.EINVAL
        finally:
            plain.stream_close(st)
