"""Sparse record delivery (CPBUS_CFG_SPARSE_RECORDS): a flagged bus gives the results of an unflagged twin that makes the
same calls — return codes, drains, sparse drains, windows, digests, folds, lagging and blockers, debug events, publish
counts and every stat but the launch-shaped ones — in throughput and lossless mode, with pairs, unicast, set_mask, cancels,
unsubscribes, one-shots, clock jumps, device batches and clocks near 2^64; and the oracle's mailboxes.  A flush whose
records reach a few mailboxes launches one kernel over them, one that reaches many runs the full fan-out, and so does a
device batch; a lossless flush the room bound cannot prove falls back and stalls where the twin stalls."""
import numpy as np
import pytest

import oracle_binding as ob  # noqa: F401  (builds the oracle the trace helpers use)
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200 import events as ev
from containerpilot_b200 import masks as mk
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from test_gpu_group import _apply, _consume, _consumers, _eq, _final, _trace
from test_gpu_sparse_ticks import _device_batch, _queries

pytestmark = pytest.mark.gpu
TOP = (1 << 64) - 1


def _twins(seed, lossless, K, R=64, B=32, n_subs0=24, n_ops=1500, jump_every=150, p_consume=0.08, t0=0, p_long=0.0,
           device_every=0):
    """One trace on a flagged bus and an unflagged one, every result compared; returns (EAGAINs, flagged bus stats)."""
    ops, n_total = _trace(seed, n_subs0, n_ops, K, jump_every=jump_every)
    rng = np.random.default_rng(seed + 91)
    kw = dict(ring_cap=R, batch_cap=B, timers_per_sub=K, lossless=lossless, device=0)
    plain, sparse = Bus(n_total + 4, **kw), Bus(n_total + 4, sparse_records=True, **kw)
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


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("K", [0, 1, 2, 4, 8])
def test_flagged_bus_equals_unflagged_twin(K, lossless):
    n_eagain, st = _twins(300 + 10 * K + lossless, lossless, K)
    assert st["kernel_launches"] > st["batches"]   # the record kernel ran
    if lossless:
        assert n_eagain > 0   # mailboxes kept nearly full: flushes the room bound cannot prove fall back


@pytest.mark.parametrize("lossless", [False, True])
def test_twins_with_device_batches(lossless):
    _twins(17 + lossless, lossless, 2, n_ops=1000, device_every=25)


@pytest.mark.parametrize("lossless", [False, True])
def test_twins_near_the_top_of_the_clock(lossless):
    _twins(41 + lossless, lossless, 4, n_ops=1000, t0=TOP - (1 << 22), p_long=0.3)


@pytest.mark.parametrize("env", [("CPBUS_PDL", "0"), ("CPBUS_HINTS", "2")])
@pytest.mark.parametrize("lossless", [False, True])
def test_twins_with_knobs(env, lossless, monkeypatch):
    monkeypatch.setenv(*env)
    _twins(65 + lossless, lossless, 4, n_ops=800)


@pytest.mark.parametrize("lossless", [False, True])
def test_flagged_bus_against_oracle(lossless):
    ops, n_total = tr.random_ops(70 + lossless, 20, 700 if lossless else 1500, timers_per_sub=2, p_pairs=0.3, p_send=0.05,
                                 period_min=20000)            # lossless: no mailbox of the oracle ever fills
    R = 1024
    orc = tr.run_oracle(ops, n_total + 4, timers_per_sub=2, keep_window=R, mailbox_cap=R if lossless else 0)
    with Bus(n_total + 4, ring_cap=R, batch_cap=256, timers_per_sub=2, lossless=lossless, sparse_records=True) as bus:
        tr.run_bus(bus, ops)
        tr.compare(bus, orc, n_total, window=R)


def _launches(bus):
    st = bus.stats()
    return st["kernel_launches"], st["batches"]


def _result(bus):
    return bus.step_result_end(bus.step_result_begin())


@pytest.mark.parametrize("lossless", [False, True])
def test_launch_counts_by_path(lossless):
    """N = 4096, so past 32 mailboxes a flush with records takes the full fan-out"""
    import torch
    N, K = 4096, 1
    kw = dict(ring_cap=1024, batch_cap=256, timers_per_sub=K, lossless=lossless, device=0)
    masks = np.full(N, 1 << 5, dtype=np.uint32)
    masks[:10] = 1 << 3                       # code 3: 10 mailboxes; code 5: the other 4,086
    masks[100:200] = 1 << 6                   # code 6: 100 mailboxes, more than the index lists (64)
    with Bus(N, **kw) as plain, Bus(N, sparse_records=True, **kw) as sparse:
        both = (plain, sparse)
        for bus in both:
            bus.subscribe_many(masks)
            bus.timer_add_many(20, 5, 1000, source_id0=7)            # 5 mailboxes due every 1,000 ns

        def step(now, code, n=1, expect=nat.OK):
            before = _launches(sparse)
            for bus in both:
                assert bus.advance(now) == nat.OK
                for _ in range(n):
                    assert bus.publish(code, 1) == nat.OK
                assert bus.flush() == expect
            return before, _launches(sparse), [_result(bus) for bus in both]

        b0, b1, (rp, rs) = step(500, 3)         # 10 mailboxes, nothing due: one record kernel, not a fan-out batch
        assert b1 == (b0[0] + 1, b0[1]) and rs[:3] == rp[:3] == (10, 0, rs[2])
        b0, b1, (rp, rs) = step(1000, 3, n=3)   # the same 10 and 5 due ticks
        assert b1 == (b0[0] + 1, b0[1]) and rs[:3] == rp[:3] and rs[0] == 35 and rs[1] == 5
        r0 = _result(sparse)
        b0, b1, _ = step(1200, 9)               # nobody takes code 9: nothing launched, the step result stays
        assert b1 == b0 and _result(sparse) == r0
        b0, b1, (rp, rs) = step(1500, 5)        # 4,086 mailboxes: the full fan-out
        assert b1[1] == b0[1] + 1 and rs[:3] == rp[:3]
        b0, b1, (rp, rs) = step(1600, 6)        # 100 mailboxes: the full fan-out (the code's list is dropped)
        assert b1[1] == b0[1] + 1 and rs[:3] == rp[:3]
        for bus in both:                        # down to 10 subscribers of code 6: the list comes back
            for s in range(110, 200):
                bus.unsubscribe(s)
        b0, b1, (rp, rs) = step(1700, 6)
        assert b1 == (b0[0] + 1, b0[1]) and rs[:3] == rp[:3] and rs[0] == 10
        for bus in both:                        # set_mask moves a mailbox between codes
            bus.set_mask(3, 1 << 6)
        b0, b1, (rp, rs) = step(1800, 6)
        assert b1 == (b0[0] + 1, b0[1]) and rs[:3] == rp[:3] and rs[0] == 11
        ev_ = np.zeros(2, dtype=EVENT_DTYPE)    # a device batch: the full fan-out, whoever it reaches
        ev_["ts_ns"], ev_["code"], ev_["target"] = 1900, 3, nat.TARGET_ALL
        d = torch.from_numpy(ev_.view(np.uint8).reshape(-1, 32).copy()).cuda()
        torch.cuda.synchronize()
        b0 = _launches(sparse)
        for bus in both:
            assert bus.publish_device(d.data_ptr(), 2, 1900) == nat.OK
        assert _launches(sparse)[1] == b0[1] + 1
        for x, y in zip(_final(plain, N), _final(sparse, N)):
            _eq(x, y, "final")


def test_lossless_fallback_stalls_where_the_twin_stalls():
    """ring_cap 64: 40 records reach 10 mailboxes (the room bound proves the fit), 40 more do not fit: the flagged bus
    runs the admission pass, delivers the same prefix and returns CPBUS_EAGAIN with its twin"""
    N = 256
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=1, lossless=True, device=0)
    masks = np.zeros(N, dtype=np.uint32)
    masks[:10] = 1 << 3
    with Bus(N, **kw) as plain, Bus(N, sparse_records=True, **kw) as sparse:
        both = (plain, sparse)
        for bus in both:
            bus.subscribe_many(masks)
        ev_ = np.zeros(1, dtype=EVENT_DTYPE)
        ev_["code"] = 3

        def burst(n):
            out = []
            for bus in both:
                rcs = []
                for _ in range(n):
                    rcs.append(bus.publish_many(ev_))
                rcs.append(bus.flush())
                out.append(rcs)
            assert out[0] == out[1]
            return out[0]

        b0 = sparse.stats()
        assert set(burst(20)) == {nat.OK}
        b1 = sparse.stats()
        assert b1["batches"] == b0["batches"] and b1["admit_passes"] == b0["admit_passes"]
        assert set(burst(20)) == {nat.OK}          # 40 in each mailbox, bound 24 left
        rcs = burst(30)                            # 30 more: only 24 fit
        assert rcs[-1] == nat.EAGAIN or nat.EAGAIN in rcs
        b2 = sparse.stats()
        assert b2["admit_passes"] > b1["admit_passes"] and b2["admit_partial"] == plain.stats()["admit_partial"] > 0
        for x, y in zip(_final(plain, 12), _final(sparse, 12)):
            _eq(x, y, "stalled")
        for bus in both:
            bus.consume_all()
            assert bus.flush() == nat.OK
        for x, y in zip(_final(plain, N), _final(sparse, N)):
            _eq(x, y, "final")


FIXED = {"": 0, "global": 1, "closed": 2, "SIGHUP": 3, "SIGUSR2": 4}


def _sid(name):
    """source ids of a Job fleet: the fixed names, then 5 per job (name, check, heartbeat, run-every, wait-timeout)"""
    if name in FIXED:
        return FIXED[name]
    base, _, suffix = name.partition(".")
    if base == "check":
        return 5 + 5 * int(suffix[3:]) + 1
    return 5 + 5 * int(base[3:]) + {"": 0, "heartbeat": 2, "run-every": 3, "wait-timeout": 4}[suffix]


def _job_fleet(n, rng):
    subs = []
    for j in range(n):
        dep = int(rng.integers(0, n))
        sw = mk.JobSwitch(f"job{j}", start_event=ev.Event(ev.ExitSuccess, f"job{dep}") if j % 3 else ev.GlobalStartup)
        m, cases = sw.cases()
        subs.append((m, [(e.Code, _sid(e.Source)) for e in cases]))
    return subs


@pytest.mark.parametrize("lossless", [False, True])
def test_job_fleet_drained_with_drain_ready(lossless):
    """a Job-shaped fleet (the switch's code mask and exact cases), 1-event and 64-event publishes, drained with
    drain_ready: the flagged bus and its twin return the same records and ready lists"""
    rng = np.random.default_rng(11 + lossless)
    N = 2048
    subs = _job_fleet(N, rng)
    kw = dict(ring_cap=256, batch_cap=64, timers_per_sub=2, lossless=lossless, device=0)
    with Bus(N, **kw) as plain, Bus(N, sparse_records=True, **kw) as sparse:
        both = (plain, sparse)
        for bus in both:
            bus.subscribe_pairs_many([m for m, _ in subs], [c for _, c in subs])
            bus.timer_add_many(0, 64, 50_000, source_id0=7)
        now = 0
        for step in range(120):
            now += 10_000
            n = 1 if step % 3 else 64
            e = np.zeros(n, dtype=EVENT_DTYPE)
            e["code"] = rng.integers(1, 17, n)
            e["source_id"] = rng.integers(0, 5 + 5 * N, n)
            res = [(bus.advance(now), bus.publish_many(e), bus.flush()) for bus in both]
            assert res[0] == res[1], (step, res)
            if step % 10 == 9:
                first = int(rng.integers(0, N))
                args = (0, N, first, 4096, 256)
                _eq(plain.drain_ready(*args), sparse.drain_ready(*args), f"step {step}")
        for x, y in zip(_final(plain, N), _final(sparse, N)):
            _eq(x, y, "final")
        assert sparse.stats()["batches"] < plain.stats()["batches"]


def test_events_bus_with_sparse_records():
    """the reference-restated EventBus scenarios of tests/test_gpu_events_api.py (those without arguments) on a bus with
    the flag; not the one that counts fan-out batches, a launch-shaped stat the flag changes"""
    import inspect
    import test_gpu_events_api as api
    names = [n for n in dir(api) if n.startswith("test_") and callable(getattr(api, n)) and "fan_out" not in n
             and not inspect.signature(getattr(api, n)).parameters]
    assert names
    orig = ev.EventBus.__init__

    def flagged(self, *a, **k):
        if k.get("devices") is None:
            k["sparse_records"] = True
        orig(self, *a, **k)
    ev.EventBus.__init__ = flagged
    try:
        ran = 0
        for n in names:
            getattr(api, n)()
            ran += 1
        assert ran > 0
    finally:
        ev.EventBus.__init__ = orig
