"""Sparse drains (CPBUS_CFG_SPARSE_DRAINS) on the GPU: a flagged bus gives the results of a twin without the flag that makes
the same calls.  Seeded traces of publishes, sends, clock steps, timers (K = 0 .. 8), subscribes, unsubscribes, re-masks,
releases and subscribe_list reuse, exact cases, device batches and consume_all run on both, drained with cpbus_drain_ready,
cpbus_take_ready + cpbus_ack_many and tickets begun and ended out of order with deliveries in between, over random ranges,
start ids, caps and ready caps; every status and output is compared byte for byte, and at the end every query and every
stat but kernel_launches.  The launches each path takes, the C oracle's mailboxes, and a Go-shaped pump on a Job fleet."""
import numpy as np
import pytest
import torch

import oracle_binding as ob  # noqa: F401  (builds the oracle the trace helpers use)
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200 import events as ev
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from test_gpu_drain_tickets import _Run, _same, _state, _status, _trace
from test_gpu_sparse_records import _job_fleet

pytestmark = pytest.mark.gpu
R, BATCH, MAX_SUBS = 64, 32, 48


def _pair(K, lossless, records=True, drop_missed=False):
    kw = dict(ring_cap=R, batch_cap=BATCH, timers_per_sub=K, lossless=lossless, device=0, sparse_ticks=True,
              sparse_records=records, drop_missed_ticks=drop_missed)
    return Bus(MAX_SUBS, **kw), Bus(MAX_SUBS, sparse_drains=True, **kw)


def _ready_result(r):
    return r if isinstance(r, int) else (r[0].tobytes(), r[1].tobytes(), r[2])


def _call(fn, *args):
    try:
        return _ready_result(fn(*args))
    except nat.CpbusError as e:
        return e.status


def _device_batch(buses, rng, n_ids):
    """the same records through cpbus_publish_device on both buses, at a watermark a little past the clock"""
    now = buses[0].stats()["now_ns"]
    n = int(rng.integers(1, 24))
    w = now + int(rng.integers(0, 3000))
    e = np.zeros(n, dtype=EVENT_DTYPE)
    e["seq"] = np.arange(n) + 10_000_000
    e["ts_ns"] = np.sort(rng.integers(now, w + 1, n))
    e["code"] = rng.integers(0, 17, n)
    e["source_id"] = rng.integers(0, 8, n)
    e["target"] = np.where(rng.random(n) < 0.2, rng.integers(0, n_ids, n), nat.TARGET_ALL)
    e["flags"] = np.where(e["target"] != nat.TARGET_ALL, nat.F_UNICAST, 0)
    d = torch.from_numpy(e.view(np.uint8).reshape(-1, 32).copy()).cuda()
    torch.cuda.synchronize()
    return [b.publish_device(d.data_ptr(), n, w) for b in buses]


def _twins(seed, K, lossless, records=True, drop_missed=False, n_ops=500):
    rng = np.random.default_rng(seed + 7000)
    a, b = _pair(K, lossless, records, drop_missed)
    both = (a, b)
    pending = []                    # (ticket on a, ticket on b, cap, ready_cap, where)
    n_list = n_none = 0
    try:
        ra, rb = _Run(a), _Run(b)

        def end(k):
            ta, tb, cap, ready_cap, where = pending.pop(k)
            assert _call(a.drain_ready_end, ta, cap, ready_cap) == _call(b.drain_ready_end, tb, cap, ready_cap), where

        def take_ack(x, args):
            r = x.take_ready(*args)
            return _ready_result(r), x.ack_many(r[1]["sub_id"], r[1]["count"]).tolist() if len(r[1]) else []

        for i, op in enumerate(_trace(seed, n_ops)):
            assert ra.step(op) == rb.step(op), (i, op)
            if not ra.ids:
                continue
            n_ids = max(ra.ids) + 1
            where = (i, op)
            if rng.random() < 0.03:
                rc = _device_batch(both, rng, n_ids)
                assert rc[0] == rc[1], where
            if rng.random() < 0.02:
                assert a.consume_all() is None and b.consume_all() is None
            if op[0] != "pump":
                continue
            if rng.random() < 0.6:
                first, n = 0, n_ids
            else:
                first = int(rng.integers(0, n_ids))
                n = int(rng.integers(1, n_ids - first + 1))
            start = first + int(rng.integers(0, n))
            cap = int(rng.choice([R, R + 7, 2 * R, 64 * R]))
            ready_cap = int(rng.choice([1, 2, 3, 64]))
            args = (first, n, start, cap, ready_cap)
            kind = rng.random()
            before = b.stats()["kernel_launches"]
            if kind < 0.35:
                assert _call(a.drain_ready, *args) == _call(b.drain_ready, *args), where
            elif kind < 0.55 and lossless:
                assert take_ack(a, args) == take_ack(b, args), where
            elif len(pending) < 9:
                take = lossless and rng.random() < 0.4
                name = "take_ready_begin" if take else "drain_ready_begin"
                ta, tb = _status(getattr(a, name), *args), _status(getattr(b, name), *args)
                assert (ta < 0) == (tb < 0) and (ta == tb if ta < 0 else True), where
                if ta >= 0:
                    pending.append((ta, tb, cap, ready_cap, where))
            added = b.stats()["kernel_launches"] - before
            n_none += added == 0
            n_list += added == 2
            while pending and (len(pending) >= 8 or rng.random() < 0.3):
                end(int(rng.integers(0, len(pending))))
        while pending:
            end(int(rng.integers(0, len(pending))))
        n_ids = max(ra.ids) + 1
        assert _state(a, 0, n_ids) == _state(b, 0, n_ids)
        assert a.publish_counts() == b.publish_counts()
        _same(a.drain_ready(0, n_ids, 0, 64 * R, 64), b.drain_ready(0, n_ids, 0, 64 * R, 64), "final")
        assert n_none > 0   # some drains needed no launch at all
    finally:
        a.close(); b.close()


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("K", [0, 1, 2, 4, 8])
def test_flagged_bus_equals_twin(K, lossless):
    _twins(100 + 10 * K + lossless, K, lossless)


@pytest.mark.parametrize("lossless", [False, True])
def test_twins_without_sparse_records(lossless):
    _twins(31 + lossless, 2, lossless, records=False)


@pytest.mark.parametrize("lossless", [False, True])
def test_twins_with_drop_missed_ticks(lossless):
    _twins(57 + lossless, 4, lossless, drop_missed=True)


def _launches(bus):
    return bus.stats()["kernel_launches"]


@pytest.mark.parametrize("lossless", [False, True])
def test_launch_counts_by_path(lossless):
    N = 4096
    kw = dict(ring_cap=1024, batch_cap=256, timers_per_sub=1, lossless=lossless, device=0)
    with Bus(N, sparse_records=True, **kw) as plain, Bus(N, sparse_records=True, sparse_drains=True, **kw) as bus:
        masks = np.full(N, 1 << 5, dtype=np.uint32)
        masks[7] = 1 << 3                               # code 3 reaches mailbox 7 alone
        drain = bus.take_ready if lossless else bus.drain_ready
        pdrain = plain.take_ready if lossless else plain.drain_ready
        for x in (plain, bus):
            x.subscribe_many(masks)

        def step(expect, code=None, start=0):
            for x in (plain, bus):
                if code is not None:
                    assert x.publish(code, 1) == nat.OK
                assert x.flush() == nat.OK
            b0 = _launches(bus)
            got = drain(0, N, start, 4096, 4096)
            want = pdrain(0, N, start, 4096, 4096)
            assert _launches(bus) - b0 == expect
            _same(want, got, (expect, code))
            if lossless:
                for x, r in ((plain, want), (bus, got)):
                    assert (x.ack_many(r[1]["sub_id"], r[1]["count"]) == nat.OK).all()
            return got

        step(0)                                          # nothing launched since creation: no launch
        got = step(2, code=3, start=100)                 # one mailbox: the list scan and the gather
        assert got[1]["sub_id"].tolist() == [7] and got[2] == 100
        step(0)                                          # after a complete drain: free again
        step(2, code=5)                                  # the full fan-out: the dense scan (2 launches) ...
        step(0)                                          # ... which was complete over the whole range: free again
        b0 = _launches(bus)                              # a ticket that finds nothing takes a slot and launches nothing
        t = (bus.take_ready_begin if lossless else bus.drain_ready_begin)(0, N, 0, 4096, 16)
        assert _launches(bus) == b0
        r = bus.drain_ready_end(t, 4096, 16)
        assert len(r[1]) == 0 and r[2] == 0
        for x in (plain, bus):                           # a partial drain after a fan-out does not make the set known
            assert x.publish(5, 2) == nat.OK and x.flush() == nat.OK
            x.drain_ready(0, N - 1, 0, 4096 * 1024, N) if not lossless else x.take_ready(0, N - 1, 0, 4096 * 1024, N)
        step(2)
        step(0)


@pytest.mark.parametrize("lossless", [False, True])
def test_flagged_bus_against_oracle(lossless):
    ops, n_total = tr.random_ops(80 + lossless, 20, 700 if lossless else 1500, timers_per_sub=2, p_pairs=0.3, p_send=0.05,
                                 period_min=20000)
    R_ = 1024
    orc = tr.run_oracle(ops, n_total + 4, timers_per_sub=2, keep_window=R_, mailbox_cap=R_ if lossless else 0)
    with Bus(n_total + 4, ring_cap=R_, batch_cap=256, timers_per_sub=2, lossless=lossless, sparse_records=True,
             sparse_drains=True) as bus:
        tr.run_bus(bus, ops)
        tr.compare(bus, orc, n_total, window=R_)


def test_go_shaped_pump_on_a_job_fleet():
    """The Go shim's loop on a Job fleet: each 1 ms step advances, flushes, takes every ready mailbox over [0, n) and acks
    it; every 10th step publishes one event first.  The flagged bus delivers what its twin delivers, and its idle steps
    launch nothing."""
    rng = np.random.default_rng(5)
    N = 2048
    subs = _job_fleet(N, rng)
    kw = dict(ring_cap=256, batch_cap=64, timers_per_sub=2, lossless=True, device=0, sparse_records=True)
    with Bus(N, **kw) as plain, Bus(N, sparse_drains=True, **kw) as bus:
        for x in (plain, bus):
            x.subscribe_pairs_many([m for m, _ in subs], [c for _, c in subs])
            x.timer_add_many(0, 32, 7_000_000, source_id0=7)
        idle = 0
        for step in range(300):
            now = (step + 1) * 1_000_000
            codes = int(rng.integers(1, 17)), int(rng.integers(0, 5 + 5 * N))
            b0 = _launches(bus)
            res = []
            for x in (plain, bus):
                r = [x.advance(now)]
                if step % 10 == 0:
                    r.append(x.publish(*codes))
                r.append(x.flush())
                got = x.take_ready(0, N, 0, 1 << 16, N)
                x.ack_many(got[1]["sub_id"], got[1]["count"])
                res.append((r, got[0].tobytes(), got[1].tobytes(), got[2]))
            assert res[0] == res[1], step
            idle += _launches(bus) == b0
        assert idle > 100
        assert _state(plain, 0, N) == _state(bus, 0, N)


def test_events_bus_with_sparse_drains():
    """the reference-restated EventBus scenarios of tests/test_gpu_events_api.py (those without arguments) on a bus with
    the flag; not the one that counts fan-out batches"""
    import inspect
    import test_gpu_events_api as api
    names = [n for n in dir(api) if n.startswith("test_") and callable(getattr(api, n)) and "fan_out" not in n
             and not inspect.signature(getattr(api, n)).parameters]
    assert names
    orig = ev.EventBus.__init__

    def flagged(self, *a, **k):
        if k.get("devices") is None:
            k["sparse_drains"] = True
        orig(self, *a, **k)
    ev.EventBus.__init__ = flagged
    try:
        for n in names:
            getattr(api, n)()
    finally:
        ev.EventBus.__init__ = orig
