"""The group (`cpbus_group_*`, `GroupBus`): one bus handle over G shards gives the results of one bus with the same
configuration — return codes, ids, drains, sparse drains, windows, digests, folds, debug events, publish counts and the
stats that are not launch-shaped — in throughput and lossless mode, and the oracle's mailboxes."""
import json
import os
import subprocess
from collections import Counter

import numpy as np
import pytest

import oracle_binding as ob
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus
from containerpilot_b200 import events
from containerpilot_b200.events import Event
from containerpilot_b200.group import GroupBus

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_vectors.json")))
LAUNCH_SHAPED = ("batches", "kernel_launches", "admit_passes", "admit_skipped", "admit_partial", "device_splits")


def _n_gpus():
    import torch
    return torch.cuda.device_count()


def _trace(seed, n_subs0, n_ops, K, jump_every=0, period=(2000, 40000)):
    """random_ops with pairs and unicast, plus set_mask ops and, every `jump_every` ops, a clock jump of hundreds of the
    shortest timer period"""
    ops, n_total = tr.random_ops(seed, n_subs0, n_ops, timers_per_sub=K, p_send=0.05, p_timer=0.04, p_member=0.02,
                                 p_pairs=0.3, p_flush=0.03, period_min=period[0], period_max=period[1])
    rng = np.random.default_rng(seed ^ 0x5EED)
    out, shift = [], 0
    for i, op in enumerate(ops):
        if op[0] == "adv":
            if jump_every and i % jump_every == 0:
                shift += int(rng.integers(200, 600)) * period[0]
            op = ("adv", op[1] + shift)
        out.append(op)
        if rng.random() < 0.01:
            out.append(("setmask", int(rng.integers(0, n_total)), int(rng.integers(0, 1 << 17))))
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


def _apply(bus, op, handles):
    k = op[0]
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
    elif isinstance(a, tuple):
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
    st = bus.stats()
    res.append({k: v for k, v in st.items() if k not in LAUNCH_SHAPED})
    res.append(_call(bus.drain_ready, 0, n_total, n_total // 2, bus.ring_cap, 3))
    return res


def _twin(seed, devices, lossless, K=4, R=64, B=32, n_subs0=24, n_ops=1500, jump_every=150, p_consume=0.08):
    ops, n_total = _trace(seed, n_subs0, n_ops, K, jump_every=jump_every)
    rng = np.random.default_rng(seed + 77)
    kw = dict(ring_cap=R, batch_cap=B, timers_per_sub=K, lossless=lossless)
    one = Bus(n_total + 4, device=devices[0], **kw)
    grp = GroupBus(n_total + 4, devices, **kw)
    ha, hb = [], []
    n_eagain = n_ids = 0
    try:
        for i, op in enumerate(ops):
            a, b = _apply(one, op, ha), _apply(grp, op, hb)
            _eq(a, b, f"op {i} {op}: {a} vs {b}")
            n_eagain += a[0] == nat.EAGAIN
            n_ids += op[0] == "sub" and a[0] == nat.OK
            if n_ids and (a[0] == nat.EAGAIN or rng.random() < p_consume):
                for _ in range(int(rng.integers(1, 4))):
                    c = _consumers(rng, n_ids, R)
                    _eq(_consume(one, c), _consume(grp, c), f"op {i} consumer {c}")
        fa, fb = _final(one, n_ids), _final(grp, n_ids)
        for j, (x, y) in enumerate(zip(fa, fb)):
            _eq(x, y, f"final item {j}")
    finally:
        one.close(); grp.close()
    return n_eagain


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("G", [1, 2, 3, 4])
def test_group_equals_one_bus(G, lossless):
    n_eagain = _twin(10 * G + lossless, [0] * G, lossless)
    if lossless:
        assert n_eagain > 0


def test_group_equals_one_bus_empty_shards():
    """capacity for far more subscribers than the trace makes: the last shards stay empty"""
    ops, n_total = _trace(5, 6, 600, 2, jump_every=100)
    kw = dict(ring_cap=64, batch_cap=32, timers_per_sub=2)
    one, grp = Bus(400, device=0, **kw), GroupBus(400, [0, 0, 0, 0], **kw)
    ha, hb = [], []
    try:
        for i, op in enumerate(ops):
            _eq(_apply(one, op, ha), _apply(grp, op, hb), f"op {i} {op}")
        for x, y in zip(_final(one, n_total), _final(grp, n_total)):
            _eq(x, y, "final")
    finally:
        one.close(); grp.close()


@pytest.mark.parametrize("lossless", [False, True])
def test_group_on_distinct_gpus(lossless):
    G = min(_n_gpus(), 4)
    if G < 2:
        pytest.skip("one GPU")
    _twin(99 + lossless, list(range(G)), lossless)


@pytest.mark.parametrize("env", [("CPBUS_PDL", "0"), ("CPBUS_HINTS", "2")])
def test_group_equals_one_bus_knobs(env, monkeypatch):
    monkeypatch.setenv(*env)
    _twin(7, [0, 0, 0], True, n_ops=800)


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("G", [2, 3])
def test_group_against_oracle(G, lossless):
    ops, n_total = tr.random_ops(40 + G, 20, 700 if lossless else 1500, timers_per_sub=2, p_pairs=0.3, p_send=0.05,
                                 period_min=20000)            # lossless: no mailbox of the oracle ever fills
    R = 1024
    orc = tr.run_oracle(ops, n_total + 4, timers_per_sub=2, keep_window=R, mailbox_cap=R if lossless else 0)
    with GroupBus(n_total + 4, [0] * G, ring_cap=R, batch_cap=256, timers_per_sub=2, lossless=lossless) as grp:
        tr.run_bus(grp, ops)
        tr.compare(grp, orc, n_total, window=R)


def test_unicast_to_shard_two_between_broadcasts():
    kw = dict(ring_cap=64, batch_cap=32)
    one, grp = Bus(9, device=0, **kw), GroupBus(9, [0, 0, 0], **kw)
    try:
        for bus in (one, grp):
            bus.subscribe_many(np.full(9, nat.MASK_ALL, dtype=np.uint32))
            for i in range(5):
                nat.check(bus.publish(1, i), "publish")
                nat.check(bus.send(7, 2, 100 + i), "send")          # id 7 lives on shard 2
            nat.check(bus.flush(), "flush")
        _eq(one.digests(0, 9), grp.digests(0, 9), "digests")
        _eq(one.drain(7), grp.drain(7), "drain")
    finally:
        one.close(); grp.close()


@pytest.mark.parametrize("lossless", [False, True])
def test_idle_step_of_a_thousand_periods(lossless):
    """K = 4, a 1 s heartbeat: a stream batch may step 8 s at most, so a 1,000 s idle step has to be cut on the single
    bus's grid; then a timer armed on a shard that had none fires at now + period."""
    period, N, R = 1_000_000_000, 12, 4096
    orc = ob.Oracle(N, timers_per_sub=4, keep_window=R)
    with GroupBus(N, [0, 0, 0], ring_cap=R, batch_cap=256, timers_per_sub=4, lossless=lossless) as grp:
        grp.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
        for s in range(N):
            orc.subscribe(nat.MASK_ALL)
        grp.timer_add(0, period, 5)                                # shard 0 only
        orc.timer_add(0, period, 5, False)
        nat.check(grp.advance(1000 * period), "advance")
        assert orc.advance(1000 * period) == 0
        tid = grp.timer_add(10, period // 2, 6, True)              # shard 2 had no timer
        orc.timer_add(10, period // 2, 6, True)
        assert tid >> 26 == 1
        nat.check(grp.advance(1002 * period), "advance")
        assert orc.advance(1002 * period) == 0
        nat.check(grp.flush(), "flush")
        st = tr.compare(grp, orc, N, window=R)
        assert st["ticks"] == 1003 and grp.stats()["now_ns"] == 1002 * period


@pytest.mark.parametrize("vec", GOLDEN["multiset"], ids=lambda v: v["name"])
def test_events_bus_on_a_group_multiset_vectors(vec):
    answers = []
    for devices in (None, [0, 0]):
        bus = events.EventBus(devices=devices)
        sub = events.Subscriber(events.Chan(1000)); sub.Subscribe(bus)
        for code, src in vec.get("direct_receives", []):
            sub.Receive(Event(code, src))
        for code, src in vec["published"]:
            bus.Publish(Event(code, src))
        got = Counter(f"{e.Code}|{e.Source}" for e in bus.DebugEvents())
        assert dict(got) == vec["debug_events"]
        answers.append(sub.Received())
        bus.close()
    assert answers[0] == answers[1]


def _job_scenario(devices):
    """a job with exact cases and a heartbeat, a watcher on another shard, and a mailbox that fills until Publish blocks"""
    bus = events.EventBus(n_max_subs=6, ring_cap=64, batch_cap=32, devices=devices)
    subs = [events.Subscriber(events.Chan(1000)) for _ in range(5)]
    for s in subs[:4]:
        s.Subscribe(bus)
    job = subs[4]
    bus.Subscribe(job, mask=1 << events.Startup, cases=[Event(events.StatusHealthy, "db"), Event(events.Stopped, "db")])
    ctx, cancel = events.WithCancel()
    events.NewEventTimer(ctx, job.Rx, 1_000_000_000, "job.heartbeat")
    out = []
    bus.Publish(events.GlobalStartup)
    bus.Advance(3_500_000_000)
    n = 0
    try:
        for i in range(200):                      # nobody drains subs[0..3]: their mailboxes fill up
            bus.Publish(Event(events.StatusHealthy, "db" if i % 3 == 0 else "web"))
            n += 1
    except BlockingIOError:
        pass
    out.append(n)
    # the consumers run: every mailbox is emptied straight from the bus (Received would flush first, and the flush is the
    # very thing that is blocked), then the blocked publish completes
    out.append([bus._bus.drain(s._id).tobytes() for s in subs])
    out.append(job.Received())
    bus.Publish(Event(events.Stopped, "db"))
    cancel()
    bus.Advance(9_000_000_000)
    out.append(job.Received())
    out.append(bus.DebugEvents())
    bus.close()
    return out


def test_events_bus_on_a_group_job_scenario():
    one, grp = _job_scenario(None), _job_scenario([0, 0])
    assert one[0] < 200                               # the full mailbox blocked the publisher
    assert one == grp


def test_cpp_mirror_on_a_group():
    exe = os.path.join(ROOT, "containerpilot_b200", "csrc", "host", "events_group_test")
    assert os.path.exists(exe), "built by the host Makefile"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
