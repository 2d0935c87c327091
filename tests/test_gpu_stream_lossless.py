"""Lossless mode on the multi-GPU stream (cpbus_stream_admit / cpbus_stream_fanout_prefix, LocalShardedBus(lossless=True)):
a stalled publish stops at the same event on every shard — the shortest prefix any shard can take — exactly where the Go
bus (events/subscriber.go:30-32) and one single-GPU lossless bus stop, and resumes from there.  Shards on whatever GPUs
this box has (all on one GPU when there is only one)."""
import numpy as np
import pytest

import oracle_binding as ob
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from containerpilot_b200.sharding import LocalShardedBus

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["1", "0"], ids=["pdl", "no-pdl"])
def _pdl(request, monkeypatch):
    """every test runs with and without programmatic dependent launch of consecutive fan-outs"""
    monkeypatch.setenv("CPBUS_PDL", request.param)


def _devices(g):
    import torch
    nd = torch.cuda.device_count()
    return [i % nd for i in range(g)]


def _counts(sb):
    return [int(c) for first, count, bus in sb.shards if count for c in bus.digests(first, count)["count"]]


@pytest.mark.parametrize("G", [1, 2, 3, 4])
@pytest.mark.parametrize("seed", [1, 2])
def test_stream_blocks_per_event_like_the_go_bus(G, seed):
    """The sharded twin of test_gpu_lossless.py::test_flush_blocks_per_event_like_the_go_bus: one global oracle that
    refuses event by event (mailbox_cap), random partial drains through the owning shard.  At every stall every
    subscriber on every shard holds exactly what the oracle holds, and drained records are byte-equal."""
    R, B, N = 128, 64, 14
    rng = np.random.default_rng(100 * G + seed)
    masks = [nat.MASK_ALL, 1 << 2, (1 << 3) | (1 << 2), nat.MASK_ALL, 1 << 5, 0, nat.MASK_ALL]
    masks = np.array((masks * 2)[:N], dtype=np.uint32)
    orc = ob.Oracle(N, keep_window=0, mailbox_cap=R)
    for m_ in masks:
        orc.subscribe(int(m_))
    sb = LocalShardedBus(N, _devices(G), ring_cap=R, batch_cap=B, stream_slots=4, lossless=True)
    try:
        sb.subscribe_many(masks)
        n_partial = 0
        for step in range(40):
            now = (step + 1) * 1000
            ev = np.zeros(B, dtype=EVENT_DTYPE)
            ev["code"] = rng.integers(1, 7, B); ev["source_id"] = step * B + np.arange(B)
            nat.check(sb.put(ev, now), "put")
            assert orc.advance(now) == 0
            i = 0
            while True:
                rc = sb.fanout(B, now)
                while i < B:                                          # the oracle publishes event by event until it blocks
                    r = orc.publish(int(ev["code"][i]), int(ev["source_id"][i]))
                    if r == ob.EAGAIN:
                        break
                    assert r == 0
                    i += 1
                assert _counts(sb) == [orc.count(s) for s in range(N)], (step, i, rc)
                if rc == nat.OK:
                    assert i == B
                    break
                assert rc == nat.EAGAIN and i < B
                n_partial += 1 if i > 0 else 0
                for s in rng.permutation(N)[:4]:                      # some consumers run (not necessarily the full one)
                    take = int(rng.integers(1, R + 1))
                    g = sb.drain(int(s), cap=take)
                    assert g.tobytes() == orc.consume(int(s), take).tobytes()
        for s in range(N):
            assert sb.drain(s, cap=R).tobytes() == orc.consume(s, R).tobytes()
        assert n_partial > 0
        for _, _, bus in sb.shards:
            st = bus.stats()
            assert st["overwritten"] == 0 and st["admit_partial"] > 0
    finally:
        sb.close()


def test_one_full_mailbox_holds_back_every_shard():
    """Only the last shard has a full mailbox.  The other shards' mailboxes have room for the whole batch, yet they must
    hold exactly the global prefix — not their own longer one."""
    R, B, N = 64, 32, 8
    orc = ob.Oracle(N, keep_window=0, mailbox_cap=R)
    for _ in range(N):
        orc.subscribe()
    sb = LocalShardedBus(N, _devices(2), ring_cap=R, batch_cap=B, stream_slots=4, lossless=True)
    full = N - 1                                                      # on shard 1; never drained until the stall
    try:
        sb.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
        rng = np.random.default_rng(3)
        batches = []
        for step in range(3):
            ev = np.zeros(B, dtype=EVENT_DTYPE)
            ev["code"] = rng.integers(1, 17, B); ev["source_id"] = step * B + np.arange(B)
            batches.append(ev)
        for step, ev in enumerate(batches[:2]):                      # 64 records: mailbox `full` is at capacity
            nat.check(sb.put(ev, 1000 * (step + 1)), "put"); orc.advance(1000 * (step + 1))
            assert sb.fanout(B, 1000 * (step + 1)) == nat.OK
            orc.publish_many(ev["code"], ev["source_id"])
            for s in range(N - 1):
                assert sb.drain(s).tobytes() == orc.consume(s, R).tobytes()
        ev = batches[2]
        nat.check(sb.put(ev, 3000), "put"); orc.advance(3000)
        assert sb.fanout(B, 3000) == nat.EAGAIN                       # nothing fits in `full`: nothing goes anywhere
        assert _counts(sb) == [2 * B] * N
        assert sb.drain(full, cap=10).tobytes() == orc.consume(full, 10).tobytes()
        assert sb.fanout(B, 3000) == nat.EAGAIN                       # 10 records of the batch, on every shard
        assert _counts(sb) == [2 * B + 10] * N
        for i in range(10):
            assert orc.publish(int(ev["code"][i]), int(ev["source_id"][i])) == 0
        assert orc.publish(int(ev["code"][10]), int(ev["source_id"][10])) == ob.EAGAIN
        for s in range(N - 1):                                        # shard 0 holds the global prefix, byte for byte
            assert sb.drain(s).tobytes() == orc.consume(s, R).tobytes()
        assert len(sb.drain(full)) == R
        orc.consume(full, R)
        assert sb.fanout(B, 3000) == nat.OK
        for i in range(10, B):
            assert orc.publish(int(ev["code"][i]), int(ev["source_id"][i])) == 0
        for s in range(N):
            assert sb.drain(s).tobytes() == orc.consume(s, R).tobytes()
    finally:
        sb.close()


def _raw_batches(seed, n_batches, B, N, dt):
    """RAW stream records stamped the way cpbus_publish / cpbus_send stamp them (running seq, ts = now, target, flags),
    with unicast records to global ids on every shard; ragged and empty batches."""
    rng = np.random.default_rng(seed)
    out, seq = [], 0
    for q in range(n_batches):
        r = rng.random()
        n = 0 if r < 0.15 else int(rng.integers(1, B + 1)) if r < 0.45 else B
        ev = np.zeros(n, dtype=EVENT_DTYPE)
        ev["seq"] = seq + np.arange(n); seq += n
        ev["ts_ns"] = (q + 1) * dt
        ev["code"] = rng.integers(0, 17, n); ev["source_id"] = rng.integers(0, 64, n)
        ev["target"] = nat.TARGET_ALL
        uni = rng.random(n) < 0.25
        ev["target"][uni] = rng.integers(0, N, int(uni.sum()))
        ev["flags"][uni] = nat.F_UNICAST
        out.append(ev)
    return out


def _publish_single(bus, ev, now):
    """the same records through the single-GPU host path: advance, then publish / send in record order"""
    nat.check(bus.advance(now), "advance")
    i = 0
    while i < len(ev):
        if ev["target"][i] != nat.TARGET_ALL:
            nat.check(bus.send(int(ev["target"][i]), int(ev["code"][i]), int(ev["source_id"][i])), "send")
            i += 1
            continue
        j = i
        while j < len(ev) and ev["target"][j] == nat.TARGET_ALL:
            j += 1
        nat.check(bus.publish_many(ev[i:j]), "publish")
        i = j


@pytest.mark.parametrize("G,K", [(2, 1), (3, 2), (4, 1)])
def test_timers_and_unicast_match_one_lossless_bus(G, K):
    """Differential against one single-GPU lossless Bus (pinned to the oracle by test_gpu_lossless.py): timers, unicast
    records to several shards, ragged and empty batches, the same drain schedule on both sides.  Counts at every stall,
    drained bytes and the final (count, digest) of every subscriber are identical."""
    R, B, N, dt = 64, 32, 23, 40_000
    periods = [90_000, 130_000][:K]
    rng = np.random.default_rng(7 * G + K)
    masks = np.where(rng.random(N) < 0.5, nat.MASK_ALL, rng.integers(0, 1 << 17, N)).astype(np.uint32)
    masks[3] = 0
    batches = _raw_batches(11 * G + K, 40, B, N, dt)
    sb = LocalShardedBus(N, _devices(G), ring_cap=R, batch_cap=B, timers_per_sub=K, stream_slots=4, lossless=True)
    one = Bus(N, ring_cap=R, batch_cap=B, timers_per_sub=K, lossless=True)
    try:
        sb.subscribe_many(masks); one.subscribe_many(masks)
        sb.timer_add_many(periods[0], source_id0=1000)                # slot 0 in bulk, a second slot one by one
        one.timer_add_many(0, N, periods[0], source_id0=1000)
        for p in periods[1:]:
            for s in range(N):
                sb.bus_of(s).timer_add(s, p, 2000 + s); one.timer_add(s, p, 2000 + s)
        n_stalls = 0
        for q, ev in enumerate(batches):
            now = (q + 1) * dt
            nat.check(sb.put(ev, now, raw=True), "put")
            _publish_single(one, ev, now)
            while True:
                rc_s, rc_1 = sb.fanout(len(ev), now), one.flush()
                assert rc_s == rc_1, (q, rc_s, rc_1)
                single = [int(c) for c in one.digests(0, N)["count"]]
                assert _counts(sb) == single, q
                if rc_s == nat.OK:
                    break
                assert rc_s == nat.EAGAIN
                n_stalls += 1
                for s in rng.permutation(N)[:6]:
                    take = int(rng.integers(1, R + 1))
                    assert sb.drain(int(s), cap=take).tobytes() == one.drain(int(s), cap=take).tobytes()
            if q % 5 == 4:                                            # one consumer sometimes keeps up
                s = int(rng.integers(0, N))
                assert sb.drain(s).tobytes() == one.drain(s).tobytes()
        assert n_stalls > 0
        for s in range(N):
            assert sb.drain(s).tobytes() == one.drain(s).tobytes()
        want = one.digests(0, N)
        got = sb.digests()
        assert (got["count"] == want["count"]).all() and (got["digest"] == want["digest"]).all()
        assert int(want["count"].sum()) > 0
    finally:
        sb.close()
        one.close()


def test_consumers_that_keep_up_stay_on_the_fast_path():
    """consume_all every step: no shard ever runs the admission pass (no kernel, no sync), and the result is the oracle's."""
    N, B, G, steps = 4096, 256, 2, 30
    rng = np.random.default_rng(9)
    masks = np.where(rng.random(N) < 0.5, nat.MASK_ALL, rng.integers(0, 1 << 17, N)).astype(np.uint32)
    orc = ob.Oracle(N, timers_per_sub=1, keep_window=8)
    for s, m in enumerate(masks):
        orc.subscribe(int(m))
    for s in range(N):
        orc.timer_add(s, 50_000, 100 + s, False)
    sb = LocalShardedBus(N, _devices(G), ring_cap=1024, batch_cap=B, timers_per_sub=1, stream_slots=8, lossless=True)
    try:
        sb.subscribe_many(masks)
        sb.timer_add_many(50_000, source_id0=100)
        for step in range(steps):
            now = (step + 1) * 100_000
            ev = np.zeros(B, dtype=EVENT_DTYPE)
            ev["code"] = rng.integers(0, 17, B); ev["source_id"] = rng.integers(0, 50, B)
            assert sb.publish(ev, now) == nat.OK
            sb.consume_all()
            orc.advance(now); orc.publish_many(ev["code"], ev["source_id"])
        sb.sync()
        got = sb.digests()
        assert (got["count"] == np.array([orc.count(s) for s in range(N)], dtype=np.uint64)).all()
        assert (got["digest"] == np.array([orc.digest(s) for s in range(N)], dtype=np.uint64)).all()
        for _, _, bus in sb.shards:
            st = bus.stats()
            assert st["admit_passes"] == 0 and st["admit_skipped"] == steps and st["admit_partial"] == 0
    finally:
        sb.close()


def test_ticks_after_the_last_record_wait_for_room():
    """RAW records older than the batch's now_ns: a tick due between the last record and now_ns follows the records.
    When every record fits but that tick does not, the last record is held back (the batch cannot complete); an empty
    batch whose tick does not fit is a stall (EAGAIN) with nothing launched."""
    R, B, P = 64, 32, 100_000
    with Bus(1, ring_cap=R, batch_cap=B, timers_per_sub=1, lossless=True) as bus:
        bus.subscribe()
        bus.timer_add(0, P, 77)                                        # due at 100,000, 200,000, ...
        st, _ = bus.stream_create(4, 1)

        def raw(q, ts):
            ev = np.zeros(B, dtype=EVENT_DTYPE)
            ev["seq"] = q * B + np.arange(B); ev["ts_ns"] = ts; ev["code"] = 1 + q; ev["target"] = nat.TARGET_ALL
            return ev
        nat.check(bus.stream_put(st, raw(0, 10), 10, raw=True), "put")
        assert bus.stream_admit(st, B, 10) == B
        assert bus.stream_fanout_prefix(st, B, 10, B) == nat.OK
        nat.check(bus.stream_put(st, raw(1, 20), 150_000, raw=True), "put")   # 32 records + the tick due at 100,000
        assert bus.stream_admit(st, B, 150_000) == B - 1                 # room for 32 records, not for the tick behind them
        assert bus.stream_fanout_prefix(st, B, 150_000, B - 1) == nat.EAGAIN
        assert int(bus.digests(0, 1)["count"][0]) == 2 * B - 1 and bus.stats()["ticks"] == 0
        assert bus.drain(0, cap=1)["code"].tolist() == [1]
        assert bus.stream_admit(st, B, 150_000) == 1
        assert bus.stream_fanout_prefix(st, B, 150_000, 1) == nat.OK
        nat.check(bus.stream_put(st, np.zeros(0, dtype=EVENT_DTYPE), 250_000, raw=True), "put")   # only the tick at 200,000
        with pytest.raises(nat.CpbusError) as ei:
            bus.stream_admit(st, 0, 250_000)
        assert ei.value.status == nat.EAGAIN
        got = bus.drain(0, cap=1)
        assert bus.stream_admit(st, 0, 250_000) == 0
        assert bus.stream_fanout_prefix(st, 0, 250_000, 0) == nat.OK
        got = np.concatenate([got, bus.drain(0)])
        tail = got[-3:]
        assert tail["code"].tolist() == [2, 8, 8] and tail["ts_ns"].tolist() == [20, 100_000, 200_000]
        assert tail["flags"].tolist() == [0, nat.F_TICK, nat.F_TICK]
        assert bus.stats()["ticks"] == 2 and bus.stats()["overwritten"] == 0
        bus.stream_close(st)


def test_errors():
    """m beyond the remainder: EINVAL.  Plain cpbus_stream_fanout on a lossless bus: EINVAL.  The publisher cannot reuse a
    slot whose batch is only partly delivered (EAGAIN).  A throughput-mode bus admits the whole remainder."""
    R, B = 64, 32
    with Bus(1, ring_cap=R, batch_cap=B, lossless=True) as bus:
        bus.subscribe()
        st, _ = bus.stream_create(4, 1)
        batches = [np.zeros(B, dtype=EVENT_DTYPE) for _ in range(8)]
        for q, ev in enumerate(batches):
            ev["code"] = 1 + q
        for q in range(4):
            nat.check(bus.stream_put(st, batches[q], 1000 * (q + 1), nowait=True), "put")
        assert bus.stream_fanout(st, B, 1000) == nat.EINVAL             # lossless: admission is the caller's job
        assert bus.stream_fanout_prefix(st, B, 1000, B + 1) == nat.EINVAL
        for q in range(2):                                             # two whole batches: the mailbox is full
            assert bus.stream_admit(st, B, 1000 * (q + 1)) == B
            assert bus.stream_fanout_prefix(st, B, 1000 * (q + 1), B) == nat.OK
        assert bus.stream_admit(st, B, 3000) == 0
        assert bus.stream_fanout_prefix(st, B, 3000, 0) == nat.EAGAIN   # no launch
        assert len(bus.drain(0, cap=5)) == 5
        assert bus.stream_admit(st, B, 3000) == 5
        assert bus.stream_fanout_prefix(st, B, 3000, 5) == nat.EAGAIN   # batch 3: 5 of 32 delivered
        assert bus.stream_fanout_prefix(st, B, 3000, B - 4) == nat.EINVAL
        bus.sync()
        nat.check(bus.stream_put(st, batches[4], 5000, nowait=True), "put")   # slots of batches 1 and 2: acknowledged
        nat.check(bus.stream_put(st, batches[5], 6000, nowait=True), "put")
        assert bus.stream_put(st, batches[6], 7000, nowait=True) == nat.EAGAIN   # slot of batch 3: only partly delivered
        got = [bus.drain(0)]
        assert bus.stream_admit(st, B, 3000) == B - 5
        assert bus.stream_fanout_prefix(st, B, 3000, B - 5) == nat.OK
        bus.sync()
        nat.check(bus.stream_put(st, batches[6], 7000, nowait=True), "put")
        got.append(bus.drain(0))
        seen = np.concatenate(got)
        assert list(seen["code"]) == [1] * (B - 5) + [2] * B + [3] * B    # FIFO across the stall, nothing lost or repeated
        assert bus.stats()["admit_partial"] == 1
        bus.stream_close(st)
    with Bus(4, ring_cap=R, batch_cap=B) as bus:                         # throughput mode: the whole remainder, no kernel
        bus.subscribe_many(np.full(4, nat.MASK_ALL, dtype=np.uint32))
        st, _ = bus.stream_create(4, 1)
        nat.check(bus.stream_put(st, batches[0], 1000), "put")
        launches = bus.stats()["kernel_launches"]
        assert bus.stream_admit(st, B, 1000) == B
        assert bus.stats()["kernel_launches"] == launches
        nat.check(bus.stream_fanout(st, B, 1000), "fanout")
        bus.stream_close(st)
