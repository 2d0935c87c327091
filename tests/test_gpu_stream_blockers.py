"""Consumer backlog on the sharded stream: `cpbus_stream_blockers` (which mailboxes a stalled lossless stream round waits
on, per shard) and the fleet-wide `LocalShardedBus.blockers` / `.lagging`.  All shards live on however many GPUs the box
has (all on one if need be).  Checked against the stream's own admission, the oracle (tests/lag_oracle.py), a twin that
never asks, and one bus holding the same mailboxes."""
import numpy as np
import pytest

import lag_oracle as lo
import oracle_binding as ob
from containerpilot_b200 import _native as nat
from containerpilot_b200 import sharding
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from containerpilot_b200.sharding import LocalShardedBus

pytestmark = pytest.mark.gpu
R, B, DT, PERIOD = 64, 32, 40_000, 90_000


def _devices(g):
    import torch
    nd = torch.cuda.device_count()
    return [i % nd for i in range(g)]


def _trace(seed, n_batches, N):
    """RAW batches stamped like cpbus_publish / cpbus_send (running seq), ragged, empty and full; record times spread over
    the batch's window; a quarter unicast to any shard's subscribers; codes that hit the exact {code, source} cases"""
    rng = np.random.default_rng(seed)
    out, seq = [], 0
    for q in range(n_batches):
        w = (q + 1) * DT
        r = rng.random()
        n = 0 if r < 0.12 else (int(rng.integers(1, 4)) if r < 0.3 else (int(rng.integers(1, B + 1)) if r < 0.55 else B))
        ev = np.zeros(n, dtype=EVENT_DTYPE)
        ev["seq"] = seq + np.arange(n); seq += n
        ev["ts_ns"] = np.sort(rng.integers(w - DT + 1, w + 1, n))
        ev["code"] = rng.integers(0, 6, n); ev["source_id"] = rng.integers(0, 6, n)
        ev["target"] = nat.TARGET_ALL
        uni = rng.random(n) < 0.25
        ev["target"][uni] = rng.integers(0, N, int(uni.sum()))
        ev["flags"][uni] = nat.F_UNICAST
        out.append((ev, w))
    return out


def _populate(sb, orc, N, K, seed):
    """masks over the trace's codes, exact {code, source} cases on every third subscriber, periodic timers on every other
    subscriber (two slots on some when K >= 2) and one-shots on some of the rest"""
    rng = np.random.default_rng(seed)
    masks = np.where(rng.random(N) < 0.3, nat.MASK_ALL, rng.integers(0, 1 << 6, N)).astype(np.uint32)
    pairs = [[(int(rng.integers(0, 6)), int(rng.integers(0, 6))) for _ in range(2)] if s % 3 == 0 else [] for s in range(N)]
    for first, count, bus in sb.shards:
        bus.subscribe_pairs_many(masks[first:first + count], pairs[first:first + count])
    for s in range(N):
        orc.subscribe(int(masks[s]), pairs=pairs[s])
    if not K:
        return
    for s in range(N):
        timers = []
        if s % 2 == 0:
            timers.append((PERIOD + 1000 * (s % 7), False))
            if K >= 2 and s % 4 == 0:
                timers.append((3 * PERIOD, False))
        elif s % 5 == 1:
            timers.append((int(PERIOD * rng.integers(2, 12)), True))
        for period, oneshot in timers:
            sb.bus_of(s).timer_add(s, period, 500 + s, oneshot=oneshot)
            orc.timer_add(s, period, 500 + s, oneshot)


def _unit(ev, off, w):
    """cpbus_stream_admit's next unit of the remainder ev[off:]: (record or None, the time its ticks are due by)"""
    rem = len(ev) - off
    if rem == 0:
        return None, w
    return ev[off], (w if rem == 1 else int(ev["ts_ns"][off]))


def _orc_blockers(orc, rec, t):
    if rec is None:
        return lo.blockers(orc, t).tolist()
    return lo.blockers(orc, t, int(rec["code"]), int(rec["source_id"]), int(rec["target"])).tolist()


def _orc_deliver(orc, ev, lo_, hi):
    for i in range(lo_, hi):
        assert orc.advance(int(ev["ts_ns"][i])) == 0
        code, src, tgt = int(ev["code"][i]), int(ev["source_id"][i]), int(ev["target"][i])
        assert (orc.publish(code, src) if tgt == nat.TARGET_ALL else orc.receive(tgt, code, src)) == 0


def _counts(sb):
    return [int(c) for first, count, bus in sb.shards for c in bus.digests(first, count)["count"]]


@pytest.mark.parametrize("G,K", [(2, 0), (2, 1), (2, 4), (4, 0), (4, 1), (4, 4)])
def test_blockers_are_the_shards_that_admit_nothing(G, K):
    """Host-driven rounds: at every round each shard's blockers are non-empty exactly when its admit gives 0 (a stall, or
    p = 0 with records left), equal the oracle's blockers of the shard's next unit within its id range, and after a stall
    draining exactly the blockers (every other stall: a few random consumers) makes every shard admit p >= 1."""
    N = 23
    sb = LocalShardedBus(N, _devices(G), ring_cap=R, batch_cap=B, timers_per_sub=K, stream_slots=64, lossless=True)
    orc = ob.Oracle(N, timers_per_sub=K, keep_window=0, mailbox_cap=R)
    rng = np.random.default_rng(40 * G + K)
    seen = {"stall": 0, "partial": 0, "nonempty": 0, "drained": 0}
    try:
        _populate(sb, orc, N, K, 3 * G + K)
        trace = _trace(900 + 10 * G + K, 40, N)
        for ev, w in trace:
            nat.check(sb.put(ev, w, raw=True), "put")
        for q, (ev, w) in enumerate(trace):
            off, drained_blockers = 0, False
            while True:
                rec, t = _unit(ev, off, w)
                exp = _orc_blockers(orc, rec, t)
                offers = []
                for g, (first, count, bus) in enumerate(sb.shards):
                    blk = bus.stream_blockers(sb._st[g]).tolist()
                    assert blk == [s for s in exp if first <= s < first + count], (q, off, g)
                    p, stalled = sharding._admit_or_stall(bus, sb._st[g], len(ev), w)
                    offers.append((p, stalled))
                    zero = stalled or (p == 0 and off < len(ev))
                    assert zero == (len(blk) > 0), (q, off, g, p, stalled, blk)
                    if drained_blockers:
                        assert not zero, (q, off, g)
                    seen["nonempty"] += len(blk) > 0
                m = None if any(s for _, s in offers) else min(p for p, _ in offers)
                rc = nat.EAGAIN
                if m is not None:
                    for g, (_, _, bus) in enumerate(sb.shards):
                        rc = sharding._fanout_prefix(bus, sb._st[g], len(ev), w, m)
                    _orc_deliver(orc, ev, off, off + m)
                    off += m
                if rc == nat.OK:
                    assert off == len(ev) and orc.advance(w) == 0
                    break
                seen["stall"] += m is None or m == 0
                seen["partial"] += bool(m)
                drained_blockers = bool(m is None or m == 0) and seen["stall"] % 2 == 1
                if drained_blockers:                       # exactly the blockers, and nothing else
                    ids = sb.blockers().tolist()
                    assert ids == exp and ids
                    for s in ids:
                        orc.consume(s, R); sb.drain(s, cap=R)
                    seen["drained"] += 1
                elif m is None or m == 0:
                    for s in rng.permutation(N)[:2]:
                        take = int(rng.integers(1, R + 1))
                        orc.consume(int(s), take); sb.drain(int(s), cap=take)
                assert _counts(sb) == [orc.count(s) for s in range(N)], (q, off)
        assert seen["stall"] > 5 and seen["drained"] > 2 and seen["nonempty"] > 5, seen
    finally:
        sb.close()


@pytest.mark.parametrize("G,K", [(2, 1), (4, 4)])
def test_device_rounds_stall_on_the_blockers(G, K):
    """run_rounds with a pump: after every resolution that shows a new stalled round the fleet's blockers are non-empty;
    draining exactly those mailboxes lets the next queued round move records."""
    N = 23
    sb = LocalShardedBus(N, _devices(G), ring_cap=R, batch_cap=B, timers_per_sub=K, stream_slots=64, lossless=True)
    orc = ob.Oracle(N, timers_per_sub=K, keep_window=0, mailbox_cap=R)
    state = {"stalled": 0, "pos": None, "checks": 0}
    try:
        _populate(sb, orc, N, K, 5 * G + K)
        trace = _trace(1900 + 10 * G + K, 30, N)
        for ev, w in trace:
            nat.check(sb.put(ev, w, raw=True), "put")

        def pump():
            done, off, stalled = sb.progress()
            if state["pos"] is not None:            # the round queued after the drain moved records
                assert (done, off) != state["pos"], state
                state["pos"] = None
                state["checks"] += 1
            if stalled > state["stalled"]:
                ids = sb.blockers()
                assert len(ids) > 0, (done, off, stalled)
                for s in ids.tolist():
                    sb.drain(s, cap=R)
                state["stalled"], state["pos"] = stalled, (done, off)

        sb.run_rounds(len(trace), pump=pump, depth=3)
        assert sb.progress()[0] == len(trace) and state["checks"] > 3, state
    finally:
        sb.close()


def test_asking_changes_nothing():
    """Twins run the same device rounds and the same consumers; one asks stream_blockers on every shard (and the fleet's
    blockers and lagging) between rounds.  Both end with identical mailboxes, digests, progress and statistics
    (kernel_launches aside)."""
    N, G, K = 23, 3, 1
    kw = dict(ring_cap=R, batch_cap=B, timers_per_sub=K, stream_slots=64, lossless=True)
    a, b = LocalShardedBus(N, _devices(G), **kw), LocalShardedBus(N, _devices(G), **kw)
    try:
        for sb in (a, b):
            _populate(sb, ob.Oracle(N, timers_per_sub=K, keep_window=0, mailbox_cap=R), N, K, 17)
        trace = _trace(4242, 25, N)
        for sb in (a, b):
            for ev, w in trace:
                nat.check(sb.put(ev, w, raw=True), "put")
        rng = np.random.default_rng(8)
        asked = 0
        while b.progress()[0] < len(trace):
            for sb in (a, b):
                for g in range(G):
                    sb.follow_rounds(g, 1)
            for g, (_, _, bus) in enumerate(a.shards):
                asked += len(bus.stream_blockers(a._st[g]))
            a.blockers(); a.lagging(0, N, start_sub=int(rng.integers(0, N)))
            pa, pb = a.progress(), b.progress()
            assert pa == pb
            for s in rng.permutation(N)[:3]:
                take = int(rng.integers(1, R + 1))
                assert a.drain(int(s), cap=take).tobytes() == b.drain(int(s), cap=take).tobytes()
        assert asked > 0 and a.progress()[2] > 0
        for s in range(N):
            assert a.drain(s).tobytes() == b.drain(s).tobytes()
        assert a.digests().tobytes() == b.digests().tobytes()
        for (_, _, x), (_, _, y) in zip(a.shards, b.shards):
            sx, sy = x.stats(), y.stats()
            sx.pop("kernel_launches"); sy.pop("kernel_launches")
            assert sx == sy
    finally:
        a.close(); b.close()


def _edge_bus(G=2, lossless=True):
    """N = 4 subscribers taking everything, a timer of period 1000 on subscriber 1 (shard 0) only"""
    sb = LocalShardedBus(4, _devices(G), ring_cap=R, batch_cap=B, timers_per_sub=1, stream_slots=8, lossless=lossless)
    sb.subscribe_many(np.full(4, nat.MASK_ALL, dtype=np.uint32))
    sb.bus_of(1).timer_add(1, 1000, 77)
    return sb


def _batch(n, ts):
    ev = np.zeros(n, dtype=EVENT_DTYPE)
    ev["seq"] = np.arange(n); ev["ts_ns"] = ts; ev["code"] = 1; ev["target"] = nat.TARGET_ALL
    return ev


def _fill(sb, n, w):
    """n records to everyone, in complete batches at watermark w"""
    while n:
        k = min(B, n)
        nat.check(sb.put(_batch(k, w), w, raw=True), "put")
        assert sb.fanout(k, w) == nat.OK
        n -= k


def _launches(sb):
    return [bus.stats()["kernel_launches"] for _, _, bus in sb.shards]


def _stream_blockers(sb):
    return [bus.stream_blockers(sb._st[g]).tolist() for g, (_, _, bus) in enumerate(sb.shards)]


def test_unreleased_batch_has_no_blockers():
    sb = _edge_bus()
    try:
        _fill(sb, R, 500)                                   # every mailbox full, the clock at 500
        k0 = _launches(sb)
        assert _stream_blockers(sb) == [[], []] and len(sb.blockers()) == 0
        assert _launches(sb) == k0                          # nothing released: the shards wait for the publisher
    finally:
        sb.close()


def test_single_record_held_back_by_its_trailing_ticks():
    """r = 1: the record fits everywhere by its own time (600, no tick due), but subscriber 1's tick due at 1000 <= the
    watermark 1500 does not fit behind it: admit holds the record back (p = 0) on shard 0, and subscriber 1 is the blocker."""
    sb = _edge_bus()
    try:
        _fill(sb, R - 1, 500)                               # one free slot in every mailbox
        nat.check(sb.put(_batch(1, 600), 1500, raw=True), "put")
        assert _stream_blockers(sb) == [[1], []]
        st = sb._st
        assert [sharding._admit_or_stall(bus, st[g], 1, 1500) for g, (_, _, bus) in enumerate(sb.shards)] == [(0, False), (1, False)]
        assert len(sb.drain(1)) == R - 1
        assert _stream_blockers(sb) == [[], []]
        assert sb.fanout(1, 1500) == nat.OK
    finally:
        sb.close()


def test_empty_remainder_whose_ticks_do_not_fit():
    """r = 0: an empty batch past subscriber 1's due time while its mailbox is full: admit stalls on shard 0 only."""
    sb = _edge_bus()
    try:
        _fill(sb, R, 500)
        nat.check(sb.put(_batch(0, 0), 1500, raw=True), "put")
        assert _stream_blockers(sb) == [[1], []] and sb.blockers().tolist() == [1]
        assert sharding._admit_or_stall(sb.shards[0][2], sb._st[0], 0, 1500) == (0, True)
        assert sharding._admit_or_stall(sb.shards[1][2], sb._st[1], 0, 1500) == (0, False)
        assert sb.fanout(0, 1500) == nat.EAGAIN
        assert len(sb.drain(1, cap=1)) == 1                 # room for the one tick: exactly enough
        assert _stream_blockers(sb) == [[], []]
        assert sb.fanout(0, 1500) == nat.OK
    finally:
        sb.close()


def test_throughput_mode_has_no_blockers_and_launches_nothing():
    sb = _edge_bus(lossless=False)
    try:
        for q in range(3):
            _fill(sb, R, 500 * (q + 1))
        nat.check(sb.put(_batch(B, 5000), 5000, raw=True), "put")
        k0 = _launches(sb)
        assert _stream_blockers(sb) == [[], []] and len(sb.blockers()) == 0
        assert _launches(sb) == k0
    finally:
        sb.close()


def test_room_bound_that_proves_the_fit_launches_nothing():
    """Right after cpbus_consume_all the room bound is the ring: U fits without a kernel.  With full mailboxes the query
    runs its one scan kernel per shard."""
    sb = _edge_bus()
    try:
        sb.consume_all()
        sb.sync()
        nat.check(sb.put(_batch(4, 700), 700, raw=True), "put")
        k0 = _launches(sb)
        assert _stream_blockers(sb) == [[], []]
        assert _launches(sb) == k0
        assert sb.fanout(4, 700) == nat.OK
        _fill(sb, R - 4, 800)                               # full; the bound no longer proves anything
        nat.check(sb.put(_batch(2, 900), 900, raw=True), "put")
        k0 = _launches(sb)
        assert _stream_blockers(sb) == [[0, 1], [2, 3]]
        assert _launches(sb) == [k + 1 for k in k0]
    finally:
        sb.close()


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("G", [2, 3, 4])
def test_lagging_equals_one_bus(G, lossless):
    """The sharded fleet fed through the stream and one bus fed with cpbus_send hold the same mailboxes; lagging over any
    range, start, min_backlog and cap (and paging by next_sub) gives the same entries, next_sub and summary."""
    N = 37
    rng = np.random.default_rng(60 + G + 10 * lossless)
    sb = LocalShardedBus(N, _devices(G), ring_cap=R, batch_cap=B, stream_slots=8, lossless=lossless)
    one = Bus(N, ring_cap=R, batch_cap=B, lossless=lossless, device=0)
    try:
        masks = rng.integers(0, 1 << 6, N).astype(np.uint32)
        sb.subscribe_many(masks); one.subscribe_many(masks)
        hot = rng.permutation(N)[:3]
        for q in range(30):
            w = (q + 1) * 1000
            n = int(rng.integers(1, B + 1))
            ev = _batch(n, w)
            ev["code"] = rng.integers(0, 17, n); ev["source_id"] = rng.integers(0, 9, n)
            ev["target"] = np.where(rng.random(n) < 0.8, hot[rng.integers(0, len(hot), n)], rng.integers(0, N, n))
            ev["flags"] = nat.F_UNICAST
            if lossless:                                       # keep the fleet from stalling: drain what could overflow
                for s in one.lagging(0, N, min_backlog=R - B + 1)[0]["sub_id"].tolist():
                    one.drain(s); sb.drain(s)
            nat.check(sb.put(ev, w, raw=True), "put")
            assert sb.fanout(n, w) == nat.OK
            one.advance(w)
            for e in ev:
                assert one.send(int(e["target"]), int(e["code"]), int(e["source_id"])) == nat.OK
            assert one.flush() == nat.OK
            for s in rng.permutation(N)[:3]:
                take = int(rng.integers(1, R + 1))
                assert len(one.drain(int(s), cap=take)) == len(sb.drain(int(s), cap=take))
        assert sb.digests()["count"].tolist() == one.digests(0, N)["count"].tolist()
        for _ in range(40):
            first = int(rng.integers(0, N))
            n = int(rng.integers(1, N - first + 1))
            args = dict(start_sub=first + int(rng.integers(0, n)), min_backlog=int(rng.integers(0, 6)), cap=int(rng.integers(0, 9)))
            x, y = one.lagging(first, n, **args), sb.lagging(first, n, **args)
            assert x[0].tobytes() == y[0].tobytes() and x[1:] == y[1:], (first, n, args)
        full, _, summ = one.lagging(0, N, start_sub=11, min_backlog=1)
        assert summ["lagging"] > 6 and summ["backlog_max"] > 0 and (summ["lost_total"] > 0) != lossless
        got, cur = [], 11
        while len(got) < summ["lagging"]:
            page, cur, s2 = sb.lagging(0, N, start_sub=cur, min_backlog=1, cap=4)
            assert s2 == summ
            got += page["sub_id"].tolist()
        assert got[:summ["lagging"]] == full["sub_id"].tolist()
    finally:
        sb.close(); one.close()
