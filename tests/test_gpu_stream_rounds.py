"""Lossless stream rounds on the device (cpbus_stream_round_next / cpbus_stream_progress): G = 1-4 shards on however many
GPUs the box has (all on one if need be).  Every round is checked against a twin LocalShardedBus(lossless=True,
agree="device") that runs the same round from the host (admit, offer, agree, fanout_prefix), and the pipelined driver
against the oracle."""
import numpy as np
import pytest

import oracle_binding as ob
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from containerpilot_b200.sharding import LocalShardedBus

pytestmark = pytest.mark.gpu


def _devices(g):
    import torch
    nd = torch.cuda.device_count()
    return [i % nd for i in range(g)]


def _counts(sb):
    return [int(c) for first, count, bus in sb.shards if count for c in bus.digests(first, count)["count"]]


def _trace(seed, n_batches, B, N, dt):
    """ragged, empty and RAW batches (unicast records to any shard's subscribers), Zipf codes"""
    rng = np.random.default_rng(seed)
    out, seq = [], 1 << 40
    for q in range(n_batches):
        w = (q + 1) * dt
        r = rng.random()
        n = 0 if r < 0.12 else (int(rng.integers(1, B + 1)) if r < 0.45 else B)
        ev = np.zeros(n, dtype=EVENT_DTYPE)
        ev["code"] = tr.zipf_codes(n, 1.0, seed + q) if n else []
        ev["source_id"] = rng.integers(0, 8, n)
        raw = bool(rng.random() < 0.35)
        if raw:
            ev["seq"] = seq + np.arange(n); seq += n
            ev["ts_ns"] = np.sort(rng.integers(w - dt + 1, w + 1, n))
            ev["target"] = nat.TARGET_ALL
            uni = rng.random(n) < 0.2
            ev["target"][uni] = rng.integers(0, N, int(uni.sum()))
            ev["flags"][uni] = nat.F_UNICAST
        out.append((ev, w, raw))
    return out


def _populate(sb, N, K, seed, period):
    """Zipf masks, every third subscriber with exact {code, source} cases, periodic timers on every other subscriber and
    one-shots on some of the rest"""
    rng = np.random.default_rng(seed)
    masks = tr.zipf_masks(N, 1.0, seed)
    pairs = [[(1, 3), (2, 5), (int(rng.integers(1, 17)), 1)] if s % 3 == 0 else [] for s in range(N)]
    for first, count, bus in sb.shards:
        if count:
            bus.subscribe_pairs_many(masks[first:first + count], pairs[first:first + count])
    if K:
        for s in range(N):
            bus = sb.bus_of(s)
            if s % 2 == 0:
                bus.timer_add(s, period, 9000 + s)
            elif s % 5 == 1:
                bus.timer_add(s, int(period * (1 + rng.integers(1, 20))), 9500 + s, oneshot=True)


def _queue_round(sb):
    for g in range(sb.world):
        sb.follow_rounds(g, 1)


VARYING = ("kernel_launches",)


def _kl(sb):
    return [(b.stats()["kernel_launches"], b.stats()["admit_passes"], b.stats()["batches"]) for _, _, b in sb.shards]


@pytest.mark.parametrize("pdl", ["0", "1"])
@pytest.mark.parametrize("G,K,hints", [(1, 1, None), (2, 4, None), (3, 1, None), (4, 4, None), (2, 1, "2"), (3, 4, "2")])
def test_rounds_match_the_host_driven_twin(G, K, hints, pdl, monkeypatch):
    """Round by round, the device round and the twin's host-driven round have the same outcome (the same m, or a stall), and
    after each the same mailboxes, drains, step results and positions; at the end the same digests, statistics, debug
    events and publish counts.  Every fifth batch both run explicit rounds, so the rounds bus switches in both directions.
    kernel_launches: a device round launches 4 kernels per shard (decide, exact pass, agree, fan-out) where the twin's round
    launches offer + agree, its admission pass if any and its fan-out if it delivered; nothing else differs."""
    monkeypatch.setenv("CPBUS_PDL", pdl)
    if hints:
        monkeypatch.setenv("CPBUS_HINTS", hints)
    R, B, N, dt, period = 64, 32, 29, 40_000, 90_000
    kw = dict(ring_cap=R, batch_cap=B, timers_per_sub=K, stream_slots=4, lossless=True, agree="device")
    r, t = LocalShardedBus(N, _devices(G), **kw), LocalShardedBus(N, _devices(G), **kw)
    rng = np.random.default_rng(7 * G + K)
    try:
        for sb in (r, t):
            _populate(sb, N, K, 11 + G, period)
        dev_rounds = stalls = 0
        gap = [0] * G                                   # expected kernel_launches(rounds bus) - kernel_launches(twin)
        for q, (ev, w, raw) in enumerate(_trace(100 + 10 * G + K, 40, B, N, dt)):
            nat.check(r.put(ev, w, raw), "put"); nat.check(t.put(ev, w, raw), "put")
            explicit = q % 5 == 4
            while True:
                kt0, kr0 = _kl(t), _kl(r)
                rc_t = t.fanout(len(ev), w)
                if explicit:
                    rc_r = r.fanout(len(ev), w)
                    assert rc_r == rc_t and r.last_round[1] == t.last_round[1], q
                else:
                    _queue_round(r)
                    dev_rounds += 1
                    done, off, _ = r.progress()
                    assert (done, off) == t.progress()[:2], q
                    assert (rc_t == nat.OK) == (done == q + 1), (q, rc_t, done)
                kt1, kr1 = _kl(t), _kl(r)
                for g in range(G):
                    if explicit:
                        assert kr1[g][0] - kr0[g][0] == kt1[g][0] - kt0[g][0]
                    else:
                        twin = kt1[g][0] - kt0[g][0]
                        assert twin == 2 + (kt1[g][1] - kt0[g][1]) + (kt1[g][2] - kt0[g][2]), q
                        assert kr1[g][0] - kr0[g][0] == 4, q
                        gap[g] += 4 - twin
                assert _counts(r) == _counts(t), q
                if rc_t == nat.OK or t.last_round[1][0]:                     # the round delivered: same step results
                    for (_, _, br), (_, _, bt) in zip(r.shards, t.shards):
                        sr, st_ = (tuple(int(x) for x in b.step_result_end(b.step_result_begin()))[:3] for b in (br, bt))
                        assert sr == st_, q
                if rc_t == nat.OK:
                    break
                stalls += 1
                for s in rng.permutation(N)[:6]:
                    take = int(rng.integers(1, R + 1))
                    assert r.drain(int(s), cap=take).tobytes() == t.drain(int(s), cap=take).tobytes()
        assert stalls > 0 and dev_rounds > 30 and r.progress()[2] > 0
        for s in range(N):
            assert r.drain(s).tobytes() == t.drain(s).tobytes()
        assert r.digests().tobytes() == t.digests().tobytes()
        for g, ((_, _, br), (_, _, bt)) in enumerate(zip(r.shards, t.shards)):
            sr, st_ = br.stats(), bt.stats()
            assert {k: v for k, v in sr.items() if k != "kernel_launches"} == {k: v for k, v in st_.items() if k != "kernel_launches"}
            assert sr["kernel_launches"] - st_["kernel_launches"] == gap[g]
            assert br.debug_events().tobytes() == bt.debug_events().tobytes()
            assert br.publish_counts() == bt.publish_counts()
            assert br.stream_status(r._st[g]) == nat.OK
    finally:
        r.close(); t.close()


@pytest.mark.parametrize("G,seed", [(1, 1), (2, 2), (3, 3), (4, 4)])
def test_rounds_block_per_event_like_the_go_bus(G, seed):
    """One global oracle that refuses event by event (mailbox_cap = ring_cap); Zipf masks and pair tables; random partial
    drains at every resolution point.  The rounds are driven by LocalShardedBus.run_rounds, told only how many batches
    there are; the oracle publishes each batch event by event, its consumers draining when it blocks."""
    R, B, N = 128, 64, 14
    rng = np.random.default_rng(900 + 10 * G + seed)
    masks = tr.zipf_masks(N, 1.0, seed)
    pairs = [[(int(rng.integers(1, 7)), int(rng.integers(0, 8))) for _ in range(int(rng.integers(1, 5)))] if s % 3 == 0 else []
             for s in range(N)]
    orc = ob.Oracle(N, keep_window=0, mailbox_cap=R)
    for s in range(N):
        orc.subscribe(int(masks[s]), pairs[s] or None)
    sb = LocalShardedBus(N, _devices(G), ring_cap=R, batch_cap=B, stream_slots=8, lossless=True, agree="device")
    try:
        for first, count, bus in sb.shards:
            bus.subscribe_pairs_many(masks[first:first + count], pairs[first:first + count])
        batches = []
        for step in range(24):
            n = B if step % 4 else int(rng.integers(0, B + 1))
            ev = np.zeros(n, dtype=EVENT_DTYPE)
            ev["code"] = tr.zipf_codes(n, 1.0, seed + step) if n else []
            ev["source_id"] = rng.integers(0, 8, n)
            batches.append(((step + 1) * 1000, ev))
        state = {"q": 0, "i": 0}

        def oracle_catch_up():
            """the oracle publishes until it blocks or is where the bus is; then both compare and some consumers drain"""
            done, off, _ = sb.progress()
            while state["q"] < done or (state["q"] == done and state["i"] < off):
                now, ev = batches[state["q"]]
                if state["i"] == 0:
                    assert orc.advance(now) == 0
                if len(ev):
                    assert orc.publish(int(ev["code"][state["i"]]), int(ev["source_id"][state["i"]])) == 0
                    state["i"] += 1
                if state["i"] == len(ev):
                    state["q"], state["i"] = state["q"] + 1, 0
            assert _counts(sb) == [orc.count(s) for s in range(N)], (done, off)
            for s in rng.permutation(N)[:4]:
                take = int(rng.integers(1, R + 1))
                assert sb.drain(int(s), cap=take).tobytes() == orc.consume(int(s), take).tobytes()

        for now, ev in batches[:6]:
            nat.check(sb.put(ev, now), "put")
        put = 6

        def pump():
            nonlocal put
            while put < len(batches) and sb.put(batches[put][1], batches[put][0]) == nat.OK:
                put += 1
            oracle_catch_up()

        rounds = sb.run_rounds(len(batches), pump=pump, depth=3)
        assert put == len(batches) and rounds > len(batches)
        oracle_catch_up()                                   # the oracle publishes what the last rounds delivered
        for s in range(N):
            assert sb.drain(s, cap=R).tobytes() == orc.consume(s, R).tobytes()
        for _, _, bus in sb.shards:
            st = bus.stats()
            assert st["overwritten"] == 0 and st["admit_partial"] > 0
    finally:
        sb.close()


@pytest.mark.parametrize("pdl", ["0", "1"])
@pytest.mark.parametrize("G,K", [(1, 1), (2, 4), (4, 1)])
def test_pipelined_rounds_and_consume_all_match_the_oracle(G, K, pdl, monkeypatch):
    """"round, consume_all, round, consume_all, ..." queued several deep with no resolution in between, some of the
    rounds queued before the publisher has put their batches; timers at K = 1 or 4.  Every subscriber's (count, digest)
    equals the oracle's, and the room bound the host ends with lets the next round skip the admission pass."""
    monkeypatch.setenv("CPBUS_PDL", pdl)
    N, B, R, dt, period = 97, 64, 256, 40_000, 90_000
    rng = np.random.default_rng(40 + G + K)
    masks = np.where(rng.random(N) < 0.5, nat.MASK_ALL, rng.integers(0, 1 << 17, N)).astype(np.uint32)
    batches = []
    for q in range(24):
        n = int(rng.integers(0, B + 1)) if q % 3 else B
        ev = np.zeros(n, dtype=EVENT_DTYPE); ev["code"] = rng.integers(1, 17, n); ev["source_id"] = rng.integers(0, 9, n)
        batches.append(ev)
    sb = LocalShardedBus(N, _devices(G), ring_cap=R, batch_cap=B, timers_per_sub=K, stream_slots=8, lossless=True,
                         agree="device")
    orc = ob.Oracle(N, timers_per_sub=K, keep_window=0)
    try:
        sb.subscribe_many(masks)
        for s in range(N):
            orc.subscribe(int(masks[s]))
        for k in range(K):
            for s in range(N):
                sb.bus_of(s).timer_add(s, period * (k + 1), 100 * k + s)
                orc.timer_add(s, period * (k + 1), 100 * k + s, False)
        for c in range(0, len(batches), 4):
            first_round_only = c % 8 == 0                     # half the chunks: rounds queued before their batches
            if first_round_only:
                for _ in range(4):
                    _queue_round(sb); sb.consume_all()
            for j in range(c, c + 4):
                nat.check(sb.put(batches[j], (j + 1) * dt), "put")
            if not first_round_only:
                for _ in range(4):
                    _queue_round(sb); sb.consume_all()
            assert sb.progress() == (c + 4, 0, 0)
        for j, ev in enumerate(batches):
            assert orc.advance((j + 1) * dt) == 0
            for code, src in zip(ev["code"], ev["source_id"]):
                assert orc.publish(int(code), int(src)) == 0
        dg = sb.digests()
        assert [int(x) for x in dg["count"]] == [orc.count(s) for s in range(N)]
        assert [int(x) for x in dg["digest"]] == [orc.digest(s) for s in range(N)]
        for _, _, bus in sb.shards:
            st = bus.stats()
            assert st["now_ns"] == len(batches) * dt and st["admit_partial"] == 0
        skipped = [bus.stats()["admit_skipped"] for _, _, bus in sb.shards]
        ev = np.zeros(1, dtype=EVENT_DTYPE); ev["code"] = 1
        nat.check(sb.put(ev, (len(batches) + 1) * dt), "put")
        _queue_round(sb)
        assert sb.progress()[:2] == (len(batches) + 1, 0)
        assert [bus.stats()["admit_skipped"] for _, _, bus in sb.shards] == [x + 1 for x in skipped]
    finally:
        sb.close()


def test_empty_remainder_whose_ticks_do_not_fit_stalls_every_shard():
    """An empty batch whose tick does not fit one shard's full mailbox: the round stalls on every shard and fires no tick
    anywhere; after a drain the next round completes it."""
    R, B, P = 64, 32, 100_000
    sb = LocalShardedBus(2, _devices(2), ring_cap=R, batch_cap=B, timers_per_sub=1, stream_slots=4, lossless=True,
                         agree="device")
    try:
        sb.subscribe_many(np.full(2, nat.MASK_ALL, dtype=np.uint32))
        sb.timer_add_many(P, source_id0=77)
        for q in range(2):
            ev = np.zeros(B, dtype=EVENT_DTYPE); ev["code"] = 1 + q
            nat.check(sb.put(ev, 10 * (q + 1)), "put")
            _queue_round(sb)
        assert sb.progress() == (2, 0, 0)
        assert len(sb.drain(0)) == R
        nat.check(sb.put(np.zeros(0, dtype=EVENT_DTYPE), 150_000), "put")
        launched = [bus.stats()["batches"] for _, _, bus in sb.shards]
        _queue_round(sb)
        assert sb.progress() == (2, 0, 1)
        assert [bus.stats()["batches"] for _, _, bus in sb.shards] == launched
        assert [bus.stats()["ticks"] for _, _, bus in sb.shards] == [0, 0]
        assert len(sb.drain(1, cap=1)) == 1
        _queue_round(sb)
        assert sb.progress() == (3, 0, 1)
        assert [bus.stats()["ticks"] for _, _, bus in sb.shards] == [1, 1]
        assert sb.drain(0)["flags"].tolist() == [nat.F_TICK] and sb.drain(1)["flags"].tolist()[-1] == nat.F_TICK
    finally:
        sb.close()


def _pair(timers):
    """two one-subscriber lossless shards on one stream; shard 0 has a 10-us periodic timer (window: 32 periods)"""
    a = Bus(1, ring_cap=256, batch_cap=32, timers_per_sub=1, lossless=True, device=_devices(2)[0])
    b = Bus(1, ring_cap=256, batch_cap=32, timers_per_sub=1, lossless=True, device=_devices(2)[1], sub_id_base=1)
    a.subscribe(); b.subscribe()
    if timers:
        a.timer_add(0, 10_000, 5)
    st0, _ = a.stream_create(4, 2)
    st1 = b.stream_attach(st0, 1)
    for bus, st in ((a, st0), (b, st1)):
        bus.stream_set_timeout(st, 20_000)                        # 20 ms
    return a, b, st0, st1


def test_out_of_order_round_is_sticky_and_times_out_the_other_shards():
    """Shard 0's round finds a batch beyond its timer window: it posts no offer and reports CPBUS_EORDER from then on; the
    round queued behind it does nothing.  Shard 1 waits for the missing offer and reports CPBUS_ETIMEDOUT.  Nothing of the
    bad batch is delivered anywhere."""
    a, b, st0, st1 = _pair(True)
    try:
        ev = np.zeros(4, dtype=EVENT_DTYPE); ev["code"] = 3
        nat.check(a.stream_put(st0, ev, 50_000, nowait=True), "put")
        nat.check(a.stream_put(st0, ev, 50_000 + 40 * 10_000, nowait=True), "put")
        for _ in range(2):
            assert a.stream_round_next(st0) == nat.OK and b.stream_round_next(st1) == nat.OK
        ra, rb = a.stream_progress(st0), b.stream_progress(st1)
        assert ra == (nat.EORDER, 1, 0, 0) and rb == (nat.ETIMEDOUT, 1, 0, 0)
        assert a.stream_round_next(st0) == nat.EORDER and a.stream_status(st0) == nat.EORDER
        assert b.stream_status(st1) == nat.ETIMEDOUT
        assert int(a.digests(0, 1)["count"][0]) == 4 + 5 and int(b.digests(1, 1)["count"][0]) == 4
        assert a.stats()["now_ns"] == 50_000 and b.stats()["now_ns"] == 50_000
    finally:
        b.stream_close(st1); a.stream_close(st0); b.close(); a.close()


def test_shard_that_never_queues_its_round_times_out_the_others():
    """The existing bounded wait: shard 1 never queues its round, shard 0's round gives up after the stream timeout
    (set short here) with CPBUS_ETIMEDOUT, sticky, and delivers nothing; shard 1 is not affected."""
    a, b, st0, st1 = _pair(False)
    try:
        ev = np.zeros(8, dtype=EVENT_DTYPE); ev["code"] = 2
        nat.check(a.stream_put(st0, ev, 1000, nowait=True), "put")
        assert a.stream_round_next(st0) == nat.OK
        assert a.stream_progress(st0) == (nat.ETIMEDOUT, 0, 0, 0)
        assert a.stream_round_next(st0) == nat.ETIMEDOUT
        assert int(a.digests(0, 1)["count"][0]) == 0 and a.stats()["batches"] == 0
        assert b.stream_status(st1) == nat.OK
    finally:
        b.stream_close(st1); a.stream_close(st0); b.close(); a.close()


def test_refusals_stay_in_place():
    """cpbus_stream_round_next on a throughput bus and cpbus_stream_fanout_next on a lossless bus give CPBUS_EINVAL; the
    Python followers of each mode refuse the other mode's call."""
    with Bus(8, ring_cap=256, batch_cap=32) as bus:
        st, _ = bus.stream_create(4, 1)
        assert bus.stream_round_next(st) == nat.EINVAL
        bus.stream_close(st)
    with Bus(8, ring_cap=256, batch_cap=32, lossless=True) as bus:
        bus.subscribe_many(np.full(8, nat.MASK_ALL, dtype=np.uint32))
        st, _ = bus.stream_create(4, 1)
        assert bus.stream_fanout_next(st) == nat.EINVAL
        ev = np.zeros(4, dtype=EVENT_DTYPE); ev["code"] = 1
        nat.check(bus.stream_put(st, ev, 100), "put")
        bus.stream_offer(st, bus.stream_admit(st, 4, 100))
        assert bus.stream_round_next(st) == nat.EINVAL            # an explicit round is open
        assert bus.stream_agree(st) == 4
        assert bus.stream_fanout_prefix(st, 4, 100, 4) == nat.OK
        bus.stream_close(st)
    sb = LocalShardedBus(8, _devices(1), ring_cap=256, batch_cap=32, lossless=True)
    try:
        with pytest.raises(nat.CpbusError):
            sb.follow(0)
    finally:
        sb.close()
    sb = LocalShardedBus(8, _devices(1), ring_cap=256, batch_cap=32)
    try:
        with pytest.raises(RuntimeError):
            sb.follow_rounds(0)
    finally:
        sb.close()
