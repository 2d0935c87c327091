"""Stream followers (cpbus_stream_fanout_next): shards that are never told a batch's shape fan out the publisher's stream
exactly as an SPMD twin that calls cpbus_stream_fanout(n, now_ns) does — G = 1-4 shards on however many GPUs the box has
(all on one if need be), with programmatic dependent launch on and off and with every CTA building its own descriptor."""
import numpy as np
import pytest

import oracle_binding as ob
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from containerpilot_b200.sharding import LocalShardedBus

pytestmark = pytest.mark.gpu

STATS = ("publishes", "batches", "deliveries", "ticks", "now_ns", "published_by_code", "kernel_launches")


def _devices(g):
    import torch
    nd = torch.cuda.device_count()
    return [i % nd for i in range(g)]


class _Shards:
    """G shard buses on one stream (shard 0's bus owns it).  Shard g holds global ids [first[g], first[g] + count[g]) and has
    `spare` more slots for subscribers added later."""

    def __init__(self, counts, B, K, slots=8, spare=0, lossless=False):
        self.buses, self.first = [], []
        base = 0
        for g, (c, dev) in enumerate(zip(counts, _devices(len(counts)))):
            self.buses.append(Bus(c + spare, ring_cap=1024, batch_cap=B, timers_per_sub=K, digest=True, device=dev,
                                  sub_id_base=base, lossless=lossless))
            self.first.append(base)
            base += c + spare
        st0, _ = self.buses[0].stream_create(slots, len(counts))
        self.st = [st0] + [self.buses[g].stream_attach(st0, g) for g in range(1, len(counts))]

    def put(self, ev, w, raw=False):
        return self.buses[0].stream_put(self.st[0], ev, w, raw, nowait=True)

    def follow(self, g):
        return self.buses[g].stream_fanout_next(self.st[g])

    def fanout(self, g, n, w):
        return self.buses[g].stream_fanout(self.st[g], n, w)

    def close(self):
        for g in range(len(self.buses) - 1, -1, -1):
            self.buses[g].stream_close(self.st[g])
        for b in self.buses:
            b.close()


def _trace(seed, n_batches, B, targets, dt):
    """(events, watermark, raw): ragged and empty batches; RAW batches carry unicast records to any shard's subscribers"""
    rng = np.random.default_rng(seed)
    out, seq = [], 1 << 40
    for q in range(n_batches):
        w = (q + 1) * dt
        r = rng.random()
        n = 0 if r < 0.1 else (int(rng.integers(1, B + 1)) if r < 0.4 else B)
        ev = np.zeros(n, dtype=EVENT_DTYPE)
        ev["code"] = tr.zipf_codes(n, 1.0, seed + q) if n else []
        ev["source_id"] = rng.integers(0, 8, n)
        raw = bool(rng.random() < 0.3)
        if raw:
            ev["seq"] = seq + np.arange(n); seq += n
            ev["ts_ns"] = np.sort(rng.integers(w - dt + 1, w + 1, n))
            ev["target"] = nat.TARGET_ALL
            uni = rng.random(n) < 0.2
            ev["target"][uni] = rng.choice(targets, int(uni.sum()))
            ev["flags"][uni] = nat.F_UNICAST
        out.append((ev, w, raw))
    return out


def _populate(sh, counts, K, seed, period):
    """Zipf masks; shard 1 (0 when alone) gives every third subscriber exact cases; periodic timers on every other
    subscriber and one-shots on some of the rest"""
    rng = np.random.default_rng(seed)
    paired = 1 if len(counts) > 1 else 0
    for g, (bus, c) in enumerate(zip(sh.buses, counts)):
        masks = tr.zipf_masks(c, 1.0, seed + g)
        for i in range(c):
            if g == paired and i % 3 == 0:
                bus.subscribe_pairs(int(masks[i]) & ~0x6, [(1, 3), (2, 5), (int(rng.integers(1, 17)), 1)])
            else:
                bus.subscribe(int(masks[i]))
        if K:
            for i in range(c):
                sid = sh.first[g] + i
                if i % 2 == 0:
                    bus.timer_add(sid, period, 9000 + sid)
                elif i % 5 == 1:
                    bus.timer_add(sid, int(period * (1 + rng.integers(1, 20))), 9500 + sid, oneshot=True)


def _step_result(bus):
    return tuple(int(x) for x in bus.step_result_end(bus.step_result_begin()))


def _assert_twins(f, t, counts, window_every=7):
    for g, c in enumerate(counts):
        bf, bt = f.buses[g], t.buses[g]
        df, dt_ = bf.digests(f.first[g], c), bt.digests(t.first[g], c)
        assert np.array_equal(df, dt_), f"shard {g}: (count, digest) differ"
        for i in range(0, c, window_every):
            assert bf.peek_window(f.first[g] + i).tobytes() == bt.peek_window(t.first[g] + i).tobytes(), (g, i)
        sf, st = bf.stats(), bt.stats()
        for k in STATS:
            assert sf[k] == st[k], (g, k, sf[k], st[k])
        assert bf.debug_events().tobytes() == bt.debug_events().tobytes(), g
        assert bf.publish_counts() == bt.publish_counts(), g


@pytest.mark.parametrize("pdl", ["0", "1"])
@pytest.mark.parametrize("G,K,hints", [(1, 1, None), (2, 4, None), (3, 1, None), (4, 4, None), (2, 1, "2"), (4, 4, "2")])
def test_followers_match_the_spmd_twin(G, K, hints, pdl, monkeypatch):
    """Ragged and empty batches, PUT_STAMP and PUT_RAW records with unicast targets on other shards, periodic and one-shot
    timers, Zipf masks, one shard with pair tables: the followers, told nothing, give what the twin gives when told."""
    monkeypatch.setenv("CPBUS_PDL", pdl)
    if hints:
        monkeypatch.setenv("CPBUS_HINTS", hints)
    B, dt, period = 64, 40_000, 90_000
    counts = [37 + 11 * g for g in range(G)]
    f, t = _Shards(counts, B, K), _Shards(counts, B, K)
    try:
        for sh in (f, t):
            _populate(sh, counts, K, 11 + G, period)
        targets = [f.first[g] + i for g, c in enumerate(counts) for i in range(c)]
        for ev, w, raw in _trace(100 + G * 10 + K, 36, B, targets, dt):
            nat.check(f.put(ev, w, raw), "put"); nat.check(t.put(ev, w, raw), "put")
            res = []
            for g in range(G):
                nat.check(f.follow(g), "cpbus_stream_fanout_next")
                nat.check(t.fanout(g, len(ev), w), "cpbus_stream_fanout")
                res.append((_step_result(f.buses[g]), _step_result(t.buses[g])))
            for a, b in res:
                assert a == b
        for g in range(G):
            assert f.buses[g].stream_status(f.st[g]) == nat.OK
            assert f.buses[g].stream_poll(f.st[g]) is None and t.buses[g].stream_poll(t.st[g]) is None
        _assert_twins(f, t, counts)
    finally:
        f.close(); t.close()


@pytest.mark.parametrize("pdl", ["0", "1"])
@pytest.mark.parametrize("G,ahead,followers_first", [(1, 0, True), (2, 2, True), (3, 5, True), (2, 3, False), (4, 5, False)])
def test_run_ahead_matches_the_oracle(G, ahead, followers_first, pdl, monkeypatch):
    """Up to 5 follower launches queued before the publisher puts their batches (each waits in the kernel), or the batches
    put first: every subscriber matches the oracle, whichever comes first (LocalShardedBus.follow)."""
    monkeypatch.setenv("CPBUS_PDL", pdl)
    N, B, dt, period = 149, 64, 40_000, 90_000
    rng = np.random.default_rng(5 + G)
    masks = np.where(rng.random(N) < 0.5, nat.MASK_ALL, rng.integers(0, 1 << 17, N)).astype(np.uint32)
    batches = [ev for ev, _, _ in _trace(31 + ahead, 30, B, [0], dt)]
    for ev in batches:   # stamped records only: the oracle publishes them like cpbus_publish
        ev["seq"] = 0; ev["ts_ns"] = 0; ev["target"] = 0; ev["flags"] = 0
    sb = LocalShardedBus(N, _devices(G), ring_cap=1024, batch_cap=B, timers_per_sub=1, stream_slots=8)
    try:
        sb.subscribe_many(masks)
        sb.timer_add_many(period, source_id0=7000)
        q = 0
        while q < len(batches):
            k = max(1, min(ahead, len(batches) - q))
            if followers_first:
                for g in range(G):
                    sb.follow(g, k)
            for j in range(q, q + k):
                nat.check(sb.put(batches[j], (j + 1) * dt), "put")
            if not followers_first:
                for g in range(G):
                    sb.follow(g, k)
            for g, (_, _, bus) in enumerate(sb.shards):   # resolve (at most 8 may be outstanding: the 9th would wait for
                assert bus.stream_status(sb._st[g]) == nat.OK   # batches this thread has not put yet)
            q += k
        for g, (first, count, bus) in enumerate(sb.shards):
            assert bus.stream_status(sb._st[g]) == nat.OK
            orc = ob.Oracle(count, timers_per_sub=1, keep_window=1024, sub_id_base=first)
            for i in range(count):
                orc.subscribe(int(masks[first + i]))
                orc.timer_add(first + i, period, 7000 + first + i, False)
            for j, ev in enumerate(batches):
                assert orc.advance((j + 1) * dt) == 0
                for c, s_ in zip(ev["code"], ev["source_id"]):
                    assert orc.publish(int(c), int(s_)) == 0
            tr.compare(bus, orc, count, sub_id_base=first)
            assert bus.stats()["now_ns"] == len(batches) * dt
    finally:
        sb.close()


@pytest.mark.parametrize("pdl", ["0", "1"])
def test_host_calls_between_followers(pdl, monkeypatch):
    """publish, send, advance, timer_add, subscribe and unsubscribe between follower launches: each is ordered behind the
    batches followed before it, as on the twin, and the clock is right after each."""
    monkeypatch.setenv("CPBUS_PDL", pdl)
    B, dt, period, G = 64, 40_000, 90_000, 2
    counts = [30, 41]
    f, t = _Shards(counts, B, 2, spare=6), _Shards(counts, B, 2, spare=6)
    rng = np.random.default_rng(77)
    try:
        for sh in (f, t):
            _populate(sh, counts, 2, 3, period)
        for q, (ev, w, raw) in enumerate(_trace(404, 30, B, [f.first[1] + 2], dt)):
            nat.check(f.put(ev, w, raw), "put"); nat.check(t.put(ev, w, raw), "put")
            for g in range(G):
                nat.check(f.follow(g), "follow"); nat.check(t.fanout(g, len(ev), w), "fanout")
            g, op = q % G, q % 6
            code = int(rng.integers(0, 17))
            for sh in (f, t):
                bus = sh.buses[g]
                if op == 0:
                    nat.check(bus.publish(code, 3), "publish")
                elif op == 1:
                    nat.check(bus.send(sh.first[g] + 1, 5, 2), "send")
                elif op == 2:
                    nat.check(bus.advance(w + dt // 2), "advance")
                elif op == 3:
                    bus.timer_add(sh.first[g] + 4 + q, period * 3, 4444, oneshot=bool(q % 4 == 3))
                elif op == 4:
                    bus.subscribe(nat.MASK_ALL)
                else:
                    bus.unsubscribe(sh.first[g] + q)
            assert f.buses[g].stats()["now_ns"] == t.buses[g].stats()["now_ns"]
        _assert_twins(f, t, [counts[0] + 5, counts[1]])   # five subscribers joined shard 0
    finally:
        f.close(); t.close()


@pytest.mark.parametrize("case", ["window", "behind"])
def test_out_of_order_batch_is_sticky(case):
    """A followed batch beyond the timer window, or behind the clock, delivers nothing, fires no timer, is not
    acknowledged and turns every follower queued behind it into a no-op; from then on the stream reports CPBUS_EORDER.
    The twin's cpbus_stream_fanout refuses the same batch with CPBUS_EORDER."""
    B, period = 32, 10_000
    f, t = _Shards([20], B, 1, slots=4), _Shards([20], B, 1, slots=4)
    try:
        for sh in (f, t):
            sh.buses[0].subscribe_many(np.full(20, nat.MASK_ALL, dtype=np.uint32))
            sh.buses[0].timer_add_many(0, 20, period, source_id0=100)
        ev = np.zeros(B, dtype=EVENT_DTYPE); ev["code"] = 4
        w1 = 5 * period
        w2 = w1 + 40 * period if case == "window" else w1 - period   # window: 32 periods at K = 1
        for sh in (f, t):
            nat.check(sh.put(ev, w1), "put"); nat.check(sh.put(ev, w2), "put"); nat.check(sh.put(ev, w2 + period), "put")
        nat.check(t.fanout(0, B, w1), "fanout")
        assert t.fanout(0, B, w2) == nat.EORDER
        for _ in range(3):
            nat.check(f.follow(0), "follow")
        bf, bt = f.buses[0], t.buses[0]
        assert bf.stream_status(f.st[0]) == nat.EORDER
        assert bf.stream_fanout_next(f.st[0]) == nat.EORDER
        assert bf.stream_fanout(f.st[0], B, w2) == nat.EORDER
        with pytest.raises(nat.CpbusError) as ex:
            bf.stream_poll(f.st[0])
        assert ex.value.status == nat.EORDER
        assert np.array_equal(bf.digests(0, 20), bt.digests(0, 20))       # batch 1 only (and its ticks)
        sf, st = bf.stats(), bt.stats()
        assert (sf["deliveries"], sf["ticks"], sf["now_ns"], sf["publishes"]) == (st["deliveries"], st["ticks"], st["now_ns"], st["publishes"])
        assert sf["now_ns"] == w1
        # batch 2's slot was never acknowledged: the publisher cannot put batch 2 + n_slots
        nat.check(f.put(ev, w2 + 2 * period), "put")                       # batch 4: a fresh slot
        nat.check(f.put(ev, w2 + 3 * period), "put")                       # batch 5: batch 1's slot, acknowledged
        assert f.put(ev, w2 + 4 * period) == nat.EAGAIN                    # batch 6: batch 2's slot, never acknowledged
    finally:
        f.close(); t.close()


def test_follower_whose_batch_never_comes_times_out():
    """The designed bounded wait, once: nothing is put, the follower gives up after the stream timeout, delivers nothing,
    and the stream reports CPBUS_ETIMEDOUT."""
    with Bus(64, ring_cap=256, batch_cap=32, digest=True) as bus:
        bus.subscribe_many(np.full(64, nat.MASK_ALL, dtype=np.uint32))
        st, _ = bus.stream_create(4, 1)
        bus.stream_set_timeout(st, 20_000)                       # 20 ms
        nat.check(bus.stream_fanout_next(st), "follow")
        assert bus.stream_status(st) == nat.ETIMEDOUT
        assert bus.stream_fanout_next(st) == nat.ETIMEDOUT
        assert bus.stats()["deliveries"] == 0
        assert int(bus.digests(0, 64)["count"].max()) == 0
        bus.stream_close(st)


def test_lossless_bus_refuses_followers():
    with Bus(8, ring_cap=256, batch_cap=32, lossless=True) as bus:
        bus.subscribe_many(np.full(8, nat.MASK_ALL, dtype=np.uint32))
        st, _ = bus.stream_create(4, 1)
        assert bus.stream_fanout_next(st) == nat.EINVAL
        bus.stream_close(st)
    sb = LocalShardedBus(8, _devices(1), ring_cap=256, batch_cap=32, lossless=True)
    try:
        with pytest.raises(nat.CpbusError):
            sb.follow(0)
    finally:
        sb.close()
