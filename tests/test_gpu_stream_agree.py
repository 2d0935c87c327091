"""Lossless stream with the shards' minimum agreed on the device (cpbus_stream_offer / cpbus_stream_agree,
LocalShardedBus(lossless=True, agree="device")): the protocol ShardedBus(lossless=True) runs across processes, here in one
process so that it can be checked against the oracle and against the host minimum.  Shards on whatever GPUs this box has
(all on one GPU when there is only one): the offer words and the agree kernel are the same either way."""
import numpy as np
import pytest

import oracle_binding as ob
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


def _pairs(rng, N):
    """every third subscriber also takes exact {code, source} cases on top of its mask"""
    return [[(int(rng.integers(1, 7)), int(rng.integers(0, 8))) for _ in range(int(rng.integers(1, 5)))] if s % 3 == 0 else []
            for s in range(N)]


def _subscribe(sb, masks, pairs):
    for first, count, bus in sb.shards:
        if count:
            bus.subscribe_pairs_many(masks[first:first + count], pairs[first:first + count])


def _check_round(sb):
    """the agreed prefix is the minimum of the offers, on every shard; a stalled offer is (0, stalled)"""
    offers, agreed = sb.last_round
    assert len(set(agreed)) == 1
    if any(s for _, s in offers):
        assert agreed[0] is None and all(p == 0 for p, s in offers if s)
    else:
        assert agreed[0] == min(p for p, _ in offers)
    return offers, agreed[0]


@pytest.mark.parametrize("G", [1, 2, 3, 4])
@pytest.mark.parametrize("seed", [1, 2])
def test_device_agreement_blocks_per_event_like_the_go_bus(G, seed):
    """One global oracle that refuses event by event (mailbox_cap = ring_cap); pair-filtered subscribers; random partial
    drains through the owning shard.  At every stall every subscriber holds exactly what the oracle holds and drained
    records are byte-equal; the agreed prefix is min(p_g) at every round."""
    R, B, N = 128, 64, 14
    rng = np.random.default_rng(500 * G + seed)
    masks = [nat.MASK_ALL, 1 << 2, (1 << 3) | (1 << 2), nat.MASK_ALL, 1 << 5, 0, nat.MASK_ALL]
    masks = np.array((masks * 2)[:N], dtype=np.uint32)
    pairs = _pairs(rng, N)
    orc = ob.Oracle(N, keep_window=0, mailbox_cap=R)
    for s in range(N):
        orc.subscribe(int(masks[s]), pairs[s] or None)
    sb = LocalShardedBus(N, _devices(G), ring_cap=R, batch_cap=B, stream_slots=4, lossless=True, agree="device")
    try:
        _subscribe(sb, masks, pairs)
        n_partial = n_rounds = 0
        for step in range(30):
            now = (step + 1) * 1000
            n = B if step % 4 else int(rng.integers(1, B + 1))          # ragged batches too
            ev = np.zeros(n, dtype=EVENT_DTYPE)
            ev["code"] = rng.integers(1, 7, n); ev["source_id"] = rng.integers(0, 12, n)
            nat.check(sb.put(ev, now), "put")
            assert orc.advance(now) == 0
            i = 0
            while True:
                rc = sb.fanout(n, now)
                n_rounds += 1
                _check_round(sb)
                while i < n:                                          # the oracle publishes event by event until it blocks
                    r = orc.publish(int(ev["code"][i]), int(ev["source_id"][i]))
                    if r == ob.EAGAIN:
                        break
                    assert r == 0
                    i += 1
                assert _counts(sb) == [orc.count(s) for s in range(N)], (step, i, rc)
                if rc == nat.OK:
                    assert i == n
                    break
                assert rc == nat.EAGAIN and i < n
                n_partial += 1 if i > 0 else 0
                for s in rng.permutation(N)[:4]:                      # some consumers run (not necessarily the full one)
                    take = int(rng.integers(1, R + 1))
                    assert sb.drain(int(s), cap=take).tobytes() == orc.consume(int(s), take).tobytes()
        for s in range(N):
            assert sb.drain(s, cap=R).tobytes() == orc.consume(s, R).tobytes()
        assert n_partial > 0 and n_rounds > 30
        for _, _, bus in sb.shards:
            st = bus.stats()
            assert st["overwritten"] == 0 and st["admit_partial"] > 0
    finally:
        sb.close()


def _raw_batches(seed, n_batches, B, N, dt):
    """RAW stream records (running seq, ts = now), with unicast records to global ids on every shard; ragged and empty
    batches"""
    rng = np.random.default_rng(seed)
    out, seq = [], 0
    for q in range(n_batches):
        r = rng.random()
        n = 0 if r < 0.15 else int(rng.integers(1, B + 1)) if r < 0.45 else B
        ev = np.zeros(n, dtype=EVENT_DTYPE)
        ev["seq"] = seq + np.arange(n); seq += n
        ev["ts_ns"] = (q + 1) * dt
        ev["code"] = rng.integers(0, 17, n); ev["source_id"] = rng.integers(0, 12, n)
        ev["target"] = nat.TARGET_ALL
        uni = rng.random(n) < 0.25
        ev["target"][uni] = rng.integers(0, N, int(uni.sum()))
        ev["flags"][uni] = nat.F_UNICAST
        out.append(ev)
    return out


@pytest.mark.parametrize("G,K", [(1, 1), (2, 1), (3, 2), (4, 1)])
def test_device_agreement_equals_the_host_minimum(G, K):
    """Twin LocalShardedBus drivers, one taking the minimum on the host and one agreeing on the device, given the same
    batches (timers, unicast records, pair filters, ragged and empty batches) and the same drain schedule.  Every round
    returns the same code, every drain the same bytes; at the end every subscriber's (count, digest) and every shard's
    statistics are identical — save the launch count, which differs by exactly the two agreement kernels per round and the
    admission passes the host driver skips once one shard has stalled."""
    R, B, N, dt = 64, 32, 23, 40_000
    periods = [90_000, 130_000][:K]
    rng = np.random.default_rng(31 * G + K)
    masks = np.where(rng.random(N) < 0.5, nat.MASK_ALL, rng.integers(0, 1 << 17, N)).astype(np.uint32)
    masks[3] = 0
    pairs = _pairs(rng, N)
    batches = _raw_batches(13 * G + K, 40, B, N, dt)
    kw = dict(ring_cap=R, batch_cap=B, timers_per_sub=K, stream_slots=4, lossless=True)
    host = LocalShardedBus(N, _devices(G), **kw)
    dev = LocalShardedBus(N, _devices(G), agree="device", **kw)
    try:
        for sb in (host, dev):
            _subscribe(sb, masks, pairs)
            sb.timer_add_many(periods[0], source_id0=1000)
            for p in periods[1:]:
                for s in range(N):
                    sb.bus_of(s).timer_add(s, p, 2000 + s)
        rounds = n_stalls = 0
        for q, ev in enumerate(batches):
            now = (q + 1) * dt
            nat.check(host.put(ev, now, raw=True), "put")
            nat.check(dev.put(ev, now, raw=True), "put")
            while True:
                rc_h, rc_d = host.fanout(len(ev), now), dev.fanout(len(ev), now)
                rounds += 1
                _check_round(dev)
                assert rc_h == rc_d, (q, rc_h, rc_d)
                assert _counts(host) == _counts(dev), q
                if rc_d == nat.OK:
                    break
                n_stalls += 1
                for s in rng.permutation(N)[:6]:
                    take = int(rng.integers(1, R + 1))
                    assert host.drain(int(s), cap=take).tobytes() == dev.drain(int(s), cap=take).tobytes()
        assert n_stalls > 0
        for s in range(N):
            assert host.drain(s).tobytes() == dev.drain(s).tobytes()
        got, want = dev.digests(), host.digests()
        assert got.tobytes() == want.tobytes() and int(want["count"].sum()) > 0
        for (_, _, bh), (_, _, bd) in zip(host.shards, dev.shards):
            sh, sd = bh.stats(), bd.stats()
            varying = ("kernel_launches", "admit_passes", "admit_skipped")
            assert {k: v for k, v in sh.items() if k not in varying} == {k: v for k, v in sd.items() if k not in varying}
            assert sd["kernel_launches"] - sd["admit_passes"] - 2 * rounds == sh["kernel_launches"] - sh["admit_passes"]
            assert sd["admit_passes"] >= sh["admit_passes"]
    finally:
        host.close()
        dev.close()


def test_empty_remainder_whose_ticks_do_not_fit_stalls_every_shard():
    """An empty batch whose tick does not fit one shard's full mailbox: that shard offers a stall, every shard's agree
    gives EAGAIN and no fan-out is launched anywhere — the shard with room does not fire its tick ahead of the other."""
    R, B, P = 64, 32, 100_000
    sb = LocalShardedBus(2, _devices(2), ring_cap=R, batch_cap=B, timers_per_sub=1, stream_slots=4, lossless=True,
                         agree="device")
    try:
        sb.subscribe_many(np.full(2, nat.MASK_ALL, dtype=np.uint32))
        sb.timer_add_many(P, source_id0=77)                         # due at 100,000
        for q in range(2):                                          # 64 records each: both mailboxes at capacity
            ev = np.zeros(B, dtype=EVENT_DTYPE); ev["code"] = 1 + q
            nat.check(sb.put(ev, 10 * (q + 1)), "put")
            assert sb.fanout(B, 10 * (q + 1)) == nat.OK
        assert len(sb.drain(0)) == R                                # shard 0 has room again, shard 1 does not
        nat.check(sb.put(np.zeros(0, dtype=EVENT_DTYPE), 150_000), "put")
        launched = [bus.stats()["batches"] for _, _, bus in sb.shards]
        assert sb.fanout(0, 150_000) == nat.EAGAIN
        offers, agreed = sb.last_round
        assert offers == [(0, False), (0, True)] and agreed == [None, None]
        assert [bus.stats()["batches"] for _, _, bus in sb.shards] == launched
        assert [bus.stats()["ticks"] for _, _, bus in sb.shards] == [0, 0]
        assert _counts(sb) == [2 * B, 2 * B]
        assert len(sb.drain(1, cap=1)) == 1
        assert sb.fanout(0, 150_000) == nat.OK
        assert [bus.stats()["ticks"] for _, _, bus in sb.shards] == [1, 1]
        assert sb.drain(0)["flags"].tolist() == [nat.F_TICK] and sb.drain(1)["flags"].tolist()[-1] == nat.F_TICK
    finally:
        sb.close()


def _raises(status, fn, *args):
    with pytest.raises(nat.CpbusError) as ei:
        fn(*args)
    assert ei.value.status == status, ei.value


def test_errors():
    """EINVAL: a throughput-mode bus, agree without an offer, a second offer in one round, a prefix beyond the remainder,
    a stalled offer with a prefix.  The round survives a refused call."""
    R, B = 64, 32
    with Bus(1, ring_cap=R, batch_cap=B) as bus:                    # throughput mode needs no agreement
        st, _ = bus.stream_create(4, 1)
        _raises(nat.EINVAL, bus.stream_offer, st, 0)
        _raises(nat.EINVAL, bus.stream_agree, st)
        bus.stream_close(st)
    with Bus(1, ring_cap=R, batch_cap=B, lossless=True) as bus:
        bus.subscribe()
        st, _ = bus.stream_create(4, 1)
        _raises(nat.EINVAL, bus.stream_agree, st)                   # no offer this round
        _raises(nat.EINVAL, bus.stream_offer, st, B + 1)            # beyond any batch (nothing admitted yet)
        ev = np.zeros(B - 8, dtype=EVENT_DTYPE); ev["code"] = 3
        nat.check(bus.stream_put(st, ev, 1000), "put")
        assert bus.stream_admit(st, B - 8, 1000) == B - 8
        _raises(nat.EINVAL, bus.stream_offer, st, B - 7)            # beyond the remainder of the admitted batch
        _raises(nat.EINVAL, bus.stream_offer, st, 1, True)          # a stall offers no prefix
        bus.stream_offer(st, 10)
        _raises(nat.EINVAL, bus.stream_offer, st, 10)               # one offer per round
        assert bus.stream_agree(st) == 10
        assert bus.stream_fanout_prefix(st, B - 8, 1000, 10) == nat.EAGAIN
        assert bus.stream_admit(st, B - 8, 1000) == B - 18
        _raises(nat.EINVAL, bus.stream_offer, st, B - 17)           # the remainder shrank
        bus.stream_offer(st, B - 18)
        assert bus.stream_agree(st) == B - 18
        assert bus.stream_fanout_prefix(st, B - 8, 1000, B - 18) == nat.OK
        assert bus.drain(0)["code"].tolist() == [3] * (B - 8)
        assert bus.stream_status(st) == nat.OK
        bus.stream_close(st)


def test_agree_whose_peer_never_offers_times_out():
    """Shard 1 never offers: shard 0's agree gives up after the stream timeout (a few ms here) with CPBUS_ETIMEDOUT,
    sticky like a batch that never arrives, and nothing is delivered."""
    B = 32
    a = Bus(1, ring_cap=64, batch_cap=B, lossless=True, device=_devices(2)[0])
    b = Bus(1, ring_cap=64, batch_cap=B, lossless=True, device=_devices(2)[1], sub_id_base=1)
    st0 = st1 = None
    try:
        a.subscribe(); b.subscribe()
        st0, _ = a.stream_create(4, 2)
        st1 = b.stream_attach(st0, 1)
        a.stream_set_timeout(st0, 5000)
        ev = np.zeros(B, dtype=EVENT_DTYPE); ev["code"] = 2
        nat.check(a.stream_put(st0, ev, 1000, nowait=True), "put")
        a.stream_offer(st0, a.stream_admit(st0, B, 1000))
        _raises(nat.ETIMEDOUT, a.stream_agree, st0)
        assert a.stream_status(st0) == nat.ETIMEDOUT                # sticky
        assert a.stream_fanout_prefix(st0, B, 1000, B) == nat.ETIMEDOUT
        _raises(nat.ETIMEDOUT, a.stream_offer, st0, 0)
        a.sync()
        assert int(a.digests(0, 1)["count"][0]) == 0 and a.stats()["batches"] == 0
        assert b.stream_status(st1) == nat.OK                       # the other shard's bus is not affected
    finally:
        if st1 is not None:
            b.stream_close(st1)
        if st0 is not None:
            a.stream_close(st0)
        b.close()
        a.close()
