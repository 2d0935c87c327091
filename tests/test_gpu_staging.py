"""Plain fan-out build: each CTA owns a contiguous range of subscribers and stages their control blocks and timer slots in
shared memory, a round at a time.  These traces run ranges of many mailboxes per warp, several staging rounds per CTA,
partial last CTAs, fixed grids and buses without subscribers, bit-exact against the CPU oracle."""
import numpy as np
import pytest

import oracle_binding as ob
import test_gpu_parity as parity
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from containerpilot_b200.sharding import LocalShardedBus

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("store", parity.STORES)
@pytest.mark.parametrize("seed,K", [(1, 0), (2, 1), (3, 2), (4, 4), (5, 8)])
def test_random_mixed_traces_16_subs_per_warp(store, seed, K, monkeypatch):
    """test_gpu_parity's mixed traces with 16 mailboxes per warp: one CTA owns all 64 subscribers."""
    monkeypatch.setenv("CPBUS_SUBS_PER_WARP", "16")
    parity.test_random_mixed_traces(store, seed, K)


@pytest.mark.parametrize("K", [1, 8])
@pytest.mark.parametrize("spw,grid,pdl", [("16", 0, None), ("16", 0, "0"), (None, 3, None), (None, 0, None)])
def test_staging_rounds(K, spw, grid, pdl, monkeypatch):
    """300 subscribers, 512-event batches: at K = 8 and 16 mailboxes per warp a CTA's 128 subscribers take three staging
    rounds and the last CTA is partial; a fixed 3-CTA grid gives each CTA 100 subscribers.  Dense and filtered masks,
    unicast sends, every timer slot armed."""
    if spw:
        monkeypatch.setenv("CPBUS_SUBS_PER_WARP", spw)
    if pdl:
        monkeypatch.setenv("CPBUS_PDL", pdl)
    n_subs, B, R = 300, 512, 4096
    n_events = B * 6 + 123
    rng = np.random.default_rng(1000 + K)
    masks = np.where(rng.random(n_subs) < 0.7, nat.MASK_ALL, tr.zipf_masks(n_subs, 1.0, 3)).astype(np.uint32)
    codes = rng.integers(0, 17, n_events).astype(np.uint32)
    srcs = rng.integers(0, 4096, n_events).astype(np.uint32)
    orc = ob.Oracle(n_subs, timers_per_sub=K, keep_window=R)
    with Bus(n_subs, ring_cap=R, batch_cap=B, timers_per_sub=K, grid_ctas=grid) as bus:
        for s, m in enumerate(masks):
            orc.subscribe(int(m)); bus.subscribe(int(m))
            for j in range(K):
                period = 150_000 + 977 * s + 13 * j
                orc.timer_add(s, period, 5000 + 8 * s + j, j == 3); bus.timer_add(s, period, 5000 + 8 * s + j, j == 3)
        for i in range(n_events):
            if i % B == 0:
                assert orc.advance(i * 500) == 0; nat.check(bus.advance(i * 500), "advance")
            if i % 211 == 0:
                orc.receive((7 * i) % n_subs, 7, 9); nat.check(bus.send((7 * i) % n_subs, 7, 9), "send")
            orc.publish(int(codes[i]), int(srcs[i])); nat.check(bus.publish(int(codes[i]), int(srcs[i])), "publish")
        nat.check(bus.flush(), "flush"); bus.sync()
        st = tr.compare(bus, orc, n_subs, window=R)
        assert st["ticks"] > 0


def _stream_batches(n_batches, B):
    rng = np.random.default_rng(77)
    out = []
    for _ in range(n_batches):
        ev = np.zeros(B, dtype=EVENT_DTYPE)
        ev["code"] = rng.integers(0, 17, B)
        ev["source_id"] = rng.integers(0, 64, B)
        out.append(ev)
    return out


@pytest.mark.parametrize("grid", [0, 3])
def test_stream_fanout_without_subscribers(grid):
    """A bus nobody has subscribed to yet still takes and acknowledges every stream batch: with 4 slots and 12 batches,
    a slot that is never acknowledged would stop the publisher.  grid = 3 is a fixed grid wider than the (empty) need."""
    B, dt = 64, 1000
    with Bus(8, ring_cap=256, batch_cap=B, grid_ctas=grid) as bus:
        st, _ = bus.stream_create(4, 1)
        try:
            for q, ev in enumerate(_stream_batches(12, B)):
                if bus.stream_put(st, ev, (q + 1) * dt, nowait=True) == nat.EAGAIN:
                    bus.sync()   # every earlier fan-out is complete: its slot must have been acknowledged
                    nat.check(bus.stream_put(st, ev, (q + 1) * dt, nowait=True), "cpbus_stream_put")
                nat.check(bus.stream_fanout(st, len(ev), (q + 1) * dt), "cpbus_stream_fanout")
            bus.sync()
            assert bus.stream_status(st) == nat.OK
            assert bus.stats()["deliveries"] == 0
        finally:
            bus.stream_close(st)


def test_stream_with_an_empty_shard():
    """One subscriber over two shards: the second shard has none and must still acknowledge every batch."""
    B, dt = 64, 1000
    batches = _stream_batches(12, B)
    sb = LocalShardedBus(1, [0, 0], ring_cap=256, batch_cap=B, stream_slots=4)
    try:
        assert [count for _, count, _ in sb.shards] == [1, 0]
        sb.subscribe_many(np.array([nat.MASK_ALL], dtype=np.uint32))
        for q, ev in enumerate(batches):
            if sb.put(ev, (q + 1) * dt) == nat.EAGAIN:
                sb.sync()    # every earlier fan-out is complete: its slot must have been acknowledged by both shards
                nat.check(sb.put(ev, (q + 1) * dt), "cpbus_stream_put")
            sb.fanout(len(ev), (q + 1) * dt)
        sb.sync()
        orc = ob.Oracle(1, keep_window=256)
        orc.subscribe(int(nat.MASK_ALL))
        for q, ev in enumerate(batches):
            assert orc.advance((q + 1) * dt) == 0
            for c, s_ in zip(ev["code"], ev["source_id"]):
                assert orc.publish(int(c), int(s_)) == 0
        for g, (first, count, bus) in enumerate(sb.shards):
            assert bus.stream_status(sb._st[g]) == nat.OK
        tr.compare(sb.shards[0][2], orc, 1, window=256)
    finally:
        sb.close()
