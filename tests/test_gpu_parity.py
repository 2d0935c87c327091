"""Parity tests proper: the CUDA bus, driven through the C-ABI, against the CPU
oracle on the same seeded traces.  Bit-exact: same records, same per-subscriber
order, same counts, same order-sensitive digests."""
import numpy as np
import pytest

import oracle_binding as ob
import ring_check as rc
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE

pytestmark = pytest.mark.gpu
STORES = [nat.STORE_V4, nat.STORE_V8, nat.STORE_BULK]


def publish_codes(bus, codes, srcs):
    ev = np.zeros(len(codes), dtype=EVENT_DTYPE)
    ev["code"], ev["source_id"] = codes, srcs
    nat.check(bus.publish_many(ev), "publish")


@pytest.mark.parametrize("store", STORES)
def test_config1_plumbing_full_sequences(store):
    """BASELINE config 1: 8 subscribers, 10k events, all-ones masks, single publisher.
    Lossless mode with a consumer draining, like the reference's blocking channels:
    the FULL per-subscriber sequence is compared."""
    n_subs, n_events = 8, 10_000
    rng = np.random.default_rng(0xC0DEB201)
    codes = rng.integers(1, 17, n_events).astype(np.uint32); srcs = rng.integers(0, 64, n_events).astype(np.uint32)
    orc = ob.Oracle(n_subs)
    for _ in range(n_subs):
        orc.subscribe()
    assert orc.publish_many(codes, srcs) == 0
    with Bus(n_subs, ring_cap=1024, batch_cap=256, lossless=True, store_path=store) as bus:
        bus.subscribe_many(np.full(n_subs, nat.MASK_ALL, dtype=np.uint32))
        got = [[] for _ in range(n_subs)]
        ev = np.zeros(1, dtype=EVENT_DTYPE)
        i = 0
        while i < n_events:
            ev["code"], ev["source_id"] = codes[i], srcs[i]
            rc = bus.publish_many(ev)
            if rc == nat.EAGAIN:                      # publisher blocked: consumers run
                for s in range(n_subs):
                    got[s].append(bus.drain(s))
                continue
            nat.check(rc, "publish")
            i += 1
        while bus.flush() == nat.EAGAIN:
            for s in range(n_subs):
                got[s].append(bus.drain(s))
        for s in range(n_subs):
            got[s].append(bus.drain(s))
            seq = np.concatenate(got[s])
            assert len(seq) == n_events
            assert seq.tobytes() == orc.mailbox(s).tobytes(), f"subscriber {s}"
        d = bus.digests(0, n_subs)
        assert all(int(d["digest"][s]) == orc.digest(s) for s in range(n_subs))
        st = bus.stats()
        assert st["deliveries"] == n_subs * n_events and st["overwritten"] == 0 and st["publishes"] == n_events
        assert st["published_by_code"] == [orc.published_by_code(c) for c in range(17)]


@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("batch_cap", [32, 256, 512])
def test_dense_throughput_mode_window(store, batch_cap):
    """All-ones masks, overwrite-oldest mode: count, digest and the last ring_cap records."""
    n_subs, n_events = 300, 5000
    rng = np.random.default_rng(5)
    codes = rng.integers(0, 17, n_events).astype(np.uint32); srcs = rng.integers(0, 4096, n_events).astype(np.uint32)
    orc = ob.Oracle(n_subs, keep_window=1024)
    for _ in range(n_subs):
        orc.subscribe()
    orc.publish_many(codes, srcs)
    with Bus(n_subs, ring_cap=1024, batch_cap=batch_cap, store_path=store) as bus:
        bus.subscribe_many(np.full(n_subs, nat.MASK_ALL, dtype=np.uint32))
        publish_codes(bus, codes, srcs)
        nat.check(bus.flush(), "flush"); bus.sync()
        st = tr.compare(bus, orc, n_subs)
        assert st["overwritten"] == n_subs * (n_events - 1024)


@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("K,zipf", [(0, None), (1, None), (0, 1.0), (2, 1.0)])
def test_largest_batches(store, K, zipf):
    """batch_cap = 1024, the largest a launch takes (every thread moves 8 chunks in the planar re-layout; 32 chunks of 32 events
    in the filter passes): dense, dense + ticks, filtered (ORDERED) and filtered + ticks + unicast, ragged last batch."""
    n_subs, n_events, B, R = 200, 1024 * 3 + 517, 1024, 4096
    rng = np.random.default_rng(77 + K)
    masks = tr.zipf_masks(n_subs, zipf, 3) if zipf else np.full(n_subs, nat.MASK_ALL, dtype=np.uint32)
    codes = (tr.zipf_codes(n_events, zipf, 4) if zipf else rng.integers(0, 17, n_events)).astype(np.uint32)
    srcs = rng.integers(0, 4096, n_events).astype(np.uint32)
    orc = ob.Oracle(n_subs, timers_per_sub=K, keep_window=R)
    with Bus(n_subs, ring_cap=R, batch_cap=B, timers_per_sub=K, store_path=store) as bus:
        for s, m in enumerate(masks):
            orc.subscribe(int(m)); bus.subscribe(int(m))
            for j in range(K):
                orc.timer_add(s, 40_000 + 977 * s + 13 * j, 5000 + 2 * s + j, False); bus.timer_add(s, 40_000 + 977 * s + 13 * j, 5000 + 2 * s + j, False)
        for i in range(n_events):
            if i % 64 == 0:
                assert orc.advance(i * 500) == 0; nat.check(bus.advance(i * 500), "advance")
            if K == 2 and i % 97 == 0:
                orc.receive(i % n_subs, 7, 9); nat.check(bus.send(i % n_subs, 7, 9), "send")
            orc.publish(int(codes[i]), int(srcs[i])); nat.check(bus.publish(int(codes[i]), int(srcs[i])), "publish")
        nat.check(bus.flush(), "flush"); bus.sync()
        st = tr.compare(bus, orc, n_subs, window=R)
        assert st["batches"] <= n_events // B + 2 + (n_events // 64 if K else 0)


@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("seed,K", [(1, 0), (2, 1), (3, 2), (4, 4), (5, 8)])
def test_random_mixed_traces(store, seed, K):
    """Filters, unicast sends, membership changes, clock advances, periodic and one-shot timers."""
    ops, n_total = tr.random_ops(seed, 40, 6000, timers_per_sub=K, max_subs=64)
    orc = tr.run_oracle(ops, 64, timers_per_sub=K)
    with Bus(64, ring_cap=2048, batch_cap=128, timers_per_sub=K, store_path=store) as bus:
        tr.run_bus(bus, ops)
        tr.compare(bus, orc, n_total, window=2048)


def test_timer_heavy_config3_shape():
    """BASELINE config 3 shape, scaled: one periodic 1 kHz timer per subscriber, 1 tick per 100 publishes."""
    n_subs, n_events, dt = 512, 20_000, 10_000      # 10 us per publish, 1 ms period
    rng = np.random.default_rng(0xC0DEB203)
    codes = rng.integers(1, 17, n_events).astype(np.uint32); srcs = rng.integers(0, 4096, n_events).astype(np.uint32)
    orc = ob.Oracle(n_subs, timers_per_sub=1, keep_window=1024)
    for s in range(n_subs):
        orc.subscribe(); orc.timer_add(s, 1_000_000, 5000 + s, False)
    assert orc.publish_many(codes, srcs, dt_ns=dt) == 0
    with Bus(n_subs, ring_cap=1024, batch_cap=256, timers_per_sub=1) as bus:
        bus.subscribe_many(np.full(n_subs, nat.MASK_ALL, dtype=np.uint32))
        bus.timer_add_many(0, n_subs, 1_000_000, source_id0=5000)
        ev = np.zeros(1, dtype=EVENT_DTYPE)
        for i in range(n_events):
            nat.check(bus.advance((i + 1) * dt), "advance")
            ev["code"], ev["source_id"] = codes[i], srcs[i]
            nat.check(bus.publish_many(ev), "publish")
        nat.check(bus.flush(), "flush"); bus.sync()
        st = tr.compare(bus, orc, n_subs)
        assert st["ticks"] == n_subs * (n_events * dt // 1_000_000)


@pytest.mark.parametrize("order_block", [None, "64", "1000", "-1"])
def test_zipf_filter_sweep_scaled(order_block, monkeypatch):
    """BASELINE config 5 shape, scaled: Zipf-skewed masks and event codes.  The mask order is built per block of consecutive
    subscribers (locality of the rings written at the same time); CPBUS_ORDER_BLOCK forces small blocks / one global order."""
    if order_block is not None:
        monkeypatch.setenv("CPBUS_ORDER_BLOCK", order_block)
    n_subs, n_events = 2048, 8000
    for s_exp in ((0.5, 1.0, 1.5) if order_block is None else (1.0,)):
        masks = tr.zipf_masks(n_subs, s_exp, 21); codes = tr.zipf_codes(n_events, s_exp, 22)
        srcs = (np.arange(n_events) % 4096).astype(np.uint32)
        orc = ob.Oracle(n_subs, keep_window=1024)
        for m in masks:
            orc.subscribe(int(m))
        orc.publish_many(codes, srcs)
        with Bus(n_subs, ring_cap=1024, batch_cap=256) as bus:
            bus.subscribe_many(masks)
            publish_codes(bus, codes, srcs)
            nat.check(bus.flush(), "flush"); bus.sync()
            st = tr.compare(bus, orc, n_subs)
            hist = np.bincount(codes, minlength=17)
            want = int(sum(int(hist[c]) * int(((masks >> np.uint32(c)) & 1).sum()) for c in range(17)))
            assert st["deliveries"] == want


def test_config2_scaled_and_device_resident_batches():
    """BASELINE config 2, scaled to what the oracle finishes in seconds, fed through
    cpbus_publish_device (HBM-resident batches, the multi-GPU / bench ingest path)."""
    import torch
    n_subs, n_events, B = 4096, 20_480, 256
    rng = np.random.default_rng(0xC0DEB202)
    codes = rng.integers(1, 17, n_events).astype(np.uint32); srcs = rng.integers(0, 4096, n_events).astype(np.uint32)
    orc = ob.Oracle(n_subs, keep_window=1024)
    for _ in range(n_subs):
        orc.subscribe()
    orc.publish_many(codes, srcs)
    ev = np.zeros(n_events, dtype=EVENT_DTYPE)
    ev["seq"] = np.arange(n_events); ev["code"], ev["source_id"], ev["target"] = codes, srcs, nat.TARGET_ALL
    dev = torch.from_numpy(ev.view(np.uint8).reshape(-1, 32)).cuda()
    stream = torch.cuda.current_stream()
    with Bus(n_subs, ring_cap=1024, batch_cap=B, stream=stream.cuda_stream) as bus:
        bus.subscribe_many(np.full(n_subs, nat.MASK_ALL, dtype=np.uint32))
        for i in range(0, n_events, B):
            nat.check(bus.publish_device(dev.data_ptr() + i * 32, B, 0), "publish_device")
        bus.sync()
        tr.compare(bus, orc, n_subs)
        fold = bus.digest_fold(0, n_subs)
        assert fold[0] == n_subs * n_events and fold[3] == n_subs
        assert fold[1] == (orc.digest(0) * n_subs) & 0xFFFFFFFFFFFFFFFF     # every mailbox holds the same sequence


def test_full_size_config2_properties():
    """BASELINE config 2 at full width (65,536 subscribers): size-independent properties.
    Every mailbox must hold the same sequence as oracle subscriber 0 (all-ones masks)."""
    import torch
    n_subs, n_events, B = 65_536, 4096, 256
    rng = np.random.default_rng(0xC0DEB202)
    codes = rng.integers(1, 17, n_events).astype(np.uint32); srcs = rng.integers(0, 4096, n_events).astype(np.uint32)
    orc = ob.Oracle(1, keep_window=1024); orc.subscribe(); orc.publish_many(codes, srcs)
    ev = np.zeros(n_events, dtype=EVENT_DTYPE)
    ev["seq"] = np.arange(n_events); ev["code"], ev["source_id"], ev["target"] = codes, srcs, nat.TARGET_ALL
    dev = torch.from_numpy(ev.view(np.uint8).reshape(-1, 32)).cuda()
    with Bus(n_subs, ring_cap=1024, batch_cap=B, stream=torch.cuda.current_stream().cuda_stream) as bus:
        bus.subscribe_many(np.full(n_subs, nat.MASK_ALL, dtype=np.uint32))
        for i in range(0, n_events, B):
            nat.check(bus.publish_device(dev.data_ptr() + i * 32, B, 0), "publish_device")
        bus.sync()
        d = bus.digests(0, n_subs)
        assert (d["count"] == n_events).all() and (d["digest"] == np.uint64(orc.digest(0))).all()
        want = orc.mailbox(0).tobytes()
        for s in (0, 1, 7, 4095, 32_768, 65_535):
            assert bus.peek_window(s).tobytes() == want
        # the ring memory itself: every mailbox's tail and ring against the fleet reference (no sampling)
        ptrs = bus.device_ptrs()
        model = rc.FleetModel(n_subs, 1024, ev, [(i, i + B, 0) for i in range(0, n_events, B)],
                              np.full(n_subs, nat.MASK_ALL, dtype=np.uint32))
        model.pin((0, 65_535))
        with rc.fleet_views(ptrs, n_subs, 1024) as views:
            assert rc.check(views, model) == n_subs * 1024
        st = bus.stats()
        assert st["deliveries"] == n_subs * n_events


def test_lossless_backpressure_and_drain():
    """A full mailbox stalls the publisher (EAGAIN), nothing is lost, order is kept."""
    orc = ob.Oracle(3)
    for m in (nat.MASK_ALL, 1 << 2, nat.MASK_ALL):
        orc.subscribe(m)
    with Bus(3, ring_cap=64, batch_cap=32, lossless=True) as bus:
        bus.subscribe_many(np.array([nat.MASK_ALL, 1 << 2, nat.MASK_ALL], dtype=np.uint32))
        got = [[], [], []]
        n_block = 0
        for i in range(1000):
            code = 1 + i % 3
            orc.publish(code, i)
            while True:
                rc = bus.publish(code, i)
                if rc == nat.EAGAIN:
                    n_block += 1
                    got[0].append(bus.drain(0)); got[2].append(bus.drain(2, cap=5))
                    got[1].append(bus.drain(1))
                    continue
                nat.check(rc, "publish"); break
        while bus.flush() == nat.EAGAIN:
            for s in range(3):
                got[s].append(bus.drain(s))
        for s in range(3):
            got[s].append(bus.drain(s))
            assert np.concatenate(got[s]).tobytes() == orc.mailbox(s).tobytes()
        assert n_block > 5 and bus.stats()["overwritten"] == 0


def test_unsubscribe_twice_and_unknown_ids():
    with Bus(4) as bus:
        s = bus.subscribe()
        bus.unsubscribe(s)
        with pytest.raises(nat.CpbusError) as e:
            bus.unsubscribe(s)
        assert e.value.status == nat.ECLOSED                      # Go: negative WaitGroup panic (bus.go:121)
        with pytest.raises(nat.CpbusError) as e:
            bus.unsubscribe(99)
        assert e.value.status == nat.ENOENT
        assert bus.publish(1, 0) == nat.OK and bus.flush() == nat.OK   # publishing to nobody is fine (jobs_test.go:33-38)
        assert bus.publish(17, 0) == nat.EINVAL
        assert bus.send(s, 1, 0) == nat.ECLOSED and bus.send(99, 1, 0) == nat.ENOENT     # direct send to a mailbox that is gone
        assert bus.advance(5) == nat.OK and bus.advance(4) == nat.EORDER


def test_empty_and_ragged_batches():
    """Edge cases: empty flush, single event, batch sizes that are not multiples of 32, ring wrap inside a batch."""
    orc = ob.Oracle(5, keep_window=64)
    for m in (nat.MASK_ALL, 0, 1 << 16, nat.MASK_ALL, 0x1FFFE):
        orc.subscribe(m)
    with Bus(5, ring_cap=64, batch_cap=32) as bus:
        bus.subscribe_many(np.array([nat.MASK_ALL, 0, 1 << 16, nat.MASK_ALL, 0x1FFFE], dtype=np.uint32))
        assert bus.flush() == nat.OK
        n = 0
        for chunk in (1, 31, 33, 7, 64, 1, 129):
            for _ in range(chunk):
                c = n % 17
                orc.publish(c, n); nat.check(bus.publish(c, n), "publish"); n += 1
            nat.check(bus.flush(), "flush")
        bus.sync()
        tr.compare(bus, orc, 5, window=64)


def test_step_result_written_by_the_kernel():
    """cpbus_step_result_begin/_end: the fan-out kernel leaves {deliveries, ticks, sum fold32(new digest), launch ordinal}
    of every launch in a ring — checked against per-mailbox digests and the oracle's counts."""
    n_subs = 777
    rng = np.random.default_rng(9)
    masks = np.where(rng.random(n_subs) < 0.5, nat.MASK_ALL, rng.integers(1, 1 << 17, n_subs)).astype(np.uint32)
    orc = ob.Oracle(n_subs, timers_per_sub=1, keep_window=1024)
    with Bus(n_subs, ring_cap=1024, batch_cap=256, timers_per_sub=1) as bus:
        bus.subscribe_many(masks)
        for m in masks:
            orc.subscribe(int(m))
        bus.timer_add_many(0, n_subs, 70_000, source_id0=100)
        for s in range(n_subs):
            orc.timer_add(s, 70_000, 100 + s, False)
        prev_counts = np.zeros(n_subs, dtype=np.uint64)
        now = 0
        for step in range(6):
            codes = rng.integers(0, 17, 200).astype(np.uint32); srcs = rng.integers(0, 50, 200).astype(np.uint32)
            d0, t0 = orc.total_deliveries(), orc.total_ticks()
            for c, s_ in zip(codes, srcs):
                now += 1000
                nat.check(bus.advance(now), "advance"); orc.advance(now)
                nat.check(bus.publish(int(c), int(s_)), "publish"); orc.publish(int(c), int(s_))
            nat.check(bus.flush(), "flush")
            res = bus.step_result_end(bus.step_result_begin())
            dig = bus.digests(0, n_subs)
            touched = dig["count"] != prev_counts
            fold = (dig["digest"] ^ (dig["digest"] >> np.uint64(32))) & np.uint64(0xFFFFFFFF)
            assert res[0] == orc.total_deliveries() - d0 and res[1] == orc.total_ticks() - t0
            assert res[2] == int(fold[touched].sum()) and res[3] == step + 1
            prev_counts = dig["count"].copy()
        tr.compare(bus, orc, n_subs)


def test_drain_after_overwrite_reports_lost_records():
    with Bus(2, ring_cap=64, batch_cap=32) as bus:
        bus.subscribe(); bus.subscribe(1 << 3)
        for i in range(200):
            nat.check(bus.publish(1 + i % 4, i), "publish")
        nat.check(bus.flush(), "flush")
        assert bus.stats()["overwritten"] == (200 - 64) + 0      # mailbox 1 only took code 3: 50 records, nothing lost
        got = bus.drain(0)
        assert len(got) == 64 and list(got["source_id"]) == list(range(136, 200))
        assert bus.stats()["overwritten"] == 0 and len(bus.drain(0)) == 0


def test_staged_ingest_is_bit_identical():
    """cpbus_publish_device_staged (CTA 0 pulls the batch, stages it locally, the other CTAs read the staged copy):
    same mailboxes as the direct path.  On one GPU the 'peer' pointer is simply local."""
    import torch
    n_subs, n_events, B = 5000, 2048, 256
    rng = np.random.default_rng(31)
    masks = np.where(rng.random(n_subs) < 0.6, nat.MASK_ALL, rng.integers(1, 1 << 17, n_subs)).astype(np.uint32)
    codes = rng.integers(0, 17, n_events).astype(np.uint32); srcs = rng.integers(0, 99, n_events).astype(np.uint32)
    orc = ob.Oracle(n_subs, timers_per_sub=1, keep_window=1024)
    for s, m in enumerate(masks):
        orc.subscribe(int(m)); orc.timer_add(s, 333_000, 7000 + s, False)
    assert orc.publish_many(codes, srcs, dt_ns=10_000) == 0
    ev = np.zeros(n_events, dtype=EVENT_DTYPE)
    ev["seq"] = np.arange(n_events); ev["ts_ns"] = (np.arange(n_events) + 1) * 10_000
    ev["code"], ev["source_id"], ev["target"] = codes, srcs, nat.TARGET_ALL
    dev = torch.from_numpy(ev.view(np.uint8).reshape(-1, 32)).cuda()
    with Bus(n_subs, ring_cap=1024, batch_cap=B, timers_per_sub=1, stream=torch.cuda.current_stream().cuda_stream) as bus:
        bus.subscribe_many(masks)
        bus.timer_add_many(0, n_subs, 333_000, source_id0=7000)
        for i in range(0, n_events, B):
            # every other call names the next batch so that both the pull-now and the prefetched paths are exercised
            d = (1, 2, 2, 1, 0)[(i // B) % 5]                       # hint the next batch, the one after it, or nothing
            nxt = dev.data_ptr() + (i + d * B) * 32 if d and i + d * B < n_events else 0
            nat.check(bus.publish_device_staged(dev.data_ptr() + i * 32, B, (i + B) * 10_000, nxt, B if nxt else 0), "cpbus_publish_device_staged")
        bus.sync()
        tr.compare(bus, orc, n_subs)


def _oracle_for_one(gid, mask, codes, srcs, dt_ns=0, timer=None, window=1024):
    """The exact sequence of ONE subscriber of a huge shard: a 1-subscriber oracle with sub_id_base = gid."""
    orc = ob.Oracle(1, timers_per_sub=1 if timer else 0, keep_window=window, sub_id_base=gid)
    orc.subscribe(int(mask))
    if timer:
        orc.timer_add(gid, timer[0], timer[1] + gid, False)
    assert orc.publish_many(codes, srcs, dt_ns=dt_ns) == 0
    return orc


def test_full_size_config3_properties():
    """BASELINE config 3 at full width: 1,048,576 subscribers, one 1 kHz timer each, ticks interleaved.
    Size-independent checks: every mailbox's count; exact digest + last-1024 window of sampled subscribers
    against a 1-subscriber oracle placed at that global id; global delivery/tick totals."""
    import torch
    n_subs, n_events, B, dt, period = 1_048_576, 1536, 256, 10_000, 1_000_000
    rng = np.random.default_rng(0xC0DEB203)
    codes = rng.integers(1, 17, n_events).astype(np.uint32); srcs = rng.integers(0, 4096, n_events).astype(np.uint32)
    ev = np.zeros(n_events, dtype=EVENT_DTYPE)
    ev["seq"] = np.arange(n_events); ev["ts_ns"] = (np.arange(n_events) + 1) * dt
    ev["code"], ev["source_id"], ev["target"] = codes, srcs, nat.TARGET_ALL
    dev = torch.from_numpy(ev.view(np.uint8).reshape(-1, 32)).cuda()
    with Bus(n_subs, ring_cap=1024, batch_cap=B, timers_per_sub=1, stream=torch.cuda.current_stream().cuda_stream) as bus:
        bus.subscribe_many(np.full(n_subs, nat.MASK_ALL, dtype=np.uint32))
        bus.timer_add_many(0, n_subs, period, source_id0=1_000_000)
        for i in range(0, n_events, B):
            nat.check(bus.publish_device(dev.data_ptr() + i * 32, B, (i + B) * dt), "cpbus_publish_device")
        bus.sync()
        n_ticks = (n_events * dt) // period
        d = bus.digests(0, n_subs)
        assert (d["count"] == n_events + n_ticks).all()
        for gid in (0, 1, 31, 4097, 65_535, 524_288, 1_048_575):
            orc = _oracle_for_one(gid, nat.MASK_ALL, codes, srcs, dt_ns=dt, timer=(period, 1_000_000))
            assert int(d["digest"][gid]) == orc.digest(gid) and int(d["count"][gid]) == orc.count(gid)
            assert bus.peek_window(gid).tobytes() == orc.mailbox(gid).tobytes()
        st = bus.stats()
        assert st["deliveries"] == n_subs * (n_events + n_ticks) and st["ticks"] == n_subs * n_ticks
        assert len(np.unique(d["digest"])) == n_subs          # tick records carry the owner's id: no two mailboxes alike


def test_full_size_config5_properties():
    """BASELINE config 5 at full width: 1,048,576 Zipf-masked subscribers."""
    import torch
    n_subs, n_events, B = 1_048_576, 1024, 256
    masks = tr.zipf_masks(n_subs, 1.0, 0xC0DEB205); codes = tr.zipf_codes(n_events, 1.0, 0xC0DEB206)
    srcs = (np.arange(n_events) % 4096).astype(np.uint32)
    ev = np.zeros(n_events, dtype=EVENT_DTYPE)
    ev["seq"] = np.arange(n_events); ev["code"], ev["source_id"], ev["target"] = codes, srcs, nat.TARGET_ALL
    dev = torch.from_numpy(ev.view(np.uint8).reshape(-1, 32)).cuda()
    with Bus(n_subs, ring_cap=1024, batch_cap=B, stream=torch.cuda.current_stream().cuda_stream) as bus:
        bus.subscribe_many(masks)
        for i in range(0, n_events, B):
            nat.check(bus.publish_device(dev.data_ptr() + i * 32, B, 0), "cpbus_publish_device")
        bus.sync()
        d = bus.digests(0, n_subs)
        hist = np.bincount(codes, minlength=17).astype(np.uint64)
        want_counts = np.zeros(n_subs, dtype=np.uint64)
        for c in range(17):
            want_counts += ((masks >> np.uint32(c)) & 1).astype(np.uint64) * hist[c]
        assert (d["count"] == want_counts).all()                # every mailbox's count, closed form
        for gid in (0, 5, 1023, 77_777, 1_048_575, int(np.argmax(want_counts)), int(np.argmin(want_counts))):
            orc = _oracle_for_one(gid, masks[gid], codes, srcs)
            assert int(d["digest"][gid]) == orc.digest(gid)
            assert bus.peek_window(gid).tobytes() == orc.mailbox(gid).tobytes()
        # mailboxes with equal masks must agree exactly (no per-subscriber state leaks into the records)
        order = np.argsort(masks, kind="stable")
        same = masks[order][1:] == masks[order][:-1]
        assert (d["digest"][order][1:][same] == d["digest"][order][:-1][same]).all()
        assert bus.stats()["deliveries"] == int(want_counts.sum())


def test_large_clock_jump_is_split_into_bounded_windows():
    """cpbus_advance over hundreds of timer periods: the host splits it so that no launch sees more than 32/K firings
    per slot; the mailboxes still match the oracle (which fires them one advance at a time)."""
    for K, period in ((1, 1000), (4, 700)):
        orc = ob.Oracle(6, timers_per_sub=K, keep_window=2048)
        with Bus(6, ring_cap=2048, batch_cap=256, timers_per_sub=K) as bus:
            for s in range(6):
                orc.subscribe(); bus.subscribe()
                orc.timer_add(s, period + 37 * s, 500 + s, False); bus.timer_add(s, period + 37 * s, 500 + s, False)
            orc.publish(14, 1); nat.check(bus.publish(14, 1), "publish")
            for now in (999, 250_000, 250_001, 900_000):
                assert orc.advance(now) == 0; nat.check(bus.advance(now), "advance")
                orc.publish(5, 2); nat.check(bus.publish(5, 2), "publish")
            nat.check(bus.flush(), "flush"); bus.sync()
            st = tr.compare(bus, orc, 6, window=2048)
            assert st["ticks"] > 1500


@pytest.mark.parametrize("K,period,staged", [(0, 0, False), (1, 900, False), (4, 700, False), (2, 1100, True)])
def test_oversize_device_batches_are_split(K, period, staged):
    """cpbus_publish_device with more records than batch_cap and a watermark step of hundreds of timer periods (round 1:
    CPBUS_EINVAL / CPBUS_EORDER): the library cuts the batch by size and by timer window; mailboxes equal the oracle's, which
    takes the same records event by event.  Timestamps repeat, and some coincide with due times (tick goes in front)."""
    import torch
    n_subs, B = 40, 256
    rng = np.random.default_rng(1234 + K)
    masks = np.where(rng.random(n_subs) < 0.5, nat.MASK_ALL, rng.integers(1, 1 << 17, n_subs)).astype(np.uint32)
    orc = ob.Oracle(n_subs, timers_per_sub=K, keep_window=8192)
    with Bus(n_subs, ring_cap=8192, batch_cap=B, timers_per_sub=K, stream=torch.cuda.current_stream().cuda_stream) as bus:
        for s, m in enumerate(masks):
            orc.subscribe(int(m)); bus.subscribe(int(m))
            for j in range(K):
                per = period + 13 * s + 101 * j
                orc.timer_add(s, per, 900 + 8 * s + j, j == 3); bus.timer_add(s, per, 900 + 8 * s + j, j == 3)
        seq, now, splits = 0, 0, 0
        for n, span in ((1500, 40_000), (0, 90_000), (700, 0), (300, 500), (B + 1, 1), (B, 30_000)):
            ts = np.sort(rng.integers(now, now + span + 1, n)).astype(np.uint64)
            if n > 8 and K:
                ts[n // 3] = ts[n // 3 + 1] = ((ts[n // 3] // period) + 1) * period      # an event exactly at a due time, twice
                ts = np.sort(np.minimum(ts, now + span))
            ev = np.zeros(n, dtype=EVENT_DTYPE)
            ev["seq"] = seq + np.arange(n); ev["ts_ns"] = ts
            ev["code"] = rng.integers(0, 17, n); ev["source_id"] = rng.integers(0, 50, n); ev["target"] = nat.TARGET_ALL
            seq += n; now += span
            assert orc.publish_records(ev, now) == 0
            dev = torch.from_numpy(ev.view(np.uint8).reshape(-1, 32).copy()).cuda() if n else None
            ptr = dev.data_ptr() if n else 0
            if staged:
                nat.check(bus.publish_device_staged(ptr, n, now, 0, 0), "cpbus_publish_device_staged")
            else:
                nat.check(bus.publish_device(ptr, n, now), "cpbus_publish_device")
            bus.sync()
        st = tr.compare(bus, orc, n_subs, window=8192)
        assert st["device_splits"] >= (1500 + B - 1) // B + 3 + 2 + 2
        if K:
            assert st["ticks"] > 1000
        # unsorted or beyond the watermark: refused before anything is launched
        bad = np.zeros(2 * B + 16, dtype=EVENT_DTYPE); bad["ts_ns"] = now + 10; bad["ts_ns"][7] = now + 5; bad["target"] = nat.TARGET_ALL
        d = torch.from_numpy(bad.view(np.uint8).reshape(-1, 32).copy()).cuda()
        before = bus.stats()["kernel_launches"]
        assert bus.publish_device(d.data_ptr(), 2 * B + 16, now + 10) == nat.EORDER
        assert bus.publish_device(d.data_ptr() + 8 * 32, 2 * B + 8, now + 9) == nat.EORDER
        assert bus.stats()["kernel_launches"] == before


def test_oversize_device_batch_in_lossless_mode_is_refused():
    import torch
    with Bus(4, ring_cap=1024, batch_cap=64, lossless=True, stream=torch.cuda.current_stream().cuda_stream) as bus:
        bus.subscribe()
        ev = np.zeros(65, dtype=EVENT_DTYPE); ev["target"] = nat.TARGET_ALL; ev["code"] = 3
        d = torch.from_numpy(ev.view(np.uint8).reshape(-1, 32).copy()).cuda()
        assert bus.publish_device(d.data_ptr(), 65, 0) == nat.EINVAL
        nat.check(bus.publish_device(d.data_ptr(), 64, 0), "cpbus_publish_device")
        bus.sync()
        assert len(bus.drain(0)) == 64


@pytest.mark.parametrize("seed", range(100, 116))
def test_random_mixed_traces_more_seeds(seed):
    K = (0, 1, 2, 4, 8)[seed % 5]
    ops, n_total = tr.random_ops(seed, 24, 3000, timers_per_sub=K, max_subs=40, p_filter=0.7, p_send=0.05, dt_max=9000)
    orc = tr.run_oracle(ops, 40, timers_per_sub=K)
    with Bus(40, ring_cap=4096, batch_cap=(32, 64, 256, 512)[seed % 4], timers_per_sub=K) as bus:
        tr.run_bus(bus, ops)
        tr.compare(bus, orc, n_total, window=4096)


def test_drain_many_bulk_bridge():
    """cpbus_drain_many: one kernel + two copies drain thousands of mailboxes; per-mailbox runs are FIFO and complete,
    a mailbox that does not fit stays for the next call, and draining twice returns nothing new."""
    n_subs = 3000
    rng = np.random.default_rng(77)
    masks = np.where(rng.random(n_subs) < 0.5, nat.MASK_ALL, rng.integers(0, 1 << 17, n_subs)).astype(np.uint32)
    orc = ob.Oracle(n_subs)
    with Bus(n_subs, ring_cap=256, batch_cap=128, lossless=True) as bus:
        bus.subscribe_many(masks)
        for m in masks:
            orc.subscribe(int(m))
        got = [[] for _ in range(n_subs)]
        for rnd in range(5):
            codes = rng.integers(0, 17, 100).astype(np.uint32); srcs = rng.integers(0, 30, 100).astype(np.uint32)
            orc.publish_many(codes, srcs)
            for c, s_ in zip(codes, srcs):
                nat.check(bus.publish(int(c), int(s_)), "publish")
            nat.check(bus.flush(), "flush")
            cap = 40_000 if rnd % 2 == 0 else 400_000        # the small capacity forces some mailboxes to wait for the next call
            for _ in range(40):
                recs, offs, cnts = bus.drain_many(0, n_subs, cap)
                if cnts.sum() == 0:
                    break
                for s in np.nonzero(cnts)[0]:
                    got[s].append(recs[offs[s]: offs[s] + cnts[s]].copy())
        for s in range(n_subs):
            seq = np.concatenate(got[s]) if got[s] else np.zeros(0, dtype=EVENT_DTYPE)
            assert seq.tobytes() == orc.mailbox(s).tobytes(), f"subscriber {s}"
        recs, offs, cnts = bus.drain_many(0, n_subs, 1000)
        assert cnts.sum() == 0 and bus.stats()["overwritten"] == 0
