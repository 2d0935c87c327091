"""Whole-fleet ring parity at the scale the library is measured at: 1,048,576 subscribers, 1,024-record rings, 256-record
batches, about 1,536 records so that every dense ring wraps inside a batch.  Every mailbox's tail and every ring slot the
records reach are compared with the plain reference of `tests/ring_check.py`; the reference itself is pinned to the C
oracle on sampled mailboxes.  Each fleet reaches a geometry that only happens at this scale: computed multi-round staging
at 16 mailboxes per warp (plain build), control blocks and timer slots past the L2-hint limit (96 MiB of hot state at
K = 2), and a paired fleet whose warps walk two or more triage blocks."""
import ctypes as C

import numpy as np
import pytest

import oracle_binding as ob
import ring_check as rc
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200 import events as ev
from containerpilot_b200 import masks as cpm
from containerpilot_b200.bus import Bus, EVENT_DTYPE

pytestmark = pytest.mark.gpu
N, B, R, E, DT = 1 << 20, 256, 1024, 1536, 10_000
PIN = (0, 1, 31, 3000, 4096 + 3000, 65_535, 524_288, 700_001, N - 1)


def _records(codes, srcs, targets=None, dt=DT):
    rec = np.zeros(len(codes), dtype=EVENT_DTYPE)
    rec["seq"], rec["ts_ns"] = np.arange(len(codes)), (np.arange(len(codes)) + 1) * dt
    rec["code"], rec["source_id"], rec["target"] = codes, srcs, nat.TARGET_ALL
    if targets is not None:
        uni = targets != nat.TARGET_ALL
        rec["target"][uni], rec["flags"][uni] = targets[uni], nat.F_UNICAST
    return rec


def _publish(bus, rec, staged=False):
    """cpbus_publish_device[_staged] in batches of B, each with the watermark of its last record: [(first, end, watermark)]"""
    import torch
    dev = torch.from_numpy(rec.view(np.uint8).reshape(-1, 32).copy()).cuda()
    batches = []
    for i in range(0, len(rec), B):
        j = min(len(rec), i + B)
        w = int(rec["ts_ns"][j - 1])
        if staged:   # hint the next batch, the one after it, or nothing: pull-now and prefetched batches both occur
            d = (1, 2, 0)[(i // B) % 3]
            nxt = dev.data_ptr() + (i + d * B) * 32 if d and i + d * B < len(rec) else 0
            nat.check(bus.publish_device_staged(dev.data_ptr() + i * 32, j - i, w, nxt, B if nxt else 0), "publish_device_staged")
        else:
            nat.check(bus.publish_device(dev.data_ptr() + i * 32, j - i, w), "publish_device")
        batches.append((i, j, w))
    bus.sync()
    return batches


def _bus(store, K=0, **kw):
    import torch
    return Bus(N, ring_cap=R, batch_cap=B, timers_per_sub=K, store_path=store, stream=torch.cuda.current_stream().cuda_stream, **kw)


def _check(bus, model, pin=PIN):
    model.pin(pin)
    with rc.fleet_views(bus.device_ptrs(), N, R) as views:
        assert rc.check(views, model) > 0


@pytest.mark.parametrize("store,staged", [(nat.STORE_V4, False), (nat.STORE_V8, False), (nat.STORE_BULK, False),
                                          (nat.STORE_BULK, True)])
def test_dense_fleet(store, staged):
    """all-ones masks, no timers: the plain build's dense run at 16 mailboxes per warp, staged in several rounds"""
    rng = np.random.default_rng(0xF1EE7 + store)
    rec = _records(rng.integers(1, 17, E), rng.integers(0, 4096, E))
    masks = np.full(N, nat.MASK_ALL, dtype=np.uint32)
    with _bus(store) as bus:
        bus.subscribe_many(masks)
        _check(bus, rc.FleetModel(N, R, rec, _publish(bus, rec, staged), masks))


@pytest.mark.parametrize("store", [nat.STORE_V4, nat.STORE_V8, nat.STORE_BULK])
def test_dense_fleet_with_ticks(store):
    """BASELINE config 3: one 1 kHz timer per subscriber, ticks interleaved with the dense runs"""
    rng = np.random.default_rng(0xC0DEB203)
    rec = _records(rng.integers(1, 17, E), rng.integers(0, 4096, E))
    masks = np.full(N, nat.MASK_ALL, dtype=np.uint32)
    timers = [{"period": np.full(N, 1_000_000, dtype=np.uint64), "source": (1_000_000 + np.arange(N)).astype(np.uint32),
               "oneshot": False}]
    with _bus(store, K=1) as bus:
        bus.subscribe_many(masks)
        bus.timer_add_many(0, N, 1_000_000, source_id0=1_000_000)
        _check(bus, rc.FleetModel(N, R, rec, _publish(bus, rec), masks, timers=timers))
        assert bus.stats()["ticks"] == N * (E * DT // 1_000_000)


@pytest.mark.parametrize("store", [nat.STORE_V8, nat.STORE_BULK])
def test_zipf_fleet(store):
    """BASELINE config 5: Zipf masks and codes, no timers (the mask-ordered build)"""
    masks = tr.zipf_masks(N, 1.0, 0xC0DEB205)
    rec = _records(tr.zipf_codes(E, 1.0, 0xC0DEB206), np.arange(E) % 4096)
    with _bus(store) as bus:
        bus.subscribe_many(masks)
        model = rc.FleetModel(N, R, rec, _publish(bus, rec), masks)
        _check(bus, model, PIN + (int(np.argmax(masks)), int(np.argmin(masks))))


def test_zipf_fleet_two_timers_and_unicast():
    """Zipf masks, a periodic and a one-shot timer per subscriber and unicast records for a few thousand mailboxes: the
    general path, with 96 MiB of control blocks and timer slots (past the evict_last limit)"""
    rng = np.random.default_rng(0x2F1EE7)
    n_uni = 2048
    masks = tr.zipf_masks(N, 1.0, 0xC0DEB207)
    codes = np.concatenate([tr.zipf_codes(E, 1.0, 0xC0DEB208), rng.integers(0, 17, n_uni)])
    targets = np.concatenate([np.full(E, nat.TARGET_ALL, dtype=np.int64), rng.choice(N, n_uni, replace=False)])
    order = rng.permutation(len(codes))
    rec = _records(codes[order], rng.integers(0, 4096, len(codes)), targets[order], dt=4_000)
    gid = np.arange(N)
    timers = [{"period": (900_000 + (gid % 1009) * 997).astype(np.uint64), "source": (2_000_000 + gid).astype(np.uint32),
               "oneshot": False},
              {"period": (2_500_000 + (gid % 7919) * 1531).astype(np.uint64), "source": (5_000_000 + gid).astype(np.uint32),
               "oneshot": True}]
    with _bus(nat.STORE_V8, K=2) as bus:
        bus.subscribe_many(masks)
        ids = np.concatenate([gid, gid])
        _, status = bus.timer_add_list(ids, np.concatenate([t["period"] for t in timers]),
                                       np.concatenate([t["source"] for t in timers]),
                                       np.concatenate([np.zeros(N, dtype=bool), np.ones(N, dtype=bool)]))
        assert (status == nat.OK).all()
        model = rc.FleetModel(N, R, rec, _publish(bus, rec), masks, timers=timers)
        hit = rec["target"][rec["target"] != nat.TARGET_ALL][:3]
        _check(bus, model, PIN + tuple(int(g) for g in hit))


def _job_shapes(n_jobs=256):
    """Job-shaped {mask, cases} (their own switches), a Metric consumer and an unfiltered one: (masks, rows, n_sources)"""
    names = ["", "global", "closed", "SIGHUP", "SIGUSR2"]
    for j in range(n_jobs):
        names += [f"job{j}", f"check.job{j}", f"job{j}.heartbeat", f"job{j}.run-every", f"job{j}.wait-timeout"]
    src_id = {s: i for i, s in enumerate(names)}
    shapes = []
    for j in range(n_jobs):
        start = ev.Event(ev.ExitSuccess, f"job{(j * 7) % 32}") if j % 3 else ev.GlobalStartup
        shapes.append(cpm.JobSwitch(f"job{j}", start_event=start).cases())
    shapes += [cpm.MetricSwitch().cases(), (nat.MASK_ALL, [])]
    masks = np.array([m for m, _ in shapes], dtype=np.uint32)
    rows = np.full((len(shapes), 16, 2), 0xFFFFFFFF, dtype=np.uint32)
    for i, (_, cases) in enumerate(shapes):
        for k, e in enumerate(cases):
            rows[i, k] = (e.Code, src_id[e.Source])
    return masks, rows, len(names)


@pytest.mark.parametrize("store", [nat.STORE_V8, nat.STORE_BULK])
def test_paired_fleet(store):
    """about 1M subscribers drawn from a few hundred Job-shaped shapes (cpbus_subscribe_pairs_many): the grid is capped at
    16 CTAs per SM, so every warp walks two or more blocks of 32 mailboxes in the triage loop"""
    rng = np.random.default_rng(0xFA1125)
    shape_masks, shape_rows, n_names = _job_shapes()
    S = len(shape_masks)
    p = np.full(S, 0.94 / (S - 2)); p[-2], p[-1] = 0.05, 0.01
    shape_of = rng.choice(S, N, p=p)
    masks, rows = shape_masks[shape_of], np.ascontiguousarray(shape_rows[shape_of])
    cnt = (rows[:, :, 0] != 0xFFFFFFFF).sum(1).astype(np.uint32)
    # sources biased towards the first jobs' names, so that their dependants' exact cases match now and then
    srcs = np.where(rng.random(E) < 0.7, rng.integers(0, 5 + 5 * 32, E), rng.integers(0, n_names, E))
    rec = _records(rng.integers(1, 17, E), srcs)
    with _bus(store) as bus:
        first = C.c_uint32()
        nat.check(bus._lib.cpbus_subscribe_pairs_many(bus._h, masks.ctypes.data, rows.ctypes.data, cnt.ctypes.data, N,
                                                      C.byref(first)), "cpbus_subscribe_pairs_many")
        assert first.value == 0
        model = rc.FleetModel(N, R, rec, _publish(bus, rec), masks, shape_rows, shape_of)
        _check(bus, model, PIN + tuple(int(np.flatnonzero(shape_of == s)[0]) for s in (0, 1, 2, S - 2, S - 1)))


def test_sparse_record_flushes():
    """CPBUS_CFG_SPARSE_RECORDS: flushes that reach at most 1,024 mailboxes go through the record kernel, interleaved with
    full flushes that wrap every ring; host publishes and direct sends, stamped by the bus clock"""
    rng = np.random.default_rng(0x5BA75E)
    gid = np.arange(N)
    masks = np.full(N, 0b11110, dtype=np.uint32)                         # codes 1-4: every mailbox
    masks[gid % 2039 == 5] |= 1 << 15                                    # ~514 mailboxes
    masks[gid % 1531 == 7] |= 1 << 16                                    # ~685 mailboxes
    recs, batches, now, sparse = [], [], 0, 0

    def put(code, src, target=nat.TARGET_ALL):
        recs.append((len(recs), now, code, src, target, 0 if target == nat.TARGET_ALL else nat.F_UNICAST))

    with _bus(nat.STORE_V8, sparse_records=True) as bus:
        bus.subscribe_many(masks)
        for step in range(6):
            for k in range(4):
                now += 1_000
                nat.check(bus.advance(now), "advance")
                first = len(recs)
                for _ in range(5):
                    src = int(rng.integers(0, 64))
                    nat.check(bus.publish(15 + k % 2, src), "publish"); put(15 + k % 2, src)
                for g in rng.integers(0, N, 3):
                    code, src = int(rng.integers(0, 17)), int(rng.integers(0, 64))
                    nat.check(bus.send(int(g), code, src), "send"); put(code, src, int(g))
                before = bus.stats()
                nat.check(bus.flush(), "flush")
                after = bus.stats()
                assert after["batches"] == before["batches"] and after["kernel_launches"] > before["kernel_launches"]
                sparse += 1
                batches.append((first, len(recs), now))
            now += 1_000
            nat.check(bus.advance(now), "advance")
            first = len(recs)
            codes, srcs = rng.integers(1, 5, B), rng.integers(0, 4096, B)
            e = np.zeros(B, dtype=EVENT_DTYPE)
            e["code"], e["source_id"] = codes, srcs
            nat.check(bus.publish_many(e), "publish")
            for c, s in zip(codes, srcs):
                put(int(c), int(s))
            nat.check(bus.flush(), "flush")
            batches.append((first, len(recs), now))
        bus.sync()
        rec = np.array(recs, dtype=[(n, EVENT_DTYPE[n]) for n in EVENT_DTYPE.names]).astype(EVENT_DTYPE)
        model = rc.FleetModel(N, R, rec, batches, masks)
        uni = [int(r["target"]) for r in rec if r["target"] != nat.TARGET_ALL][:3]
        _check(bus, model, PIN + (5, 7, 2039 + 5, 1531 + 7) + tuple(uni))
    assert sparse == 24


def test_checker_names_a_flipped_word():
    """the checker on a small bus: it passes, then one ring word flipped through the view is named by mailbox, slot and
    word — and the oracle compare of tests/trace.py catches the same flip"""
    n, r = 300, 512   # a ring holds at least two batches
    rng = np.random.default_rng(0x5E1F)
    masks = np.where(rng.random(n) < 0.5, nat.MASK_ALL, rng.integers(0, 1 << 17, n)).astype(np.uint32)
    rec = _records(rng.integers(0, 17, 1500), rng.integers(0, 64, 1500))
    timers = [{"period": (40_000 + 977 * np.arange(n)).astype(np.uint64), "source": (100 + np.arange(n)).astype(np.uint32),
               "oneshot": False}]
    import torch
    with Bus(n, ring_cap=r, batch_cap=B, timers_per_sub=1, stream=torch.cuda.current_stream().cuda_stream) as bus:
        bus.subscribe_many(masks)
        bus.timer_add_list(np.arange(n), timers[0]["period"], timers[0]["source"])
        model = rc.FleetModel(n, r, rec, _publish(bus, rec), masks, timers=timers)
        orc = ob.Oracle(n, timers_per_sub=1, keep_window=r)
        for s in range(n):
            orc.subscribe(int(masks[s])); orc.timer_add(s, int(timers[0]["period"][s]), int(timers[0]["source"][s]))
        for a, b, w in model.batches:
            assert orc.publish_records(rec[a:b], w) == 0
        model.pin(range(n))
        tr.compare(bus, orc, n, window=r)
        with rc.fleet_views(bus.device_ptrs(), n, r) as (ring, ctl):
            assert rc.check((ring, ctl), model) == int(np.minimum([orc.count(s) for s in range(n)], r).sum())
            gid = 137
            slot = (int(ctl[gid, 0]) - 1) & (r - 1)                        # the newest record
            ring[gid, slot, 2] ^= 1 << 40                                    # one bit of its source_id
            torch.cuda.synchronize()
            with pytest.raises(AssertionError, match=f"mailbox {gid} slot {slot} word 2:"):
                rc.check((ring, ctl), model)
            with pytest.raises(AssertionError, match=f"mailbox mismatch at subscriber {gid}"):
                tr.compare(bus, orc, n, window=r)
