"""Complete records and clocks at their edges, bit-exact against the CPU oracle: broadcast codes outside the enum in every
ingest path and every fan-out path, the lossless mode with such codes and mailboxes kept nearly full, timer due times
near 2^64, ids at the top of the 32-bit space and the publish ordinal after a device batch.

Rules (include/cpbus.h): a broadcast record whose code is >= CPBUS_N_CODES reaches no mailbox and is not counted per code,
but is a publish and enters the debug ring; due times saturate at "never" instead of wrapping; sub_id_base + n_max_subs
stays below CPBUS_TARGET_ALL; a device batch of n records advances the bus's publish ordinal by n."""
import numpy as np
import pytest

import oracle_binding as ob
import test_gpu_parity as parity
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from containerpilot_b200.group import GroupBus
from containerpilot_b200.sharding import LocalShardedBus

pytestmark = pytest.mark.gpu

U64 = (1 << 64) - 1
# 17..31 hit the mask word's bookkeeping bits on a kernel that shifts the raw code: 24..27 the armed-slot hint, 28 the pair
# flag, 31 the subscribed flag; >= 32 shifts out of the word
OUT = [17, 20, 23, 24, 25, 27, 28, 29, 31, 32, 1000, 0xFFFFFFFF]
FLEETS = ["dense", "dense_ticks_1", "dense_ticks_4", "dense_ticks_8", "filtered", "filtered_ticks", "unicast", "pairs"]
INGEST = ["device", "staged", "staged_next", "stream", "follow"]


def _cuda(ev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(ev).view(np.uint8).reshape(-1, 32).copy()).cuda() if len(ev) else None


def _fleet(kind, n, seed):
    """(K, masks, pairs per subscriber, [(sub, slot, period, oneshot)]).  Ticks fleets arm s % (K + 1) slots on subscriber
    s, so every value of the armed-slot hint (and each of its bits) occurs."""
    rng = np.random.default_rng(seed)
    K = int(kind.rsplit("_", 1)[1]) if kind.startswith("dense_ticks") else (2 if kind in ("filtered_ticks", "unicast") else 0)
    if kind == "pairs":
        K = 4
    masks = np.full(n, tr.MASK_ALL, dtype=np.uint32)
    if kind in ("filtered", "filtered_ticks", "unicast", "pairs"):
        masks = tr.zipf_masks(n, 1.0, seed)
        masks[::5] = tr.MASK_ALL
    pairs = [[] for _ in range(n)]
    if kind == "pairs":
        for s in range(0, n, 2):
            pairs[s] = [(int(rng.integers(1, 17)), int(rng.integers(0, 8))) for _ in range(int(rng.integers(1, 6)))]
    timers = []
    for s in range(n):
        for k in range(min(s % (K + 1), K) if K else 0):
            timers.append((s, k, int(25_000 + 997 * s + 131 * k), (s + k) % 3 == 2))
    return K, masks, pairs, timers


def _setup(bus, orc, masks, pairs, timers):
    for s, m in enumerate(masks):
        if pairs[s]:
            bus.subscribe_pairs(int(m), pairs[s]); orc.subscribe(int(m), pairs[s])
        else:
            bus.subscribe(int(m)); orc.subscribe(int(m))
    base = bus.sub_id_base
    for s, _, period, oneshot in timers:
        bus.timer_add(base + s, period, 700 + s, oneshot); orc.timer_add(base + s, period, 700 + s, oneshot)


def _batches(seed, n_subs, B, dt, unicast, base=0, first_seq=1 << 20, oversize=False):
    """(records, watermark) batches: valid codes with out-of-range ones mixed in, a batch of out-of-range codes only, a
    batch of one such record, an empty batch and (oversize) a batch of 2B + 5 records that the library has to cut."""
    rng = np.random.default_rng(seed)
    sizes = [B, int(rng.integers(1, B)), B, 1, 0, B, int(rng.integers(1, B))] + ([2 * B + 5] if oversize else []) + [B]
    out, seq, now = [], first_seq, 0
    for q, n in enumerate(sizes):
        w = now + dt
        ev = np.zeros(n, dtype=EVENT_DTYPE)
        ev["seq"] = seq + np.arange(n); seq += n
        ev["ts_ns"] = np.sort(rng.integers(now + 1, w + 1, n))
        ev["code"] = rng.integers(0, 17, n)
        odd = rng.random(n) < 0.3
        if q == 2 or q == 3:
            odd[:] = True                                  # a batch of out-of-range codes only; a batch of one
        ev["code"][odd] = rng.choice(OUT, int(odd.sum()))
        ev["source_id"] = rng.integers(0, 8, n)
        ev["target"] = nat.TARGET_ALL
        ev["flags"] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32) & ~np.uint32(3)
        if unicast:
            uni = rng.random(n) < 0.15
            ev["target"][uni] = base + rng.integers(0, n_subs, int(uni.sum()))
            ev["flags"][uni] = nat.F_UNICAST
        out.append((ev, w))
        now = w
    return out


def _expected_counts(batches, host=()):
    want = {}
    for ev, _ in batches:
        for c, s, t in zip(ev["code"], ev["source_id"], ev["target"]):
            if t == nat.TARGET_ALL and c < nat.N_CODES and c != 13:
                want[(int(c), int(s))] = want.get((int(c), int(s)), 0) + 1
    for c, s in host:
        if c != 13:
            want[(c, s)] = want.get((c, s), 0) + 1
    return want


def _compare_no_digest(bus, orc, n_subs, R):
    """tr.compare for a bus built without the digest (its digests stay 0): counts, windows, deliveries, ticks"""
    got = bus.digests(0, n_subs)
    for s in range(n_subs):
        assert int(got["count"][s]) == orc.count(s), (s, int(got["count"][s]), orc.count(s))
        o = orc.mailbox(s)[-R:]
        assert bus.peek_window(s).tobytes() == o.tobytes(), s
    st = bus.stats()
    assert (st["deliveries"], st["ticks"]) == (orc.total_deliveries(), orc.total_ticks())
    return st


def _check(bus, orc, n_subs, R, counts, publishes, base=0, digest=True):
    nat.check(bus.flush(), "flush"); bus.sync()
    st = tr.compare(bus, orc, n_subs, sub_id_base=base, window=R) if digest else _compare_no_digest(bus, orc, n_subs, R)
    assert st["published_by_code"] == [orc.published_by_code(c) for c in range(nat.N_CODES)]
    assert st["publishes"] == publishes
    assert st["overwritten"] == 0
    assert bus.publish_counts() == counts
    assert bus.debug_events().tobytes() == orc.debug_events().tobytes()
    return st


def _ingest(bus, batches, how, orc):
    """every batch through one ingest path; the oracle takes the same records"""
    devs = [_cuda(ev) for ev, _ in batches]
    import torch
    torch.cuda.synchronize()
    st = bus.stream_create(8, 1)[0] if how in ("stream", "follow") else None
    try:
        for q, (ev, w) in enumerate(batches):
            ptr = devs[q].data_ptr() if devs[q] is not None else 0
            if how == "device":
                nat.check(bus.publish_device(ptr, len(ev), w), "publish_device")
            elif how in ("staged", "staged_next"):
                nxt = q + 1 < len(batches) and how == "staged_next" and devs[q + 1] is not None and len(batches[q + 1][0]) <= bus.batch_cap
                nat.check(bus.publish_device_staged(ptr, len(ev), w, devs[q + 1].data_ptr() if nxt else 0,
                                                    len(batches[q + 1][0]) if nxt else 0), "publish_device_staged")
            else:
                rc = bus.stream_put(st, ev, w, raw=True, nowait=True)
                if rc == nat.EAGAIN:
                    bus.sync(); nat.check(bus.flush(), "flush")
                    rc = bus.stream_put(st, ev, w, raw=True, nowait=True)
                nat.check(rc, "stream_put")
                if how == "stream":
                    nat.check(bus.stream_fanout(st, len(ev), w), "stream_fanout")
                else:
                    nat.check(bus.stream_fanout_next(st), "stream_fanout_next")
            assert orc.publish_records(ev, w) == 0
        bus.sync()
        nat.check(bus.flush(), "flush")
        if st is not None:
            assert bus.stream_status(st) == nat.OK
    finally:
        if st is not None:
            bus.stream_close(st)
    del devs


def _run_codes(fleet, how, store, digest, seed):
    n, B, R, dt = 45, 64, 2048, 7_000
    K, masks, pairs, timers = _fleet(fleet, n, seed)
    orc = ob.Oracle(n, timers_per_sub=K, keep_window=R)
    with Bus(n, ring_cap=R, batch_cap=B, timers_per_sub=K, digest=digest, store_path=store) as bus:
        _setup(bus, orc, masks, pairs, timers)
        batches = _batches(seed, n, B, dt, fleet == "unicast", oversize=how in ("device", "staged"))
        _ingest(bus, batches, how, orc)
        st = _check(bus, orc, n, R, _expected_counts(batches), sum(len(ev) for ev, _ in batches), digest=digest)
        if K and fleet != "pairs":
            assert st["ticks"] > 0
        if how in ("device", "staged"):
            assert st["device_splits"] > 0


@pytest.mark.parametrize("how", INGEST)
@pytest.mark.parametrize("fleet", FLEETS)
def test_out_of_range_codes_every_ingest(fleet, how):
    """Every fan-out path (dense, dense with ticks at K = 1, 4, 8 with every armed-slot hint, the ORDERED build, the
    timers build's filtered path, the general path with unicast records, the PAIRS build) through every ingest
    (publish_device with a batch it has to split, publish_device_staged with and without a next-batch hint, RAW stream
    batches fanned out by cpbus_stream_fanout and by followers).  The hint of the empty batch names the next batch: on a
    bus with no timer armed nothing is launched for it, so nothing may be taken from the prefetch cache afterwards."""
    i = FLEETS.index(fleet) * len(INGEST) + INGEST.index(how)
    _run_codes(fleet, how, parity.STORES[i % 3], (i // 3) % 2 == 0, 100 + i)


@pytest.mark.parametrize("digest", [True, False])
@pytest.mark.parametrize("store", parity.STORES)
@pytest.mark.parametrize("fleet", FLEETS)
def test_out_of_range_codes_every_store_path(fleet, store, digest):
    _run_codes(fleet, "device", store, digest, 300 + FLEETS.index(fleet))


# ---- lossless mode: admission and fan-out must count the same records ------------------------------------------------

def _lossless_fleet(n, seed):
    """MASK_ALL and filtered masks, pair tables, and timer slots armed with a period that never comes due in the test: the
    armed-slot hint takes every value without a single tick"""
    rng = np.random.default_rng(seed)
    masks = np.where(rng.random(n) < 0.6, tr.MASK_ALL, tr.zipf_masks(n, 1.0, seed)).astype(np.uint32)
    pairs = [[(int(rng.integers(1, 17)), int(rng.integers(0, 8)))] if s % 4 == 1 else [] for s in range(n)]
    timers = [(s, k, 1 << 50, False) for s in range(n) for k in range(s % 9)]
    return masks, pairs, timers


def _drain_some(drain, orc, n, rng, base=0, most=12):
    for s in range(n):
        take = int(rng.integers(1, most))
        assert drain(base + s, take).tobytes() == orc.consume(base + s, take).tobytes(), s


def test_lossless_publish_device_never_overwrites():
    n, R, B = 27, 64, 32
    masks, pairs, timers = _lossless_fleet(n, 5)
    orc = ob.Oracle(n, timers_per_sub=8, keep_window=0, mailbox_cap=R)
    rng = np.random.default_rng(6)
    import torch
    with Bus(n, ring_cap=R, batch_cap=B, timers_per_sub=8, lossless=True) as bus:
        _setup(bus, orc, masks, pairs, timers)
        batches = _batches(7, n, B, 5_000, True)
        batches += _batches(8, n, B, 5_000, True, first_seq=1 << 30)
        now = 0
        stalls = 0
        for ev, w in batches:
            ev = ev.copy(); ev["ts_ns"] += now; w += now
            d = _cuda(ev); torch.cuda.synchronize()
            while True:
                rc = bus.publish_device(d.data_ptr() if d is not None else 0, len(ev), w)
                if rc == nat.OK:
                    break
                assert rc == nat.EAGAIN and stalls < 2000
                stalls += 1
                _drain_some(lambda s, c: bus.drain(s, cap=c), orc, n, rng)
            assert orc.publish_records(ev, w) == 0
            now = w
        assert stalls > 0
        for s in range(n):
            assert bus.drain(s, cap=R).tobytes() == orc.consume(s, R).tobytes(), s
        assert bus.stats()["overwritten"] == 0


def _stream_batches(seed, N, B, n_batches):
    out = []
    now = 0
    for q in range(0, n_batches, 9):
        for ev, w in _batches(seed + q, N, B, 3_000, True, first_seq=(q + 1) << 34):
            ev = ev.copy(); ev["ts_ns"] += now
            out.append((ev, w + now))
        now = out[-1][1]
    return out[:n_batches]


def _orc_catch_up(orc, batches, state, done, off):
    """the oracle takes record by record what the shards have delivered: batch done is at offset off"""
    while state["q"] < done or (state["q"] == done and state["i"] < off):
        ev, w = batches[state["q"]]
        if state["i"] < len(ev):
            assert orc.publish_records(ev[state["i"]:state["i"] + 1], 0) == 0
            state["i"] += 1
        if state["i"] == len(ev):
            assert orc.advance(w) == 0
            state["q"], state["i"] = state["q"] + 1, 0


@pytest.mark.parametrize("G", [1, 2])
def test_lossless_stream_admit_and_prefix_never_overwrite(G):
    """cpbus_stream_admit + cpbus_stream_fanout_prefix on G shards of one GPU (the host minimum of the shards' prefixes)"""
    N, R, B = 23, 64, 32
    masks, pairs, timers = _lossless_fleet(N, 20 + G)
    orc = ob.Oracle(N, timers_per_sub=8, keep_window=0, mailbox_cap=R)
    rng = np.random.default_rng(30 + G)
    sb = LocalShardedBus(N, [0] * G, ring_cap=R, batch_cap=B, timers_per_sub=8, stream_slots=8, lossless=True, agree="host")
    try:
        for s in range(N):
            orc.subscribe(int(masks[s]), pairs[s] or None)
        for first, count, bus in sb.shards:
            bus.subscribe_pairs_many(masks[first:first + count], pairs[first:first + count])
        for s, _, period, oneshot in timers:
            sb.bus_of(s).timer_add(s, period, 700 + s, oneshot); orc.timer_add(s, period, 700 + s, oneshot)
        batches = _stream_batches(40 + G, N, B, 18)
        state, stalls = {"q": 0, "i": 0}, 0
        for q, (ev, w) in enumerate(batches):
            nat.check(sb.put(ev, w, raw=True), "put")
            while True:
                rc = sb.fanout(len(ev), w)
                done, off, _ = sb.progress()
                _orc_catch_up(orc, batches, state, done, off)
                if rc == nat.OK:
                    assert done == q + 1
                    break
                stalls += 1
                assert stalls < 2000
                _drain_some(lambda s, c: sb.drain(s, cap=c), orc, N, rng)
        assert stalls > 0
        for s in range(N):
            assert sb.drain(s, cap=R).tobytes() == orc.consume(s, R).tobytes(), s
        for _, _, bus in sb.shards:
            assert bus.stats()["overwritten"] == 0
    finally:
        sb.close()


@pytest.mark.parametrize("G", [1, 2])
def test_lossless_stream_rounds_never_overwrite(G):
    """cpbus_stream_round_next: admission, agreement and the fan-out of the agreed prefix all on the device"""
    N, R, B = 23, 64, 32
    masks, pairs, timers = _lossless_fleet(N, 50 + G)
    orc = ob.Oracle(N, timers_per_sub=8, keep_window=0, mailbox_cap=R)
    rng = np.random.default_rng(60 + G)
    sb = LocalShardedBus(N, [0] * G, ring_cap=R, batch_cap=B, timers_per_sub=8, stream_slots=8, lossless=True, agree="device")
    try:
        for s in range(N):
            orc.subscribe(int(masks[s]), pairs[s] or None)
        for first, count, bus in sb.shards:
            bus.subscribe_pairs_many(masks[first:first + count], pairs[first:first + count])
        for s, _, period, oneshot in timers:
            sb.bus_of(s).timer_add(s, period, 700 + s, oneshot); orc.timer_add(s, period, 700 + s, oneshot)
        batches = _stream_batches(70 + G, N, B, 18)
        state = {"q": 0, "i": 0}
        for ev, w in batches[:4]:
            nat.check(sb.put(ev, w, raw=True), "put")
        put = 4

        def pump():
            nonlocal put
            while put < len(batches) and sb.put(batches[put][0], batches[put][1], raw=True) == nat.OK:
                put += 1
            done, off, _ = sb.progress()
            _orc_catch_up(orc, batches, state, done, off)
            _drain_some(lambda s, c: sb.drain(s, cap=c), orc, N, rng, most=6)

        rounds = sb.run_rounds(len(batches), pump=pump, depth=2)
        assert put == len(batches) and rounds > len(batches)
        done, off, _ = sb.progress()
        _orc_catch_up(orc, batches, state, done, off)
        for s in range(N):
            assert sb.drain(s, cap=R).tobytes() == orc.consume(s, R).tobytes(), s
        for _, _, bus in sb.shards:
            assert bus.stats()["overwritten"] == 0
    finally:
        sb.close()


# ---- clocks near 2^64 ---------------------------------------------------------------------------------------------------

PERIODS = [1, 977, (1 << 31) + 1, 1 << 62, (1 << 63) - 1, U64]


@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("K", [1, 2, 8])
@pytest.mark.parametrize("T0", [(1 << 32) + 7, 1 << 62, (1 << 63) - 1, (1 << 64) - (1 << 40)])
def test_clocks_near_the_top(T0, K, path):
    """Three phases, each arming every slot at its start and cancelling every timer at its end (the cancels must find the
    same armed timers on both sides: a saturated due time stays armed, a fired one-shot is gone).  Phase 1 arms every
    period, one-shot and periodic, at T0 and steps the clock ~1,000 ns with records at tick due times; phase 2 arms
    periods from 2^31 + 1 and steps 2^33 ns; phase 3 arms periods from 2^62 and jumps to the top: records with ts up to
    2^64 - 2, a final watermark of UINT64_MAX.  Device records carry seq >= 2^32 and arbitrary flags.  Due-time sums
    that pass 2^64 - 2 never fire."""
    n, R, B = 12, 4096, 64
    rng = np.random.default_rng(T0 % 1000 + 10 * K + (path == "device"))
    orc = ob.Oracle(n, timers_per_sub=K, keep_window=R)
    import torch
    with Bus(n, ring_cap=R, batch_cap=B, timers_per_sub=K) as bus:
        for s in range(n):
            bus.subscribe(tr.MASK_ALL if s % 3 else 0x00FF); orc.subscribe(tr.MASK_ALL if s % 3 else 0x00FF)
        nat.check(bus.advance(T0), "advance"); assert orc.advance(T0) == 0
        seq, pubs, fired = 1 << 33, 0, 0
        state = {"now": T0}

        def arm(periods):
            out = []
            for s in range(n):
                for k in range(K):
                    period, oneshot = periods[(s + k) % len(periods)], (s // 6 + k) % 2 == 1
                    out.append((bus.timer_add(s, period, 100 * s + k, oneshot), orc.timer_add(s, period, 100 * s + k, oneshot)))
            return out

        def cancel_all(handles):
            armed = 0
            for hb, ho in handles:
                rc_o = orc.timer_cancel(ho)
                rc_b = bus._lib.cpbus_timer_cancel(bus._h, hb)
                assert rc_b == rc_o, (rc_b, rc_o)
                armed += rc_o == 0
            assert bus.stats()["n_timers"] == 0
            return armed

        def step(w, ts_list):
            nonlocal seq, pubs
            ts_list = sorted({t for t in ts_list if state["now"] <= t <= w})
            if path == "host":
                for t in ts_list:
                    nat.check(bus.advance(t), "advance"); assert orc.advance(t) == 0
                    c, src = int(rng.integers(0, 17)), int(rng.integers(0, 4))
                    nat.check(bus.publish(c, src), "publish"); assert orc.publish(c, src) == 0
                    pubs += 1
                nat.check(bus.advance(w), "advance"); assert orc.advance(w) == 0
                nat.check(bus.flush(), "flush")
            else:
                ev = np.zeros(len(ts_list), dtype=EVENT_DTYPE)
                ev["seq"] = seq + 3 * np.arange(len(ev)); seq += 3 * len(ev)
                ev["ts_ns"] = np.array(ts_list, dtype=np.uint64)
                ev["code"] = rng.integers(0, 17, len(ev)); ev["source_id"] = rng.integers(0, 4, len(ev))
                ev["target"] = nat.TARGET_ALL
                ev["flags"] = rng.integers(0, 1 << 32, len(ev), dtype=np.uint64).astype(np.uint32)
                d = _cuda(ev); torch.cuda.synchronize()
                nat.check(bus.publish_device(d.data_ptr() if d is not None else 0, len(ev), w), "publish_device")
                assert orc.publish_records(ev, w) == 0
                pubs += len(ev)
                bus.sync()
            state["now"] = w

        # phase 1: every period, ~1,000 ns; records at the due times of the 977 ns timers
        handles = arm(PERIODS)
        for _ in range(40):
            now = state["now"]
            w = now + int(rng.integers(1, 50))
            step(w, [now + 1, w, T0 + 977, T0 + 2 * 977] + [now + int(x) for x in rng.integers(0, w - now + 1, 2)])
        saturated = cancel_all(handles)
        # phase 2: from 2^31 + 1, 2^33 ns
        t1 = state["now"]
        handles = arm(PERIODS[2:])
        p31 = (1 << 31) + 1
        for w in (t1 + p31 - 1, t1 + 2 * p31, t1 + (1 << 33) + 5):
            step(w, [t1 + p31, t1 + 2 * p31, w])
        cancel_all(handles)
        # phase 3: from 2^62, up to UINT64_MAX
        t2 = state["now"]
        handles = arm(PERIODS[3:])
        tops = sorted({min(U64, max(t2 + 1, c)) for c in (t2 + (1 << 62), (1 << 63) + 10, U64 - 2, U64 - 1, U64)})
        for w in tops:
            step(w, [min(w, U64 - 1), t2 + (1 << 62), t2 + (1 << 63) - 1, t2 + 3 * (1 << 62)])
        nat.check(bus.flush(), "flush"); bus.sync()
        st = tr.compare(bus, orc, n, window=R)
        assert st["now_ns"] == U64 and st["publishes"] == pubs and st["ticks"] > 0
        assert saturated > 0
        cancel_all(handles)


# ---- ids at the top of the 32-bit space --------------------------------------------------------------------------------

def test_last_gid_below_target_all():
    """sub_id_base puts the last gid at 0xFFFFFFFE: a send to it, a device unicast record to it and broadcasts reach exactly
    the mailboxes they should."""
    n, base, R = 4, 0xFFFFFFFF - 4, 256
    orc = ob.Oracle(n, keep_window=R, sub_id_base=base)
    import torch
    with Bus(n, ring_cap=R, batch_cap=64, sub_id_base=base) as bus:
        ids = [bus.subscribe() for _ in range(n)]
        for _ in range(n):
            orc.subscribe()
        assert ids[-1] == 0xFFFFFFFE
        nat.check(bus.publish(3, 1), "publish"); assert orc.publish(3, 1) == 0
        nat.check(bus.send(ids[-1], 5, 2), "send"); assert orc.receive(ids[-1], 5, 2) == 0
        nat.check(bus.flush(), "flush")
        ev = np.zeros(3, dtype=EVENT_DTYPE)
        ev["seq"] = [10, 11, 12]; ev["ts_ns"] = [5, 6, 7]; ev["code"] = [7, 9, 31]; ev["source_id"] = [4, 4, 4]
        ev["target"] = [ids[-1], nat.TARGET_ALL, ids[-1]]; ev["flags"] = [nat.F_UNICAST, 0, nat.F_UNICAST]
        d = _cuda(ev); torch.cuda.synchronize()
        nat.check(bus.publish_device(d.data_ptr(), 3, 10), "publish_device"); assert orc.publish_records(ev, 10) == 0
        nat.check(bus.send(ids[0], 6, 2), "send"); assert orc.receive(ids[0], 6, 2) == 0
        nat.check(bus.flush(), "flush"); bus.sync()
        tr.compare(bus, orc, n, sub_id_base=base, window=R)
        assert [int(x) for x in bus.peek_window(ids[-1])["code"]] == [3, 5, 7, 9, 31]
        assert [int(x) for x in bus.peek_window(ids[1])["code"]] == [3, 9]


@pytest.mark.parametrize("base,n", [(0xFFFFFFFF - 3, 4), (0xFFFFFFFF, 1), (0xFFFFFFF0, 64), (0xFFFFF000, 0x1001)])
def test_ids_that_reach_target_all_are_refused(base, n):
    for make in (lambda: Bus(n, ring_cap=64, batch_cap=32, sub_id_base=base),
                 lambda: GroupBus(n, [0], ring_cap=64, batch_cap=32, sub_id_base=base)):
        with pytest.raises(nat.CpbusError) as e:
            make()
        assert e.value.status == nat.EINVAL


# ---- the publish ordinal after a device batch ---------------------------------------------------------------------------

@pytest.mark.parametrize("how", ["device", "stream"])
def test_seq_after_a_device_batch_counts_its_records(how):
    """The records' seqs do not continue the host's (2^40 and 5 below it); the next host publish and send carry the
    previous ordinal + the batch's record count."""
    n, R = 3, 256
    orc = ob.Oracle(n, keep_window=R)
    with Bus(n, ring_cap=R, batch_cap=64) as bus:
        for _ in range(n):
            bus.subscribe(); orc.subscribe()
        for c in (1, 2):
            nat.check(bus.publish(c, 1), "publish"); assert orc.publish(c, 1) == 0
        nat.check(bus.flush(), "flush")
        ev = np.zeros(4, dtype=EVENT_DTYPE)
        ev["seq"] = [1 << 40, 5, 4, 3]; ev["ts_ns"] = [1, 2, 3, 4]; ev["code"] = [3, 4, 5, 6]
        ev["target"] = [nat.TARGET_ALL, nat.TARGET_ALL, 1, nat.TARGET_ALL]; ev["flags"][2] = nat.F_UNICAST
        batches = [(ev, 10)]
        _ingest(bus, batches, how, orc)
        nat.check(bus.advance(20), "advance"); assert orc.advance(20) == 0
        nat.check(bus.publish(7, 1), "publish"); assert orc.publish(7, 1) == 0
        nat.check(bus.send(2, 8, 1), "send"); assert orc.receive(2, 8, 1) == 0
        _check(bus, orc, n, R, _expected_counts(batches, [(1, 1), (2, 1), (7, 1)]), 8)
        assert [int(x) for x in bus.peek_window(2)["seq"]] == [0, 1, 1 << 40, 5, 3, 6, 7]
