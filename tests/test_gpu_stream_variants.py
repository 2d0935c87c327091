"""Stream followers, lossless device rounds and host-agreed prefixes on every store path and every fan-out build, checked
on the rings themselves.

The fan-out body compiles three times: `fanout_kernel`, `fanout_follow_kernel` (cpbus_stream_fanout_next) and
`fanout_round_kernel` (cpbus_stream_round_next), each for 3 store paths and 8 builds.  A follower or a round takes n and
the watermark from the slot header or RoundDev rather than from its launch, is sized for batch_cap, always stages the
batch through the lead CTA's copy, and a round reads its records at an offset into the slot.  A mailbox's digest is
computed from the staged batch, so a store that puts a record in the wrong slot or with its halves swapped leaves counts
and digests right: every cell here compares every tail and every written ring slot of every shard with the plain
reference of `ring_check.py`, and every mailbox with the C oracle.

A cell is one ingest kind x one store x one build:
  follow   cpbus_stream_fanout_next, the publisher 0 and then 3 batches ahead (batches from the slot and from the prefetch
           buffer);
  round    cpbus_stream_round_next through LocalShardedBus(lossless=True, agree="device").run_rounds;
  prefix   cpbus_stream_admit + cpbus_stream_fanout_prefix (agree="host"): the plain kernel launched with stream_off > 0.
In the lossless kinds one all-ones mailbox (D) is never drained except by exactly the records that admit the prefix the
cell wants, so rounds stop at chosen offsets (odd ones, ones that are not a multiple of 32, one record short of the end)
and the round after each cut stalls; every other mailbox is drained around it.  Each cell also runs under torch.profiler
and asserts that the fan-out kernels that ran are exactly the instantiation it names, so a cell whose fleet takes another
build fails instead of passing vacuously.  `test_every_follower_and_round_kernel_has_a_cell` (no GPU) holds the matrix to
what the library compiles."""
import contextlib
import os
import re
import subprocess

import numpy as np
import pytest

import oracle_binding as ob
import ring_check as rc
import test_gpu_fleet_rings as fleet_rings
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import EVENT_DTYPE
from containerpilot_b200.sharding import LocalShardedBus
from test_gpu_record_edges import _compare_no_digest

KINDS = ("follow", "round", "prefix")
STORES = (nat.STORE_V4, nat.STORE_V8, nat.STORE_BULK)
BUILDS = ("dense", "timers", "ordered", "pairs")
KERNEL = {"follow": "fanout_follow_kernel", "round": "fanout_round_kernel", "prefix": "fanout_kernel"}
FANOUT = re.compile(r"fanout_(?:follow_|round_)?kernel<[^>]*>")

G, R, DT = 2, 1024, 20_000
D = 5                                                    # the designated all-ones mailbox (global id, on shard 0)
NEVER = 1 << 50                                          # D's timer period: armed, never due in a cell
# batch b's length for batch_cap B; D (which takes every broadcast record) is full before batch 11
SIZES = lambda B: [B, 1, 31, 0, 32, 33, 255, B, B, B, 0, 256, 129, 97]
CUTS = {11: (77, 160, 255), 12: (1,), 13: (33,)}         # where lossless rounds must stop, as offsets into the batch


def kernel_name(kind, store, build, digest):
    """the fan-out instantiation a cell runs: <STORE, TIMERS, DIGEST, ORDERED, PAIRS> (cpbus.cu, launch_fanout)"""
    flags = (build in ("timers", "pairs"), digest, build == "ordered", build == "pairs")
    return f"{KERNEL[kind]}<{store}, " + ", ".join("true" if f else "false" for f in flags) + ">"


def _compiled_stream_kernels():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    tool = os.path.join(os.path.dirname(os.path.realpath(nvcc)), "cuobjdump")
    out = subprocess.run([tool, "-symbols", nat.LIB_PATH], capture_output=True, text=True, check=True).stdout
    pat = re.compile(r"(fanout_(?:follow|round)_kernel)ILi(\d+)ELb([01])ELb([01])ELb([01])ELb([01])EE")
    return {f"{m[0]}<{m[1]}, " + ", ".join("true" if b == "1" else "false" for b in m[2:]) + ">" for m in pat.findall(out)}


def test_every_follower_and_round_kernel_has_a_cell():
    """the follower and round instantiations in libcpbus.so are exactly the ones the matrix below runs"""
    compiled = _compiled_stream_kernels()
    cells = {kernel_name(k, s, b, d) for k in ("follow", "round") for s in STORES for b in BUILDS for d in (True, False)}
    assert len(cells) == 48
    assert compiled == cells, (sorted(compiled - cells), sorted(cells - compiled))


# ---- fleets and batches ------------------------------------------------------------------------------------------------

def _devices(g):
    import torch
    nd = torch.cuda.device_count()
    return [i % nd for i in range(g)]


class _Fleet:
    """masks, optional Job-shaped pair tables (shape rows + shape of each subscriber) and timer slots of n subscribers"""

    def __init__(self, build, n, seed, K=2):
        rng = np.random.default_rng(seed)
        gid = np.arange(n)
        self.build, self.n, self.rows, self.shape_of, self.timers, self.n_sources = build, n, None, None, [], 64
        if build == "dense":
            self.masks = np.full(n, nat.MASK_ALL, dtype=np.uint32)
        elif build == "timers":
            self.masks = tr.zipf_masks(n, 1.0, seed)
            for k in range(K):                  # even slots periodic, odd slots one-shot
                oneshot = k % 2 == 1
                period = ((60_000 + ((gid * 7 + k * 13) % 89) * 2_203) if oneshot
                          else (12_000 + ((gid * 5 + k * 11) % 97) * 331)).astype(np.uint64)
                period[D] = NEVER
                self.timers.append({"period": period, "source": (100_000 * (k + 1) + gid).astype(np.uint32),
                                    "oneshot": oneshot})
        elif build == "ordered":
            self.masks = tr.zipf_masks(n, 1.0, seed)
            self.masks[::5] = nat.MASK_ALL
        else:
            shape_masks, self.rows, self.n_sources = fleet_rings._job_shapes()
            self.shape_of = rng.integers(0, len(shape_masks), n)
            self.shape_of[D] = len(shape_masks) - 1          # the unfiltered shape: all ones, no cases
            self.masks = shape_masks[self.shape_of]
        self.masks = np.asarray(self.masks, dtype=np.uint32)
        self.masks[D] = nat.MASK_ALL
        self.K = len(self.timers)

    def pairs(self, i):
        if self.rows is None:
            return []
        return [(int(c), int(s)) for c, s in self.rows[self.shape_of[i]] if c != 0xFFFFFFFF]

    def populate(self, sb):
        for first, count, bus in sb.shards:
            if self.rows is None:
                bus.subscribe_many(self.masks[first:first + count])
            else:
                bus.subscribe_pairs_many(self.masks[first:first + count], [self.pairs(i) for i in range(first, first + count)])
            if self.timers:
                ids = np.arange(first, first + count)
                _, status = bus.timer_add_list(np.tile(ids, self.K),
                                               np.concatenate([t["period"][first:first + count] for t in self.timers]),
                                               np.concatenate([t["source"][first:first + count] for t in self.timers]),
                                               np.repeat([t["oneshot"] for t in self.timers], count))
                assert (status == nat.OK).all()

    def model(self, first, count, rec, spans):
        sl = slice(first, first + count)
        timers = [{"period": t["period"][sl], "source": t["source"][sl], "oneshot": t["oneshot"]} for t in self.timers]
        return rc.FleetModel(count, R, rec, spans, self.masks[sl], self.rows,
                             None if self.shape_of is None else self.shape_of[sl], timers, sub_id_base=first)

    def oracle(self, first, count, batches):
        orc = ob.Oracle(count, timers_per_sub=self.K, keep_window=R, sub_id_base=first)
        for i in range(first, first + count):
            orc.subscribe(int(self.masks[i]), self.pairs(i) or None)
        for t in self.timers:
            for i in range(first, first + count):
                orc.timer_add(i, int(t["period"][i]), int(t["source"][i]), t["oneshot"])
        for ev, w in batches:
            assert orc.publish_records(ev, w) == 0
        return orc


def _batches(fl, B, seed, cuts):
    """RAW batches of SIZES(B) records: explicit seq, ts in (w - DT, w] in clock order, watermark w = (q + 1) DT.  The
    timers build carries unicast records to either shard (never to D); the record at each cut is a broadcast, so D stops
    the admitted prefix exactly there.  Paired fleets draw sources biased towards the first jobs' names."""
    rng = np.random.default_rng(seed)
    out, seq = [], 1 << 36
    for q, m in enumerate(SIZES(B)):
        w = (q + 1) * DT
        ev = np.zeros(m, dtype=EVENT_DTYPE)
        ev["seq"] = seq + np.arange(m); seq += m
        ev["ts_ns"] = np.sort(rng.integers(w - DT + 1, w + 1, m))
        ev["code"] = rng.integers(0, 17, m)
        ev["source_id"] = (np.where(rng.random(m) < 0.7, rng.integers(0, 5 + 5 * 32, m), rng.integers(0, fl.n_sources, m))
                           if fl.rows is not None else rng.integers(0, fl.n_sources, m))
        ev["target"] = nat.TARGET_ALL
        if fl.build == "timers":
            uni = rng.random(m) < 0.15
            uni[[c for c in cuts.get(q, ()) if c < m]] = False
            to = rng.integers(0, fl.n - 1, int(uni.sum()))
            ev["target"][uni] = to + (to >= D)
            ev["flags"][uni] = nat.F_UNICAST
        out.append((ev, w))
    return out


# ---- drivers -----------------------------------------------------------------------------------------------------------

def _put(sb, ev, w):
    rc_ = sb.put(ev, w, raw=True)
    if rc_ == nat.EAGAIN:                                # the slot's previous batch is still being fanned out
        sb.sync()
        rc_ = sb.put(ev, w, raw=True)
    nat.check(rc_, "put")


def _follow(sb, batches):
    """followers on every shard; the publisher puts each batch just before its followers, then runs 3 batches ahead"""
    T, put = len(batches), 0
    for q in range(T):
        while put < min(T, q + 1 + (0 if q < T // 2 else 3)):
            _put(sb, *batches[put]); put += 1
        for g in range(sb.world):
            sb.follow(g)
    assert sb.progress()[:2] == (T, 0)


class _Cutter:
    """Lossless rounds that stop where the cell says.  Before each round every mailbox but D is drained (drain_many below D
    and on the other shard, drain_ready above D); D is drained by exactly the records it needs for the next segment: all
    of the batch's remainder, or up to the next cut, where D has to be full so that the first record it cannot take is
    the cut.  The round after a cut finds D full and stalls."""

    def __init__(self, sb, batches, cuts):
        self.sb, self.batches, self.cuts = sb, batches, cuts
        self.d_bus, self.d_head = sb.bus_of(D), 0
        self.expect, self.after_cut, self.n_cuts, self.n_stalls = (0, 0), False, 0, 0

    def _drain_others(self):
        for first, count, bus in self.sb.shards:
            if first <= D < first + count:
                lo, hi = D - first, first + count - D - 1
                if lo:
                    bus.drain_many(first, lo, lo * R)
                if hi:
                    _, ready, _ = bus.drain_ready(D + 1, hi, D + 1, hi * R, hi)
                    assert len(ready) <= hi
            elif count:
                bus.drain_many(first, count, count * R)

    def prepare(self):
        done, off, _ = self.sb.progress()
        self._drain_others()
        if done == len(self.batches):
            return
        if self.after_cut:                               # leave D full: this round moves nothing
            self.after_cut, self.n_stalls = False, self.n_stalls + 1
            self.expect = (done, off)
            return
        ev = self.batches[done][0]
        end = min([c for c in self.cuts.get(done, ()) if c > off], default=len(ev))
        need = int((ev["target"][off:end] == nat.TARGET_ALL).sum())
        free = R - (int(self.d_bus.digests(D, 1)["count"][0]) - self.d_head)
        if end < len(ev):
            assert free <= need and ev["target"][end] == nat.TARGET_ALL, (done, off, end, free, need)
            self.after_cut, self.n_cuts = True, self.n_cuts + 1
        take = max(0, need - free)
        if take:
            assert len(self.d_bus.drain(D, cap=take)) == take
            self.d_head += take
        self.expect = (done + 1, 0) if end == len(ev) else (done, end)

    def check(self):
        assert self.sb.progress()[:2] == self.expect

    def pump(self):
        self.check()
        self.prepare()


def _lossless(sb, batches, kind, cuts):
    cut = _Cutter(sb, batches, cuts)
    for q, (ev, w) in enumerate(batches):
        _put(sb, ev, w)
        cut.prepare()
        if kind == "round":
            sb.run_rounds(q + 1, pump=cut.pump, depth=1)
            cut.check()
        else:
            while True:
                rc_ = sb.fanout(len(ev), w)
                cut.check()
                if rc_ == nat.OK:
                    break
                assert rc_ == nat.EAGAIN
                cut.prepare()
    assert cut.n_cuts == sum(len(c) for q, c in cuts.items() if q < len(batches))
    if kind == "round":
        assert sb.progress()[2] == cut.n_stalls == cut.n_cuts
    return cut


@contextlib.contextmanager
def _fanout_kernels(ran: set):
    """collect the names of the fan-out kernels that run inside the block (torch.profiler, CUDA activities)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        yield
        torch.cuda.synchronize()
    ran.update(m.group(0) for e in prof.events() for m in [FANOUT.search(e.name)] if m)


def _check_rings(sb, fl, batches, devices, digest, lossless):
    """(a) every shard's rings against the reference, pinned to the oracle on its first, last, designated and a unicast
    target's mailbox; (b) every mailbox against the C oracle; (c) nothing overwritten in lossless mode"""
    import torch
    rec = np.concatenate([ev for ev, _ in batches])
    spans, a = [], 0
    for ev, w in batches:
        spans.append((a, a + len(ev), w)); a += len(ev)
    uni = rec["target"][rec["target"] != nat.TARGET_ALL]
    for g, (first, count, bus) in enumerate(sb.shards):
        model = fl.model(first, count, rec, spans)
        hit = [int(t) - first for t in uni if first <= t < first + count][:1]
        model.pin(sorted({0, count - 1, *hit} | ({D - first} if first <= D < first + count else set())))
        with torch.cuda.device(devices[g]), rc.fleet_views(bus.device_ptrs(), count, R) as views:
            assert rc.check(views, model) > 0
        orc = fl.oracle(first, count, batches)
        if digest:
            tr.compare(bus, orc, count, sub_id_base=first, window=R)
        else:
            _compare_no_digest(bus, orc, count, R, base=first)
        if lossless:
            assert bus.stats()["overwritten"] == 0


def _run(kind, store, fl, digest, seed, B=256, grid=0):
    lossless = kind != "follow"
    batches = _batches(fl, B, seed, CUTS if lossless else {})
    devices = _devices(G)
    sb = LocalShardedBus(fl.n, devices, ring_cap=R, batch_cap=B, timers_per_sub=fl.K, digest=digest, stream_slots=8,
                         lossless=lossless, agree="device" if kind == "round" else "host", store_path=store,
                         grid_ctas=grid)
    try:
        fl.populate(sb)
        ran = set()
        with _fanout_kernels(ran):
            if lossless:
                _lossless(sb, batches, kind, CUTS)
            else:
                _follow(sb, batches)
            sb.sync()
        want = kernel_name(kind, store, fl.build, digest)
        assert ran == {want}, f"ran {sorted(ran)}, expected {want}"
        _check_rings(sb, fl, batches, devices, digest, lossless)
    finally:
        sb.close()


# ---- the matrix --------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("digest", [True, False])
@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("kind", KINDS)
def test_cell(kind, store, build, digest):
    """301 subscribers on two shards, ~1,860 records in 14 batches of 0-256 records: every dense ring wraps"""
    seed = 1000 * KINDS.index(kind) + 100 * store + 10 * BUILDS.index(build) + digest
    _run(kind, store, _Fleet(build, 301, seed), digest, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("kind", ["follow", "round"])
@pytest.mark.parametrize("geometry", ["spw16_k8", "grid3", "pairs_grid1"])
def test_geometry(geometry, kind, store, monkeypatch):
    """spw16_k8: 16 mailboxes per warp, K = 8, 512-record batches, 300 subscribers (a CTA's 128 mailboxes take three staging
    rounds, the last CTA is partial); grid3: a fixed 3-CTA grid; pairs_grid1: ~900 paired subscribers on one CTA per shard,
    so that warps walk several triage blocks"""
    seed = 5000 + 100 * store + 10 * ["follow", "round"].index(kind) + ["spw16_k8", "grid3", "pairs_grid1"].index(geometry)
    if geometry == "spw16_k8":
        monkeypatch.setenv("CPBUS_SUBS_PER_WARP", "16")
        _run(kind, store, _Fleet("timers", 300, seed, K=8), True, seed, B=512)
    elif geometry == "grid3":
        _run(kind, store, _Fleet("timers", 300, seed), True, seed, grid=3)
    else:
        _run(kind, store, _Fleet("pairs", 900, seed), True, seed, grid=1)


# ---- full scale: 1,048,576 subscribers, checked like test_gpu_fleet_rings ------------------------------------------------

def _full_scale(kind, store, K, period):
    import torch
    N, B, E, dt = fleet_rings.N, fleet_rings.B, fleet_rings.E, fleet_rings.DT
    rng = np.random.default_rng(0xF011 + store)
    rec = fleet_rings._records(rng.integers(1, 17, E), rng.integers(0, 4096, E))
    masks = np.full(N, nat.MASK_ALL, dtype=np.uint32)
    batches = [(rec[i:i + B], int(rec["ts_ns"][min(E, i + B) - 1])) for i in range(0, E, B)]
    spans = [(i, min(E, i + B), w) for i, (_, w) in zip(range(0, E, B), batches)]
    timers = [{"period": np.full(N, period, dtype=np.uint64), "source": (1_000_000 + np.arange(N)).astype(np.uint32),
               "oneshot": False}] if K else []
    sb = LocalShardedBus(N, [torch.cuda.current_device()], ring_cap=R, batch_cap=B, timers_per_sub=K, stream_slots=8,
                         lossless=kind == "round", agree="device", store_path=store)
    try:
        _, _, bus = sb.shards[0]
        sb.subscribe_many(masks)
        if K:
            sb.timer_add_many(period, source_id0=1_000_000)
        ran = set()
        with _fanout_kernels(ran):
            for ev, w in batches:
                _put(sb, ev, w)
            if kind == "follow":
                sb.follow(0, len(batches))
            else:
                sb.run_rounds(len(batches), pump=sb.consume_all, depth=4)
            assert sb.progress() == (len(batches), 0, 0)
            sb.sync()
        assert ran == {kernel_name(kind, store, "timers" if K else "dense", True)}, ran
        model = rc.FleetModel(N, R, rec, spans, masks, timers=timers)
        model.pin(fleet_rings.PIN)
        with rc.fleet_views(bus.device_ptrs(), N, R) as views:
            assert rc.check(views, model) > 0
        st = bus.stats()
        assert st["ticks"] == (N * (E * dt // period) if K else 0)
        if kind == "round":
            assert st["overwritten"] == 0
    finally:
        sb.close()


@pytest.mark.gpu
def test_full_scale_dense_bulk_followers():
    """a dense BULK follower fleet: the TMA store of dense runs whose length comes from the slot header, at the computed
    16 mailboxes per warp"""
    _full_scale("follow", nat.STORE_BULK, 0, 0)


@pytest.mark.gpu
def test_full_scale_config3_lossless_rounds():
    """BASELINE config 3's shape (one 1 kHz timer per subscriber) as a lossless V8 round fleet, consume_all as the pump"""
    _full_scale("round", nat.STORE_V8, 1, 1_000_000)
