"""Multi-GPU bus (SURVEY.md §8e): the subscriber set partitions into contiguous shards, one `Bus` per GPU; rings,
control blocks and timers never move.  The only thing every shard must see is the publisher's batch sequence, and that
exchange is fused into the fan-out kernel (libcpbus `cpbus_stream_*`: a flagged ring in the publisher GPU's HBM that the
other GPUs' lead CTAs pull over NVLink) — there is no collective on the data path.  Because records carry GLOBAL
subscriber ids (`cpbus_config.sub_id_base`), a subscriber's sequence and digest do not depend on the shard count.

Two drivers over the same C-ABI:

* `ShardedBus`      — one process per GPU (`torch.distributed.run`); torch.distributed (NCCL or gloo) is used ONLY for the
                      construction handshake (the 64-byte CUDA-IPC handle) and for reducing statistics.  Also in lossless
                      mode: the ranks agree on the minimum admitted prefix through offer words in the publisher's memory
                      (`cpbus_stream_offer` / `cpbus_stream_agree`).
* `LocalShardedBus` — one process driving G buses (what a cgo shim inside the single ContainerPilot process does):
                      `cpbus_stream_attach`, peer access instead of IPC; also runs with all shards on ONE GPU.  Also in
                      lossless mode (`cpbus_stream_admit` on every shard, then `cpbus_stream_fanout_prefix` of the minimum).
"""
from __future__ import annotations

import numpy as np

from . import _native as nat
from .bus import Bus, EVENT_DTYPE


def shard_range(n_total: int, world: int, rank: int) -> tuple[int, int]:
    """Contiguous, near-even partition: returns (first_global_id, count) of `rank`'s shard."""
    if not (0 <= rank < world):
        raise ValueError("rank out of range")
    base, extra = divmod(n_total, world)
    first = rank * base + min(rank, extra)
    return first, base + (1 if rank < extra else 0)


def owner_of(sub_id: int, n_total: int, world: int) -> int:
    """Rank that holds global subscriber `sub_id` (inverse of shard_range)."""
    base, extra = divmod(n_total, world)
    cut = extra * (base + 1)
    return sub_id // (base + 1) if sub_id < cut else extra + (sub_id - cut) // max(base, 1)


def stamp_trace(codes: np.ndarray, sources: np.ndarray, dt_ns: int, first_seq: int = 0) -> np.ndarray:
    """Complete 32-byte records for a device-resident trace: seq = publish ordinal, ts = (seq+1)*dt."""
    n = len(codes)
    ev = np.zeros(n, dtype=EVENT_DTYPE)
    ev["seq"] = first_seq + np.arange(n, dtype=np.uint64)
    ev["ts_ns"] = (first_seq + 1 + np.arange(n, dtype=np.uint64)) * np.uint64(dt_ns)
    ev["code"], ev["source_id"], ev["target"] = codes, sources, 0xFFFFFFFF
    return ev


def broadcast_events(dist, events_u8, src: int = 0):
    """Fallback ingest when no peer mapping can be made (no NVLink/IPC): broadcast a batch (uint8 tensor [n, 32] on the
    backend's device) from `src` with the collective backend — NCCL on GPUs, gloo in the CPU tests."""
    dist.broadcast(events_u8, src=src)
    return events_u8


def _admit_or_stall(bus, st, n: int, now_ns: int) -> tuple[int, bool]:
    """(prefix, stalled) this shard offers: what cpbus_stream_admit admits, or (0, True) when it reports a stall."""
    try:
        return bus.stream_admit(st, n, now_ns), False
    except nat.CpbusError as ex:
        if ex.status != nat.EAGAIN:
            raise
        return 0, True


def _agree(bus, st) -> int | None:
    """the agreed prefix of this round, or None when some shard stalled"""
    try:
        return bus.stream_agree(st)
    except nat.CpbusError as ex:
        if ex.status != nat.EAGAIN:
            raise
        return None


def _fanout_prefix(bus, st, n: int, now_ns: int, m: int) -> int:
    """cpbus_stream_fanout_prefix of the agreed prefix m: nat.OK (batch complete) or nat.EAGAIN (records remain)"""
    rc = bus.stream_fanout_prefix(st, n, now_ns, m)
    if rc not in (nat.OK, nat.EAGAIN):
        nat.check(rc, "cpbus_stream_fanout_prefix")
    return rc


def drive_rounds(queue_round, progress, T: int, pump=None, depth: int = 4) -> int:
    """Lossless followers told only the number of batches T: queue admission rounds until batch T is complete.

    `queue_round()` enqueues ONE round on every shard the caller drives (cpbus_stream_round_next); `progress()` resolves and
    returns (batches complete, offset, stalled rounds) (cpbus_stream_progress); `pump()` lets the consumers run.  At most
    min(depth, T - batches) rounds are queued between resolutions — one round completes at most one batch, so none reaches
    past batch T — and the pump runs between rounds and after each resolution.  Every rank that runs this with the same T
    sees the same outcomes, so every rank queues the same rounds and all stop together.  Returns the rounds queued."""
    if not 1 <= depth <= 8:
        raise ValueError("depth must be 1..8 (outstanding rounds per bus)")
    queued = 0
    done = progress()[0]
    while done < T:
        for i in range(min(depth, T - done)):
            if i and pump is not None:
                pump()
            queue_round()
            queued += 1
        done = progress()[0]
        if done < T and pump is not None:
            pump()
    return queued


def _walk(ranges, first_sub: int, n: int, start_sub: int) -> list[tuple[int, int, int]]:
    """cpbus_group_lagging's walk over shards that own the contiguous id ranges `ranges` [(first, count)]: mailboxes
    [first_sub, first_sub + n) in cyclic order from start_sub, as pieces (shard, first id, count) in visiting order."""
    if n <= 0 or not first_sub <= start_sub < first_sub + n:
        raise nat.CpbusError(nat.EINVAL, "lagging")
    out, done = [], 0
    while done < n:
        i = first_sub + (start_sub - first_sub + done) % n
        k = next((k for k, (f, c) in enumerate(ranges) if f <= i < f + c), None)
        if k is None:
            raise nat.CpbusError(nat.ENOENT, "lagging")
        f, c = ranges[k]
        cnt = min(n - done, f + c - i, first_sub + n - i)
        out.append((k, i, cnt))
        done += cnt
    return out


_SUMMARY_WORDS = ("active", "lagging", "backlog_total", "backlog_max", "lost_total")


def _merge_lagging(pieces, cap: int, start_sub: int):
    """pieces in visiting order, each (entries, next_sub, summary) of one shard's part scanned with at least the cap left
    at that point: (entries, next_sub, summary) of the whole walk.  Entries are taken with the cap that is left; the first
    piece that cannot return all of its lagging mailboxes sets next_sub; summaries add, backlog_max is the maximum."""
    ents, got, nxt, cut = [], 0, start_sub, False
    acc = {"active": 0, "lagging": 0, "backlog_total": 0, "backlog_max": 0, "lost_total": 0, "hist": [0] * 33}
    for e, nx, s in pieces:
        left = cap - got
        ents.append(e[:left])
        got += len(ents[-1])
        if not cut and s["lagging"] > len(ents[-1]):
            nxt, cut = (int(e["sub_id"][left]) if left < len(e) else nx), True
        for k in ("active", "lagging", "backlog_total", "lost_total"):
            acc[k] += s[k]
        acc["backlog_max"] = max(acc["backlog_max"], s["backlog_max"])
        acc["hist"] = [a + b for a, b in zip(acc["hist"], s["hist"])]
    return (np.concatenate(ents) if ents else np.zeros(0, dtype=nat.LAG_DTYPE)), nxt, acc


class _ShardOps:
    """What both drivers share: a shard is a `Bus` plus its end of the publisher's stream."""

    bus: Bus
    first: int
    count: int

    # -- membership / timers on this shard (global ids) --------------------
    def subscribe_many(self, masks) -> int:
        return self.bus.subscribe_many(masks)

    def timer_add_many(self, period_ns: int, source_id0: int = 0, source_ids=None, oneshot: bool = False):
        self.bus.timer_add_many(self.first, self.count, period_ns, source_ids=source_ids,
                                source_id0=source_id0 + (0 if source_ids is not None else self.first), oneshot=oneshot)

    def digests(self):
        return self.bus.digests(self.first, self.count)


class ShardedBus(_ShardOps):
    """One rank's shard; constructed collectively by every rank of `dist` (torch.distributed, already initialised).

    Data path per step (SPMD: every rank knows n and now_ns of each batch):
        rank 0       : put(events, now_ns)            host batch -> the stream ring (H2D + release), may run ahead
        every rank   : fanout(n, now_ns)              one fan-out launch; the batch is pulled inside the kernel
    Device-resident traces (the publisher's events already in its HBM): attach_trace / fanout_trace.

    `lossless=True` gives every shard the reference's blocking semantics (a publish stops at the event the Go bus would
    block on, on every rank): `fanout` runs one admission round — admit, offer, agree, fan out the agreed prefix — and
    returns nat.OK (batch complete) or nat.EAGAIN (drain, then every rank calls `fanout` again with the same n, now_ns).
    The ranks agree through offer words in the publisher's memory, with no collective.  Device-batch paths
    (fanout_trace, fanout_broadcast) stay throughput-only.
    """

    def __init__(self, n_subs_total: int, dist=None, rank: int = 0, world: int = 1, device: int = -1, ring_cap: int = 1024,
                 batch_cap: int = 512, timers_per_sub: int = 0, digest: bool = True, stream_slots: int = 64,
                 stream=None, store_path: int = nat.STORE_AUTO, grid_ctas: int = 0, subs_per_rank: int | None = None,
                 bus_factory=Bus, lossless: bool = False):
        self.dist, self.rank, self.world = dist, rank, world
        self.lossless = lossless
        if subs_per_rank is not None:               # weak scaling: fixed shard size
            self._ranges = [(r * subs_per_rank, subs_per_rank) for r in range(world)]
        else:
            self._ranges = [shard_range(n_subs_total, world, r) for r in range(world)]
        self.first, self.count = self._ranges[rank]
        self.bus = bus_factory(max(self.count, 1), ring_cap=ring_cap, batch_cap=batch_cap, timers_per_sub=timers_per_sub, digest=digest,
                       device=device, sub_id_base=self.first, store_path=store_path, stream=stream, grid_ctas=grid_ctas,
                       lossless=lossless)
        self.batch_cap = batch_cap
        self._st = None
        self._peer_trace = None      # (mapped pointer, owner?) of the attached device trace
        self._trace_ptr = None
        self._trace_local = False
        self.ingest = "local"
        self._open_stream(stream_slots)

    # -- construction handshake -------------------------------------------
    def _all_ok(self, ok: bool) -> bool:
        if self.world == 1:
            return ok
        import torch
        dev = "cuda" if self.dist.get_backend() == "nccl" else "cpu"
        t = torch.tensor([1 if ok else 0], device=dev)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MIN)
        return bool(int(t.item()))

    def _open_stream(self, slots: int):
        ok, handle = True, None
        if self.rank == 0:
            try:
                self._st, handle = self.bus.stream_create(slots, self.world)
            except nat.CpbusError as ex:                    # pragma: no cover - depends on the box
                self._err = ex
                ok, handle = False, None
        if self.world > 1:
            box = [handle]
            self.dist.broadcast_object_list(box, src=0)
            if self.rank != 0:
                if box[0] is None:
                    ok = False
                else:
                    try:
                        self._st = self.bus.stream_open(box[0], self.rank)
                    except nat.CpbusError as ex:            # pragma: no cover
                        self._err = ex
                        ok = False
        self.stream_ok = self._all_ok(ok)
        if self.stream_ok:
            self.ingest = "nvlink-stream (flagged ring, pulled inside the fan-out kernel)" if self.world > 1 else "local stream"

    # -- host batches ------------------------------------------------------
    def put(self, events: np.ndarray, now_ns: int, raw: bool = False) -> int:
        """Publisher rank only (no-op elsewhere).  EAGAIN: the consumers are a whole ring behind."""
        if self.rank != 0:
            return nat.OK
        return self.bus.stream_put(self._st, events, now_ns, raw)

    def fanout(self, n: int, now_ns: int) -> int:
        if not self.lossless:
            return self.bus.stream_fanout(self._st, n, now_ns)
        # one admission round; every rank runs it, so every rank's round ordinal advances together
        prefix, stalled = _admit_or_stall(self.bus, self._st, n, now_ns)
        self.bus.stream_offer(self._st, prefix, stalled)
        m = _agree(self.bus, self._st)
        if m is None:
            return nat.EAGAIN                       # some rank stalled: nothing goes out anywhere
        return _fanout_prefix(self.bus, self._st, n, now_ns, m)

    def follow(self, k: int = 1):
        """Enqueue fan-outs of the stream's next `k` batches on this rank without knowing their shapes: each launch takes
        n and the watermark from the slot header (`cpbus_stream_fanout_next`), so a rank that holds only subscriber shards
        never sees the events and never syncs per batch.  Throughput mode only."""
        if self.lossless:
            raise RuntimeError("a lossless ShardedBus agrees on every batch's admitted prefix (fanout), which needs its shape")
        for _ in range(k):
            nat.check(self.bus.stream_fanout_next(self._st), "cpbus_stream_fanout_next")

    def follow_rounds(self, k: int = 1):
        """Lossless mode: enqueue `k` admission rounds on this rank without knowing the batches' shapes
        (`cpbus_stream_round_next`): admit, offer, agree and the fan-out of the agreed prefix all run on the device, and the
        host never waits for them.  Every rank must queue the same rounds."""
        if not self.lossless:
            raise RuntimeError("rounds agree on an admitted prefix: a throughput-mode ShardedBus follows with follow()")
        for _ in range(k):
            nat.check(self.bus.stream_round_next(self._st), "cpbus_stream_round_next")

    def progress(self) -> tuple[int, int, int]:
        """Resolve outstanding followers / rounds: (batches complete, records of the next one delivered, stalled rounds)."""
        rc, done, off, stalled = self.bus.stream_progress(self._st)
        nat.check(rc, "cpbus_stream_progress")
        return done, off, stalled

    def run_rounds(self, T: int, pump=None, depth: int = 4) -> int:
        """Lossless followers: queue rounds until this rank has completely fanned out T batches (`drive_rounds`)."""
        return drive_rounds(lambda: self.follow_rounds(1), self.progress, T, pump, depth)

    def publish(self, events: np.ndarray, now_ns: int) -> int:
        """put + fanout for callers that do not pipeline.  Lossless mode: one round, no retry (EAGAIN: drain, then
        `fanout` again)."""
        rc = self.put(events, now_ns)
        return rc if rc else self.fanout(len(events), now_ns)

    # -- device-resident trace (publisher's events already in its HBM) ----
    def attach_trace(self, nbytes: int):
        """Rank 0 allocates a shareable buffer of `nbytes` and returns its device pointer (fill it, then call
        `trace_ready()`); the other ranks map it over NVLink.  Returns the local pointer on rank 0, None elsewhere."""
        ok, handle, ptr = True, None, None
        if self.rank == 0:
            try:
                ptr, handle = self.bus.shared_alloc(nbytes)
            except nat.CpbusError as ex:                    # pragma: no cover
                self._err = ex
                ok = False
        if self.world > 1:
            box = [handle]
            self.dist.broadcast_object_list(box, src=0)
            if self.rank != 0:
                if box[0] is None:
                    ok = False
                else:
                    try:
                        self._peer_trace = self.bus.shared_open(box[0])
                    except nat.CpbusError as ex:            # pragma: no cover
                        self._err = ex
                        ok = False
        self.trace_ok = self._all_ok(ok)
        self._trace_ptr = ptr if self.rank == 0 else self._peer_trace
        if self.trace_ok and self.world > 1:
            self.ingest = "nvlink-peer-pull (fused into the fan-out kernel)"
        return ptr

    def _no_device_batches_in_lossless(self):
        if self.lossless:
            raise RuntimeError("device-resident batches are all-or-nothing per shard: a lossless ShardedBus takes its "
                               "batches through put / fanout only")

    def use_local_trace(self, ptr: int):
        """The trace already sits in THIS GPU's memory at `ptr` (single GPU, or a replicated / NCCL-broadcast copy)."""
        self._trace_ptr, self._trace_local = ptr, True

    def fanout_trace(self, offset_bytes: int, n: int, watermark_ns: int, next_offset_bytes: int | None = None, next_n: int = 0) -> int:
        """Fan out records [offset, offset + 32 n) of the attached trace; `next_offset_bytes` names a LATER batch (best: the
        one after next) that this launch pulls across the link while its stores are in flight."""
        self._no_device_batches_in_lossless()
        base = self._trace_ptr
        if self.world == 1 or self._trace_local:
            return self.bus.publish_device(base + offset_bytes, n, watermark_ns)
        nxt = base + next_offset_bytes if next_offset_bytes is not None else 0
        return self.bus.publish_device_staged(base + offset_bytes, n, watermark_ns, nxt, next_n if nxt else 0)

    def fanout_broadcast(self, batch_u8, n: int, watermark_ns: int) -> int:
        """Fallback (no peer mapping): `batch_u8` is a [n, 32] uint8 CUDA tensor, valid on rank 0; NCCL broadcast, then a
        local fan-out.  One collective per call — the caller batches several steps per call to amortise it."""
        self._no_device_batches_in_lossless()
        if self.world > 1:
            broadcast_events(self.dist, batch_u8, src=0)
        return self.bus.publish_device(batch_u8.data_ptr(), n, watermark_ns)

    def barrier(self):
        if self.world > 1:
            self.dist.barrier()

    # -- consumer backlog over every shard (collective: every rank calls, every rank gets the same answer) --
    def _all_gather_words(self, words: np.ndarray) -> list[np.ndarray]:
        """every rank's uint64 vector: one all_gather of the lengths, one of the padded vectors"""
        if self.world == 1:
            return [words]
        import torch
        dev = "cuda" if self.dist.get_backend() == "nccl" else "cpu"
        n = torch.tensor([words.size], dtype=torch.int64, device=dev)
        ns = [torch.zeros_like(n) for _ in range(self.world)]
        self.dist.all_gather(ns, n)
        ns = [int(x) for x in ns]
        buf = torch.zeros(max(1, max(ns)), dtype=torch.int64, device=dev)
        buf[:words.size] = torch.from_numpy(np.ascontiguousarray(words, dtype=np.uint64).view(np.int64)).to(dev)
        got = [torch.zeros_like(buf) for _ in range(self.world)]
        self.dist.all_gather(got, buf)
        return [g[:k].cpu().numpy().view(np.uint64) for g, k in zip(got, ns)]

    def blockers(self, cap: int | None = None) -> np.ndarray:
        """Lossless mode: the global ids of the mailboxes the stream's current round waits on, over every rank, ascending
        (the first `cap`; default all).  Each rank asks its own shard (cpbus_stream_blockers); one exchange merges them.
        Resolves this rank's outstanding rounds: call it between run_rounds / follow_rounds calls, on every rank."""
        mine = self.bus.stream_blockers(self._st, cap).astype(np.uint64)
        ids = np.sort(np.concatenate(self._all_gather_words(mine))).astype(np.uint32)
        return ids if cap is None else ids[:cap]

    def lagging(self, first_sub: int, n: int, start_sub: int | None = None, min_backlog: int = 1, cap: int | None = None):
        """`Bus.lagging` over mailboxes [first_sub, first_sub+n) of every rank: the walk of cpbus_group_lagging over the
        ranks' shards (entries in cyclic order from start_sub, the first `cap`; next_sub; summaries added, backlog_max the
        maximum).  Each rank scans its own pieces; one exchange merges them.  Collective, like `blockers`."""
        start_sub = first_sub if start_sub is None else start_sub
        cap = n if cap is None else cap
        walk = _walk(self._ranges, first_sub, n, start_sub)
        words = []                                  # per own piece: j, entries, next_sub, summary, entries' words
        for j, (k, a, cnt) in enumerate(walk):
            if k != self.rank:
                continue
            e, nx, s = self.bus.lagging(a, cnt, start_sub=a, min_backlog=min_backlog, cap=cap)
            words += [j, len(e), nx] + [s[f] for f in _SUMMARY_WORDS] + list(s["hist"])
            words += [int(x) for r in e for x in (r["sub_id"], r["backlog"], r["lost"])]
        pieces = {}
        for w in self._all_gather_words(np.array(words, dtype=np.uint64)):
            at = 0
            while at < len(w):
                j, m, nx = (int(x) for x in w[at:at + 3])
                s = dict(zip(_SUMMARY_WORDS, (int(x) for x in w[at + 3:at + 8])))
                s["hist"] = [int(x) for x in w[at + 8:at + 41]]
                e = np.zeros(m, dtype=nat.LAG_DTYPE)
                rows = w[at + 41:at + 41 + 3 * m].reshape(m, 3)
                e["sub_id"], e["backlog"], e["lost"] = rows[:, 0], rows[:, 1], rows[:, 2]
                pieces[j] = (e, nx, s)
                at += 41 + 3 * m
        return _merge_lagging([pieces[j] for j in range(len(walk))], cap, start_sub)

    # -- reductions (verification, statistics) -----------------------------
    def digest_fold_all(self):
        """(sum count, sum digest, xor H(digest, count, id), n) over EVERY shard — equal for any shard count."""
        f = self.bus.digest_fold(self.first, self.count)
        if self.world == 1:
            return f
        gathered = [None] * self.world
        self.dist.all_gather_object(gathered, tuple(int(x) for x in f))
        M = (1 << 64) - 1
        c = d = x = n = 0
        for g in gathered:
            c = (c + g[0]) & M; d = (d + g[1]) & M; x ^= g[2]; n += g[3]
        return (c, d, x, n)

    def close(self):
        if self._peer_trace is not None:
            try:
                self.bus.shared_close(self._peer_trace)
            except nat.CpbusError:                          # pragma: no cover - teardown only
                pass
            self._peer_trace = None
        if self.world > 1 and self.rank != 0 and self._st is not None:
            self.bus.stream_close(self._st); self._st = None   # importers unmap before the owner frees
        if self.world > 1:
            self.dist.barrier()
        if self._st is not None:
            self.bus.stream_close(self._st); self._st = None
        self.bus.close()


class LocalShardedBus:
    """G shards driven by ONE process (shard g on `devices[g]`; all on one GPU is allowed): what a cgo shim inside the
    single ContainerPilot process does.  Same stream protocol as `ShardedBus`, attached in-process.  `lossless=True` gives every
    shard the reference's blocking semantics: a publish stops at the event the Go bus would block on, on every shard.
    The shards' minimum prefix is taken on the host (`agree="host"`) or, with `agree="device"`, through the offer words
    in the publisher's memory and the agree kernel — the protocol `ShardedBus(lossless=True)` runs across processes."""

    def __init__(self, n_subs_total: int, devices, ring_cap: int = 1024, batch_cap: int = 512, timers_per_sub: int = 0,
                 digest: bool = True, stream_slots: int = 64, lossless: bool = False, agree: str = "host",
                 store_path: int = nat.STORE_AUTO, grid_ctas: int = 0):
        if agree not in ("host", "device"):
            raise ValueError(f"agree must be 'host' or 'device', not {agree!r}")
        self.world = len(devices)
        self.lossless, self.agree = lossless, agree
        self.last_round = None                      # agree="device": ([(prefix, stalled)], [agreed m or None]) per shard
        self.shards = []
        for g, dev in enumerate(devices):
            first, count = shard_range(n_subs_total, self.world, g)
            self.shards.append((first, count, Bus(max(count, 1), ring_cap=ring_cap, batch_cap=batch_cap, timers_per_sub=timers_per_sub,
                                                  lossless=lossless, digest=digest, device=dev, sub_id_base=first,
                                                  store_path=store_path, grid_ctas=grid_ctas)))
        pub = self.shards[0][2]
        st0, _ = pub.stream_create(stream_slots, self.world)
        self._st = [st0] + [self.shards[g][2].stream_attach(st0, g) for g in range(1, self.world)]

    def bus_of(self, sub_id: int) -> Bus:
        for first, count, bus in self.shards:
            if first <= sub_id < first + count:
                return bus
        raise KeyError(sub_id)

    def subscribe_many(self, masks):
        """global masks array, split by shard"""
        masks = np.asarray(masks, dtype=np.uint32)
        for first, count, bus in self.shards:
            if count:
                bus.subscribe_many(masks[first:first + count])

    def timer_add_many(self, period_ns: int, source_id0: int = 0):
        for first, count, bus in self.shards:
            if count:
                bus.timer_add_many(first, count, period_ns, source_id0=source_id0 + first)

    def publish(self, events: np.ndarray, now_ns: int, raw: bool = False) -> int:
        """One batch to every shard: put once, fan out on each GPU (never ahead of its own fan-outs, so it may wait).
        Lossless mode: returns what `fanout` returns (EAGAIN: drain, then call `fanout` with the same shape)."""
        nat.check(self.shards[0][2].stream_put(self._st[0], events, now_ns, raw), "cpbus_stream_put")
        return self.fanout(len(events), now_ns)

    def put(self, events: np.ndarray, now_ns: int, raw: bool = False) -> int:
        """Run ahead of the fan-outs.  One thread drives publisher and consumers here, so this never waits: EAGAIN means
        "fan out (or sync) first" — the slot's previous batch has not been pulled by every shard yet."""
        return self.shards[0][2].stream_put(self._st[0], events, now_ns, raw, nowait=True)

    def fanout(self, n: int, now_ns: int) -> int:
        """Fan the next batch out to every shard.  Lossless mode: every shard admits what its mailboxes can take and every
        shard delivers the shortest of those prefixes, so a stalled publish stops at the same event everywhere.  Returns
        nat.OK (batch complete) or nat.EAGAIN (records remain: let the consumers drain, then call again with the same
        n and now_ns — the batch resumes at its first undelivered record)."""
        if not self.lossless:
            for g, (_, _, bus) in enumerate(self.shards):
                nat.check(bus.stream_fanout(self._st[g], n, now_ns), "cpbus_stream_fanout")
            return nat.OK
        m = self._agree_device(n, now_ns) if self.agree == "device" else self._agree_host(n, now_ns)
        if m is None:
            return nat.EAGAIN                       # some shard stalled: nothing goes out anywhere
        rc = nat.OK
        for g, (_, _, bus) in enumerate(self.shards):
            rc = _fanout_prefix(bus, self._st[g], n, now_ns, m)
        return rc

    def _agree_host(self, n: int, now_ns: int) -> int | None:
        """The shortest prefix any shard admits, or None at the first shard that stalls (the later ones are not admitted:
        their room bounds and admission counters stay as they are)."""
        m = None
        for g, (_, _, bus) in enumerate(self.shards):
            p, stalled = _admit_or_stall(bus, self._st[g], n, now_ns)
            if stalled:
                return None
            m = p if m is None else min(m, p)
        return m

    def _agree_device(self, n: int, now_ns: int) -> int | None:
        """One admission round through the publisher's memory (what `ShardedBus(lossless=True)` does on each rank): every
        shard offers before any shard waits, and every shard agrees, so the round advances in lockstep.  The agreed prefix,
        or None when some shard stalled."""
        offers = []
        for g, (_, _, bus) in enumerate(self.shards):
            offers.append(_admit_or_stall(bus, self._st[g], n, now_ns))
            bus.stream_offer(self._st[g], *offers[-1])
        agreed = []
        for g, (_, _, bus) in enumerate(self.shards):
            agreed.append(_agree(bus, self._st[g]))
        self.last_round = (offers, agreed)
        if len(set(agreed)) != 1:                   # every agree kernel read the same words
            raise RuntimeError(f"shards agreed on different prefixes: {agreed}")
        return agreed[0]

    def follow(self, g: int, k: int = 1):
        """Enqueue fan-outs of the stream's next `k` batches on shard `g` without their shapes (`cpbus_stream_fanout_next`)."""
        for _ in range(k):
            nat.check(self.shards[g][2].stream_fanout_next(self._st[g]), "cpbus_stream_fanout_next")

    def follow_rounds(self, g: int, k: int = 1):
        """Lossless mode: enqueue `k` admission rounds on shard `g` (`cpbus_stream_round_next`).  A round waits on the
        device for every shard's offer, so queue each round on every shard before the host resolves any of them
        (`run_rounds` does)."""
        if not self.lossless:
            raise RuntimeError("rounds agree on an admitted prefix: a throughput-mode bus follows with follow()")
        for _ in range(k):
            nat.check(self.shards[g][2].stream_round_next(self._st[g]), "cpbus_stream_round_next")

    def progress(self) -> tuple[int, int, int]:
        """Resolve every shard: (batches complete, records of the next one delivered, stalled rounds), equal on every shard."""
        got = []
        for g, (_, _, bus) in enumerate(self.shards):
            rc, done, off, stalled = bus.stream_progress(self._st[g])
            nat.check(rc, "cpbus_stream_progress")
            got.append((done, off, stalled))
        if len(set(got)) != 1:
            raise RuntimeError(f"shards resolved to different positions: {got}")
        return got[0]

    def run_rounds(self, T: int, pump=None, depth: int = 4) -> int:
        """Lossless followers on every shard: queue rounds (each on every shard in turn) until T batches are complete."""
        def one():
            for g in range(self.world):
                self.follow_rounds(g, 1)
        return drive_rounds(one, self.progress, T, pump, depth)

    def drain(self, sub_id: int, cap: int | None = None) -> np.ndarray:
        """Consumer side: up to `cap` records of global subscriber `sub_id`, from the shard that owns it."""
        return self.bus_of(sub_id).drain(sub_id, cap)

    def consume_all(self):
        """Device-side consumer on every shard: every mailbox read to the end, records discarded."""
        for _, _, bus in self.shards:
            bus.consume_all()

    def blockers(self, cap: int | None = None) -> np.ndarray:
        """Lossless mode: the global ids of the mailboxes the stream's current round waits on, over every shard, ascending
        (the first `cap`; default all): each shard's cpbus_stream_blockers.  Resolves outstanding rounds: call it between
        run_rounds / follow_rounds calls."""
        ids = np.sort(np.concatenate([bus.stream_blockers(self._st[g], cap) for g, (_, _, bus) in enumerate(self.shards)]))
        return ids if cap is None else ids[:cap]

    def lagging(self, first_sub: int, n: int, start_sub: int | None = None, min_backlog: int = 1, cap: int | None = None):
        """`Bus.lagging` over mailboxes [first_sub, first_sub+n) of every shard, as one bus with the same mailboxes answers
        it: the walk of cpbus_group_lagging, each shard's piece scanned with the cap still left."""
        start_sub = first_sub if start_sub is None else start_sub
        cap = n if cap is None else cap
        pieces, got = [], 0
        for k, a, cnt in _walk([(f, c) for f, c, _ in self.shards], first_sub, n, start_sub):
            pieces.append(self.shards[k][2].lagging(a, cnt, start_sub=a, min_backlog=min_backlog, cap=cap - got))
            got += len(pieces[-1][0])
        return _merge_lagging(pieces, cap, start_sub)

    def sync(self):
        for _, _, bus in self.shards:
            bus.sync()

    def digests(self):
        """(count, digest) of every subscriber, in global id order"""
        parts = [bus.digests(first, count) for first, count, bus in self.shards if count]
        return np.concatenate(parts)

    def close(self):
        for g in range(self.world - 1, -1, -1):
            self.shards[g][2].stream_close(self._st[g])
        for _, _, bus in self.shards:
            bus.close()
