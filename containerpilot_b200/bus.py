"""`Bus`: a thin numpy-friendly wrapper over the libcpbus C-ABI (include/cpbus.h).

One `Bus` = one GPU's shard of subscriber mailboxes.  Every method maps 1:1 to a
`cpbus_*` entry point; no event ever takes a Python/CPU data path.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as nat

EVENT_DTYPE = np.dtype([("seq", "<u8"), ("ts_ns", "<u8"), ("code", "<u4"), ("source_id", "<u4"),
                        ("target", "<u4"), ("flags", "<u4")])
assert EVENT_DTYPE.itemsize == 32
# cpbus_ready: one entry of cpbus_drain_ready's ready list
READY_DTYPE = np.dtype([("sub_id", "<u4"), ("count", "<u4"), ("offset", "<u4"), ("pad", "<u4"), ("lost", "<u8")])
assert READY_DTYPE.itemsize == 24


class _SingleBusOnly:
    """A `Bus` method that `GroupBus` does not have (the group has no C twin of it): on a class that sets `_GROUP`, and
    its instances, the name does not exist."""

    def __init__(self, fn):
        self._fn = fn
        self.__doc__, self.__name__ = fn.__doc__, fn.__name__

    def __get__(self, obj, owner=None):
        if getattr(owner if owner is not None else type(obj), "_GROUP", False):
            raise AttributeError(f"{self.__name__} has no cpbus_group_* counterpart")
        return self._fn if obj is None else self._fn.__get__(obj, owner)


class Bus:
    def __init__(self, n_max_subs: int, ring_cap: int = 1024, batch_cap: int = 256, timers_per_sub: int = 0,
                 lossless: bool = False, digest: bool = True, device: int = -1, sub_id_base: int = 0,
                 store_path: int = nat.STORE_AUTO, stream: int | None = None, grid_ctas: int = 0, sparse_ticks: bool = False,
                 sparse_records: bool = False, drop_missed_ticks: bool = False, sparse_drains: bool = False):
        """`sparse_ticks`: CPBUS_CFG_SPARSE_TICKS, a flush with no staged event costs what is due (no streams on such a bus).
        `sparse_records`: CPBUS_CFG_SPARSE_RECORDS (implies sparse_ticks), a flush whose events reach few mailboxes
        launches only over them.
        `sparse_drains`: CPBUS_CFG_SPARSE_DRAINS (implies sparse_ticks), a ready drain whose range holds no candidate
        launches nothing, and one with few scans only them.
        `drop_missed_ticks`: CPBUS_CFG_DROP_MISSED_TICKS, a clock step that crosses several periods of a periodic timer
        delivers only its last tick, like Go's time.Ticker (no streams or device batches on such a bus)"""
        self._lib = nat.load()
        cfg = nat.Config()
        cfg.n_max_subs, cfg.ring_cap, cfg.batch_cap, cfg.timers_per_sub = n_max_subs, ring_cap, batch_cap, timers_per_sub
        cfg.flags = ((nat.CFG_LOSSLESS if lossless else 0) | (nat.CFG_DIGEST if digest else 0)
                     | (nat.CFG_SPARSE_TICKS if sparse_ticks or sparse_records or sparse_drains else 0)
                     | (nat.CFG_SPARSE_RECORDS if sparse_records else 0)
                     | (nat.CFG_SPARSE_DRAINS if sparse_drains else 0)
                     | (nat.CFG_DROP_MISSED_TICKS if drop_missed_ticks else 0))
        cfg.device, cfg.sub_id_base, cfg.store_path, cfg.grid_ctas = device, sub_id_base, store_path, grid_ctas
        cfg.stream = C.c_void_p(stream) if stream else None
        self._h = C.c_void_p()
        nat.check(self._lib.cpbus_create(C.byref(cfg), C.byref(self._h)), "cpbus_create")
        self.ring_cap, self.batch_cap, self.sub_id_base = ring_cap, batch_cap, sub_id_base

    # -- lifecycle ---------------------------------------------------------
    def close(self):
        if self._h:
            self._lib.cpbus_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- intern ------------------------------------------------------------
    def intern(self, s: str) -> int:
        raw = s.encode()
        out = C.c_uint32()
        nat.check(self._lib.cpbus_intern(self._h, raw, len(raw), C.byref(out)), "cpbus_intern")
        return out.value

    def intern_ephemeral(self, s: str) -> int:
        """payload strings (Metric "key|value"): ids from the bounded, recycled region"""
        raw = s.encode()
        out = C.c_uint32()
        nat.check(self._lib.cpbus_intern_ephemeral(self._h, raw, len(raw), C.byref(out)), "cpbus_intern_ephemeral")
        return out.value

    def source(self, source_id: int) -> str:
        n = C.c_size_t()
        nat.check(self._lib.cpbus_source(self._h, source_id, None, 0, C.byref(n)), "cpbus_source")
        buf = C.create_string_buffer(max(1, n.value))
        nat.check(self._lib.cpbus_source(self._h, source_id, buf, n.value, C.byref(n)), "cpbus_source")
        return buf.raw[: n.value].decode()

    # -- membership --------------------------------------------------------
    def subscribe(self, mask: int = nat.MASK_ALL) -> int:
        out = C.c_uint32()
        nat.check(self._lib.cpbus_subscribe(self._h, mask, C.byref(out)), "cpbus_subscribe")
        return out.value

    def subscribe_many(self, masks) -> int:
        m = np.ascontiguousarray(masks, dtype=np.uint32)
        out = C.c_uint32()
        nat.check(self._lib.cpbus_subscribe_many(self._h, m.ctypes.data, m.size, C.byref(out)), "cpbus_subscribe_many")
        return out.value

    def subscribe_pairs(self, mask: int, pairs) -> int:
        """second-level filter: `pairs` = exact (code, source_id) cases delivered on top of the code mask"""
        pr = np.ascontiguousarray([(int(c), int(s)) for c, s in pairs], dtype=np.uint32).reshape(-1, 2)
        out = C.c_uint32()
        nat.check(self._lib.cpbus_subscribe_pairs(self._h, mask, pr.ctypes.data if len(pr) else None, len(pr), C.byref(out)),
                  "cpbus_subscribe_pairs")
        return out.value

    def subscribe_pairs_many(self, masks, pairs_per_sub) -> int:
        """a whole fleet in one call: masks[i] and pairs_per_sub[i] = list of (code, source_id), at most 16 each"""
        m = np.ascontiguousarray(masks, dtype=np.uint32)
        n = m.size
        rows = np.full((n, 16, 2), 0xFFFFFFFF, dtype=np.uint32)
        cnt = np.zeros(n, dtype=np.uint32)
        for i, pr in enumerate(pairs_per_sub):
            if len(pr) > 16:
                raise nat.CpbusError(nat.EINVAL, "cpbus_subscribe_pairs_many")
            cnt[i] = len(pr)
            if len(pr):
                rows[i, :len(pr)] = np.asarray(pr, dtype=np.uint32).reshape(-1, 2)
        out = C.c_uint32()
        nat.check(self._lib.cpbus_subscribe_pairs_many(self._h, m.ctypes.data, rows.ctypes.data, cnt.ctypes.data, n, C.byref(out)),
                  "cpbus_subscribe_pairs_many")
        return out.value

    def set_mask(self, sub_id: int, mask: int):
        nat.check(self._lib.cpbus_set_mask(self._h, sub_id, mask), "cpbus_set_mask")

    def unsubscribe(self, sub_id: int):
        nat.check(self._lib.cpbus_unsubscribe(self._h, sub_id), "cpbus_unsubscribe")

    def _membership_many(self, name: str, arrays) -> np.ndarray:
        n = arrays[0].size
        status = np.zeros(n, dtype=np.int32)
        nat.check(getattr(self._lib, name)(self._h, *[a.ctypes.data if n else None for a in arrays], n,
                                           status.ctypes.data if n else None, None), name)
        return status

    def unsubscribe_many(self, sub_ids) -> np.ndarray:
        """cpbus_unsubscribe for every id in order, in one call: the int32 status each single call would have returned
        (OK, ENOENT or ECLOSED).  Raises on any other return, CPBUS_EAGAIN included (nothing was applied)."""
        return self._membership_many("cpbus_unsubscribe_many", [np.ascontiguousarray(sub_ids, dtype=np.uint32)])

    def set_mask_many(self, sub_ids, masks) -> np.ndarray:
        """cpbus_set_mask(sub_ids[i], masks[i]) in order, in one call: the per-element statuses, as unsubscribe_many"""
        ids, m = np.ascontiguousarray(sub_ids, dtype=np.uint32), np.ascontiguousarray(masks, dtype=np.uint32)
        if ids.shape != m.shape:
            raise ValueError("sub_ids and masks differ in length")
        return self._membership_many("cpbus_set_mask_many", [ids, m])

    def release_many(self, sub_ids) -> np.ndarray:
        """cpbus_release_many: give unsubscribed ids back for subscribe_list to hand out again.  The int32 status of each
        element: OK, ENOENT (never handed out, or already released) or EINVAL (still subscribed).  Raises on any other
        return, CPBUS_EAGAIN included (nothing was released).  An id must not be used after it is released."""
        return self._membership_many("cpbus_release_many", [np.ascontiguousarray(sub_ids, dtype=np.uint32)])

    def subscribe_list(self, masks, pairs=None) -> np.ndarray:
        """cpbus_subscribe_list: subscribe len(masks) subscribers on the lowest free ids (released ones first) and return
        their uint32 ids.  `pairs` (optional) = one list of exact (code, source_id) cases per subscriber, at most 16 each."""
        m = np.ascontiguousarray(masks, dtype=np.uint32)
        n = m.size
        rows = cnt = None
        if pairs is not None:
            rows = np.full((max(n, 1), 16, 2), 0xFFFFFFFF, dtype=np.uint32)
            cnt = np.zeros(max(n, 1), dtype=np.uint32)
            for i, pr in enumerate(pairs):
                if len(pr) > 16:
                    raise nat.CpbusError(nat.EINVAL, "cpbus_subscribe_list")
                cnt[i] = len(pr)
                if len(pr):
                    rows[i, :len(pr)] = np.asarray(pr, dtype=np.uint32).reshape(-1, 2)
        ids = np.zeros(max(n, 1), dtype=np.uint32)
        nat.check(self._lib.cpbus_subscribe_list(self._h, m.ctypes.data if n else None, None if rows is None else rows.ctypes.data,
                                                  None if cnt is None else cnt.ctypes.data, n, ids.ctypes.data),
                  "cpbus_subscribe_list")
        return ids[:n]

    # -- timers ------------------------------------------------------------
    def timer_add(self, sub_id: int, period_ns: int, source_id: int, oneshot: bool = False) -> int:
        out = C.c_uint32()
        nat.check(self._lib.cpbus_timer_add(self._h, sub_id, period_ns, source_id, int(oneshot), C.byref(out)), "cpbus_timer_add")
        return out.value

    def timer_add_many(self, first_sub: int, n: int, period_ns: int, source_ids=None, source_id0: int = 0, oneshot: bool = False):
        ptr = None
        if source_ids is not None:
            arr = np.ascontiguousarray(source_ids, dtype=np.uint32)
            ptr = arr.ctypes.data
        nat.check(self._lib.cpbus_timer_add_many(self._h, first_sub, n, period_ns, ptr, source_id0, int(oneshot)), "cpbus_timer_add_many")

    def timer_add_list(self, sub_ids, periods_ns, source_ids, oneshot=False) -> tuple[np.ndarray, np.ndarray]:
        """cpbus_timer_add(sub_ids[i], periods_ns[i], source_ids[i], oneshot[i]) in order, in one call: (timer_ids, status),
        the uint32 id of each armed timer (0 where status[i] is not OK) and the int32 status each single call would have
        returned.  `oneshot` is one flag for every timer or one per timer.  Raises on any other return, CPBUS_EAGAIN
        included (nothing was applied)."""
        ids = np.ascontiguousarray(sub_ids, dtype=np.uint32)
        n = ids.size
        specs = np.zeros(n, dtype=nat.TIMER_SPEC_DTYPE)
        specs["sub_id"] = ids
        specs["period_ns"] = np.asarray(periods_ns, dtype=np.uint64)
        specs["source_id"] = np.asarray(source_ids, dtype=np.uint32)
        specs["oneshot"] = np.asarray(oneshot, dtype=bool)
        timer_ids, status = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.int32)
        ptrs = [a.ctypes.data if n else None for a in (specs, timer_ids, status)]
        nat.check(self._lib.cpbus_timer_add_list(self._h, ptrs[0], n, ptrs[1], ptrs[2], None), "cpbus_timer_add_list")
        return timer_ids, status

    def timer_cancel(self, timer_id: int):
        nat.check(self._lib.cpbus_timer_cancel(self._h, timer_id), "cpbus_timer_cancel")

    def timer_cancel_many(self, timer_ids) -> np.ndarray:
        """cpbus_timer_cancel for every id in order, in one call: the per-element statuses (OK or ENOENT)"""
        return self._membership_many("cpbus_timer_cancel_many", [np.ascontiguousarray(timer_ids, dtype=np.uint32)])

    # -- hot path ----------------------------------------------------------
    def publish(self, code: int, source_id: int = 0) -> int:
        ev = nat.Event(0, 0, code, source_id, 0, 0)
        return self._lib.cpbus_publish(self._h, C.byref(ev), 1)

    def publish_many(self, events: np.ndarray) -> int:
        """events: EVENT_DTYPE array (only code/source_id are read)."""
        ev = np.ascontiguousarray(events, dtype=EVENT_DTYPE)
        return self._lib.cpbus_publish(self._h, ev.ctypes.data, ev.size)

    def send(self, sub_id: int, code: int, source_id: int = 0) -> int:
        ev = nat.Event(0, 0, code, source_id, 0, 0)
        return self._lib.cpbus_send(self._h, sub_id, C.byref(ev))

    def advance(self, now_ns: int) -> int:
        return self._lib.cpbus_advance(self._h, now_ns)

    def flush(self) -> int:
        return self._lib.cpbus_flush(self._h)

    def sync(self):
        nat.check(self._lib.cpbus_sync(self._h), "cpbus_sync")

    def publish_device(self, dev_ptr: int, n: int, watermark_ns: int) -> int:
        return self._lib.cpbus_publish_device(self._h, C.c_void_p(dev_ptr), n, watermark_ns)

    def publish_device_staged(self, dev_ptr: int, n: int, watermark_ns: int, next_ptr: int = 0, next_n: int = 0) -> int:
        """dev_ptr / next_ptr may be peer-mapped pointers into another GPU's HBM (fused NVLink ingest)."""
        return self._lib.cpbus_publish_device_staged(self._h, C.c_void_p(dev_ptr), n, watermark_ns,
                                                     C.c_void_p(next_ptr) if next_ptr else None, next_n)

    # -- the publisher's stream across GPUs (one process per GPU) ------------
    def stream_create(self, n_slots: int, n_consumers: int):
        """publisher rank: (stream handle, 64-byte IPC handle for the other ranks)"""
        st, handle = C.c_void_p(), C.create_string_buffer(64)
        nat.check(self._lib.cpbus_stream_create(self._h, n_slots, n_consumers, C.byref(st), handle), "cpbus_stream_create")
        return st, handle.raw

    def stream_open(self, handle: bytes, consumer_index: int):
        st = C.c_void_p()
        nat.check(self._lib.cpbus_stream_open(self._h, handle, consumer_index, C.byref(st)), "cpbus_stream_open")
        return st

    def stream_attach(self, owner_stream, consumer_index: int):
        """same-process consumer of a stream created by another Bus of this process (peer access instead of IPC)"""
        st = C.c_void_p()
        nat.check(self._lib.cpbus_stream_attach(self._h, owner_stream, consumer_index, C.byref(st)), "cpbus_stream_attach")
        return st

    def stream_put(self, st, events: np.ndarray, now_ns: int, raw: bool = False, nowait: bool = False) -> int:
        ev = np.ascontiguousarray(events, dtype=EVENT_DTYPE)
        flags = (nat.PUT_RAW if raw else nat.PUT_STAMP) | (nat.PUT_NOWAIT if nowait else 0)
        return self._lib.cpbus_stream_put(st, ev.ctypes.data if ev.size else None, ev.size, now_ns, flags)

    def stream_fanout(self, st, n: int, now_ns: int) -> int:
        return self._lib.cpbus_stream_fanout(st, n, now_ns)

    def stream_admit(self, st, n: int, now_ns: int) -> int:
        """lossless stream: how many of the current batch's undelivered records this shard can take.  Raises on an error,
        CPBUS_EAGAIN included (an empty remainder whose ticks do not fit, or this bus's own staged events are blocked)."""
        prefix = C.c_size_t()
        nat.check(self._lib.cpbus_stream_admit(st, n, now_ns, C.byref(prefix)), "cpbus_stream_admit")
        return prefix.value

    def stream_fanout_prefix(self, st, n: int, now_ns: int, m: int) -> int:
        """lossless stream: fan out the next m undelivered records; OK = batch complete, EAGAIN = records remain"""
        return self._lib.cpbus_stream_fanout_prefix(st, n, now_ns, m)

    def stream_offer(self, st, prefix: int, stalled: bool = False):
        """lossless stream across processes: post this shard's admitted prefix for the current round (async)"""
        nat.check(self._lib.cpbus_stream_offer(st, prefix, 1 if stalled else 0), "cpbus_stream_offer")

    def stream_agree(self, st) -> int:
        """lossless stream across processes: the minimum of every shard's offer of this round.  Raises on an error,
        CPBUS_EAGAIN included (some shard stalled: drain, then run the round again)."""
        m = C.c_size_t()
        nat.check(self._lib.cpbus_stream_agree(st, C.byref(m)), "cpbus_stream_agree")
        return m.value

    def stream_poll(self, st):
        """(n, now_ns) of the next batch if the publisher has released it, else None — for consumers that are not told"""
        ready, n, now = C.c_int(), C.c_size_t(), C.c_uint64()
        nat.check(self._lib.cpbus_stream_poll(st, C.byref(ready), C.byref(n), C.byref(now)), "cpbus_stream_poll")
        return (n.value, now.value) if ready.value else None

    def stream_fanout_next(self, st) -> int:
        """follower: enqueue the fan-out of the stream's next batch without knowing its shape (n and the watermark come
        from the slot header inside the kernel); returns at once.  Outstanding followers are resolved by the next call
        that reads or changes this bus's host state."""
        return self._lib.cpbus_stream_fanout_next(st)

    def stream_round_next(self, st) -> int:
        """lossless follower: enqueue one admission round (admit, offer, agree, fan out the agreed prefix) on the device for
        this shard's current batch; returns at once.  Every shard must enqueue the same sequence of rounds."""
        return self._lib.cpbus_stream_round_next(st)

    def stream_progress(self, st) -> tuple[int, int, int, int]:
        """resolve outstanding followers and rounds: (status, batches completely fanned out, records of the next batch
        already delivered, rounds that moved nothing).  status is the sticky stream error (OK when none)."""
        b, off, stalled = C.c_uint64(), C.c_size_t(), C.c_uint64()
        rc = self._lib.cpbus_stream_progress(st, C.byref(b), C.byref(off), C.byref(stalled))
        if rc not in (nat.OK, nat.EORDER, nat.ETIMEDOUT):
            nat.check(rc, "cpbus_stream_progress")
        return rc, b.value, off.value, stalled.value

    def stream_status(self, st) -> int:
        return self._lib.cpbus_stream_status(st)

    def stream_set_timeout(self, st, microseconds: int):
        nat.check(self._lib.cpbus_stream_set_timeout(st, microseconds), "cpbus_stream_set_timeout")

    def stream_close(self, st):
        nat.check(self._lib.cpbus_stream_close(st), "cpbus_stream_close")

    def shared_alloc(self, nbytes: int):
        """(device pointer, 64-byte IPC handle) of a new buffer on this bus's GPU, mappable by the other GPUs."""
        ptr, handle = C.c_void_p(), C.create_string_buffer(64)
        nat.check(self._lib.cpbus_shared_alloc(self._h, nbytes, C.byref(ptr), handle), "cpbus_shared_alloc")
        return ptr.value, handle.raw

    def shared_open(self, handle: bytes) -> int:
        ptr = C.c_void_p()
        nat.check(self._lib.cpbus_shared_open(self._h, handle, C.byref(ptr)), "cpbus_shared_open")
        return ptr.value

    def shared_close(self, ptr: int):
        nat.check(self._lib.cpbus_shared_close(self._h, C.c_void_p(ptr)), "cpbus_shared_close")

    # -- consumer side -----------------------------------------------------
    def drain(self, sub_id: int, cap: int | None = None):
        cap = cap or self.ring_cap
        out = np.zeros(cap, dtype=EVENT_DTYPE)
        n, lost = C.c_size_t(), C.c_uint64()
        nat.check(self._lib.cpbus_drain(self._h, sub_id, out.ctypes.data, cap, C.byref(n), C.byref(lost)), "cpbus_drain")
        return out[: n.value]

    def consume_all(self):
        """device-side consumer: every mailbox read to the end, records discarded"""
        nat.check(self._lib.cpbus_consume_all(self._h), "cpbus_consume_all")

    def drain_many(self, first_sub: int, n: int, cap: int, out=None):
        """Bulk drain: returns (records, offsets, counts); mailbox i's FIFO run is records[offsets[i]:offsets[i]+counts[i]].
        `out`: a preallocated EVENT_DTYPE array of at least `cap` records (pinned memory makes the D2H a straight DMA)."""
        if out is None:
            out = np.zeros(cap, dtype=EVENT_DTYPE)
        offs, cnts = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint32)
        total = C.c_size_t()
        nat.check(self._lib.cpbus_drain_many(self._h, first_sub, n, out.ctypes.data, cap, offs.ctypes.data, cnts.ctypes.data,
                                             C.byref(total)), "cpbus_drain_many")
        return out, offs, cnts

    def drain_ready(self, first_sub: int, n: int, start_sub: int, cap: int, ready_cap: int, out=None):
        """Sparse drain of mailboxes [first_sub, first_sub+n) in cyclic order from start_sub: returns (records, ready,
        next_sub).  ready is a READY_DTYPE array with one entry per mailbox taken; entry i's FIFO run is
        records[ready[i].offset : ready[i].offset + ready[i].count].  Pass next_sub back as start_sub to continue.
        `out`: a preallocated EVENT_DTYPE array of at least `cap` records; records is a view of it."""
        return self._ready_call("cpbus_drain_ready", first_sub, n, start_sub, cap, ready_cap, out)

    def take_ready(self, first_sub: int, n: int, start_sub: int, cap: int, ready_cap: int, out=None):
        """Lossless mode: drain_ready that keeps the records' room until ack_many releases it (the records stay held in
        their mailboxes and count against them).  Same arguments and return shape as drain_ready."""
        return self._ready_call("cpbus_take_ready", first_sub, n, start_sub, cap, ready_cap, out)

    def _ready_call(self, name: str, first_sub: int, n: int, start_sub: int, cap: int, ready_cap: int, out):
        if out is None:
            out = np.zeros(cap, dtype=EVENT_DTYPE)
        if len(out) < cap:
            raise ValueError("out holds fewer than cap records")
        ready = np.zeros(min(ready_cap, n), dtype=READY_DTYPE)
        n_ready, total, next_sub = C.c_size_t(), C.c_size_t(), C.c_uint32()
        nat.check(getattr(self._lib, name)(self._h, first_sub, n, start_sub, out.ctypes.data, cap, ready.ctypes.data,
                                           ready_cap, C.byref(n_ready), C.byref(total), C.byref(next_sub)), name)
        return out[: total.value], ready[: n_ready.value], next_sub.value

    @_SingleBusOnly
    def drain_ready_begin(self, first_sub: int, n: int, start_sub: int, cap: int, ready_cap: int) -> int:
        """drain_ready enqueued on the bus stream: returns a ticket for drain_ready_end, which returns what drain_ready
        would have returned here.  At most 8 tickets are outstanding (a 9th begin raises with ENOSPC)."""
        return self._ready_begin("cpbus_drain_ready_begin", first_sub, n, start_sub, cap, ready_cap)

    @_SingleBusOnly
    def take_ready_begin(self, first_sub: int, n: int, start_sub: int, cap: int, ready_cap: int) -> int:
        """Lossless mode: take_ready enqueued on the bus stream; collect it with drain_ready_end."""
        return self._ready_begin("cpbus_take_ready_begin", first_sub, n, start_sub, cap, ready_cap)

    def _ready_begin(self, name: str, first_sub: int, n: int, start_sub: int, cap: int, ready_cap: int) -> int:
        t = C.c_uint32()
        nat.check(getattr(self._lib, name)(self._h, first_sub, n, start_sub, cap, ready_cap, C.byref(t)), name)
        # the entries _end can return: min(ready_cap, n), as drain_ready sizes its list
        self.__dict__.setdefault("_ticket_rows", {})[t.value] = min(ready_cap, n)
        return t.value

    @_SingleBusOnly
    def drain_ready_end(self, ticket: int, cap: int, ready_cap: int, out=None):
        """Waits for the ticket of drain_ready_begin or take_ready_begin and returns (records, ready, next_sub), as
        drain_ready does; cap and ready_cap are at least the begin's.  `out`: a preallocated EVENT_DTYPE array of at least
        `cap` records; records is a view of it."""
        if out is None:
            out = np.zeros(cap, dtype=EVENT_DTYPE)
        if len(out) < cap:
            raise ValueError("out holds fewer than cap records")
        rows = self.__dict__.get("_ticket_rows", {})
        ready = np.zeros(max(1, min(ready_cap, rows.get(ticket, ready_cap))), dtype=READY_DTYPE)
        n_ready, total, next_sub = C.c_size_t(), C.c_size_t(), C.c_uint32()
        nat.check(self._lib.cpbus_drain_ready_end(self._h, ticket, out.ctypes.data, cap, ready.ctypes.data, ready_cap,
                                                  C.byref(n_ready), C.byref(total), C.byref(next_sub)), "cpbus_drain_ready_end")
        rows.pop(ticket, None)
        return out[: total.value], ready[: n_ready.value], next_sub.value

    def ack_many(self, sub_ids, counts) -> np.ndarray:
        """Lossless mode: release the oldest counts[i] held records of sub_ids[i], in order, in one call: the int32 status
        of each element (OK, ENOENT for an unknown id, EINVAL for more than the mailbox holds at that element's turn)."""
        ids, cnt = np.ascontiguousarray(sub_ids, dtype=np.uint32), np.ascontiguousarray(counts, dtype=np.uint32)
        if ids.shape != cnt.shape:
            raise ValueError("sub_ids and counts differ in length")
        return self._membership_many("cpbus_ack_many", [ids, cnt])

    def lagging(self, first_sub: int, n: int, start_sub: int | None = None, min_backlog: int = 1, cap: int | None = None):
        """Read-only consumer backlog of mailboxes [first_sub, first_sub+n) in cyclic order from start_sub (default
        first_sub): returns (entries, next_sub, summary).  entries is a LAG_DTYPE array of the first `cap` (default n)
        subscribed mailboxes with backlog >= min_backlog; next_sub continues the walk; summary is a dict over the whole
        range (active, lagging, backlog_total, backlog_max, lost_total, hist)."""
        start_sub = first_sub if start_sub is None else start_sub
        cap = n if cap is None else cap
        out = np.zeros(max(1, min(cap, n)), dtype=nat.LAG_DTYPE)
        n_out, next_sub, s = C.c_size_t(), C.c_uint32(), nat.LagSummary()
        nat.check(self._lib.cpbus_lagging(self._h, first_sub, n, start_sub, min_backlog, out.ctypes.data if cap else None, cap,
                                          C.byref(n_out), C.byref(next_sub), C.byref(s)), "cpbus_lagging")
        summary = {k: getattr(s, k) for k, _ in nat.LagSummary._fields_ if k != "hist"}
        summary["hist"] = list(s.hist)
        return out[: n_out.value], next_sub.value, summary

    def blockers(self, cap: int | None = None) -> np.ndarray:
        """Lossless mode: the global ids of the mailboxes the next flush cannot get past, ascending (the first `cap`;
        default all of them).  Empty in throughput mode."""
        n = C.c_size_t()
        want = 1024 if cap is None else cap
        while True:
            out = np.zeros(max(1, want), dtype=np.uint32)
            nat.check(self._lib.cpbus_blockers(self._h, out.ctypes.data if want else None, want, C.byref(n)), "cpbus_blockers")
            if cap is not None or n.value <= want:   # (the query changes no state: asking again gives the same list)
                return out[: min(want, n.value)]
            want = n.value

    def stream_blockers(self, st, cap: int | None = None) -> np.ndarray:
        """Lossless stream shard: the global ids of the mailboxes that give this shard an admissible prefix of 0 for its
        current batch, ascending (the first `cap`; default all of them).  Empty in throughput mode and while the publisher
        has not released the batch."""
        n = C.c_size_t()
        want = 1024 if cap is None else cap
        while True:
            out = np.zeros(max(1, want), dtype=np.uint32)
            nat.check(self._lib.cpbus_stream_blockers(st, out.ctypes.data if want else None, want, C.byref(n)),
                      "cpbus_stream_blockers")
            if cap is not None or n.value <= want:   # (the query changes no state: asking again gives the same list)
                return out[: min(want, n.value)]
            want = n.value

    def peek_window(self, sub_id: int, cap: int | None = None) -> np.ndarray:
        cap = cap or self.ring_cap
        out = np.zeros(cap, dtype=EVENT_DTYPE)
        n = C.c_size_t()
        nat.check(self._lib.cpbus_peek_window(self._h, sub_id, out.ctypes.data, cap, C.byref(n)), "cpbus_peek_window")
        return out[: n.value]

    def digests(self, first_sub: int, n: int):
        out = np.zeros(n, dtype=[("count", "<u8"), ("digest", "<u8")])
        nat.check(self._lib.cpbus_digest(self._h, first_sub, n, out.ctypes.data), "cpbus_digest")
        return out

    def digest_fold(self, first_sub: int, n: int):
        out = (C.c_uint64 * 4)()
        nat.check(self._lib.cpbus_digest_fold(self._h, first_sub, n, C.byref(out)), "cpbus_digest_fold")
        return tuple(out)

    def digest_fold_begin(self, first_sub: int, n: int) -> int:
        t = C.c_uint32()
        nat.check(self._lib.cpbus_digest_fold_begin(self._h, first_sub, n, C.byref(t)), "cpbus_digest_fold_begin")
        return t.value

    def digest_fold_end(self, ticket: int):
        out = (C.c_uint64 * 4)()
        nat.check(self._lib.cpbus_digest_fold_end(self._h, ticket, C.byref(out)), "cpbus_digest_fold_end")
        return tuple(out)

    def step_result_begin(self) -> int:
        t = C.c_uint32()
        nat.check(self._lib.cpbus_step_result_begin(self._h, C.byref(t)), "cpbus_step_result_begin")
        return t.value

    def step_result_end(self, ticket: int):
        out = (C.c_uint64 * 4)()
        nat.check(self._lib.cpbus_step_result_end(self._h, ticket, C.byref(out)), "cpbus_step_result_end")
        return tuple(out)

    def debug_events(self):
        out = np.zeros(10, dtype=EVENT_DTYPE)
        n = C.c_size_t()
        nat.check(self._lib.cpbus_debug_events(self._h, out.ctypes.data, 10, C.byref(n)), "cpbus_debug_events")
        return out[: n.value]

    def stats(self) -> dict:
        st = nat.Stats()
        nat.check(self._lib.cpbus_stats(self._h, C.byref(st)), "cpbus_stats")
        d = {k: getattr(st, k) for k, _ in nat.Stats._fields_ if k != "published_by_code"}
        d["published_by_code"] = list(st.published_by_code)
        return d

    def publish_counts(self) -> dict:
        """{(code, source_id): count} — the reference's containerpilot_events{code, source} counter (Metric excluded)"""
        n = C.c_size_t()
        nat.check(self._lib.cpbus_publish_counts(self._h, None, 0, C.byref(n)), "cpbus_publish_counts")
        buf = (nat.PairCount * max(1, n.value))()
        nat.check(self._lib.cpbus_publish_counts(self._h, buf, n.value, C.byref(n)), "cpbus_publish_counts")
        return {(buf[i].code, buf[i].source_id): buf[i].count for i in range(n.value)}

    def device_ptrs(self) -> dict:
        ring, ctl = C.c_void_p(), C.c_void_p()
        nat.check(self._lib.cpbus_device_ptrs(self._h, C.byref(ring), C.byref(ctl)), "cpbus_device_ptrs")
        return {"ring": ring.value, "ctl": ctl.value}
