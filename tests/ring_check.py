"""Whole-fleet ring parity: every mailbox's ring memory against a plain reference built on the device.  Test infrastructure.

The per-mailbox digest is computed from the staged batch, not read back from the ring, so a record stored to the wrong
slot, with its halves swapped or from the wrong plane leaves counts and digests right.  `check` reads the rings
themselves: it wraps `cpbus_device_ptrs` in zero-copy torch views (ring int64 [N, R, 4], control blocks int64 [N, 4] =
{tail, head, digest, mask|pad}, DESIGN.md §3) and compares them, a chunk of mailboxes at a time, with the image that
`FleetModel.expected` builds from what the test published.  The reference shares no code with the kernels: a match
matrix, cumulative positions, ticks merged by (due, slot) in front of the records with ts >= due, and the last
min(count, R) records at slot j & (R - 1).  `FleetModel.pin` checks the reference itself against the C oracle."""
from __future__ import annotations

import contextlib

import numpy as np
import torch

import oracle_binding as ob

TARGET_ALL, F_TICK, TIMER_EXPIRED, N_CODES = 0xFFFFFFFF, 0x1, 8, 17
MASK_ALL = (1 << N_CODES) - 1
low_water = {"free_bytes": None}   # the least free device memory any check() saw


class _DeviceArray:
    """A device pointer as a __cuda_array_interface__ object (no ownership: the bus owns the memory)."""

    def __init__(self, ptr: int, shape: tuple[int, ...]):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "<i8", "data": (ptr, False), "strides": None,
                                         "version": 3}


@contextlib.contextmanager
def fleet_views(ptrs: dict, n_subs: int, ring_cap: int):
    """(ring int64 [n_subs, ring_cap, 4], ctl int64 [n_subs, 4]) over the bus's own memory, from `bus.device_ptrs()`.
    Use inside the bus's lifetime; on exit both views are emptied, so they cannot outlive it."""
    dev = torch.device("cuda", torch.cuda.current_device())
    ring = torch.as_tensor(_DeviceArray(ptrs["ring"], (n_subs, ring_cap, 4)), device=dev)
    ctl = torch.as_tensor(_DeviceArray(ptrs["ctl"], (n_subs, 4)), device=dev)
    try:
        yield ring, ctl
    finally:
        ring.set_(); ctl.set_()


class FleetModel:
    """What a fresh bus (tails at 0, subscribers 0..n_subs-1 subscribed in order, never unsubscribed) was given.
    Mailbox i holds global id sub_id_base + i (a shard of a sharded bus): unicast records and tick targets use that id.

    records: EVENT_DTYPE array in publish order, as the rings hold them (seq, ts, code, source_id, target, flags), ts
        non-decreasing; batches: [(first, end, watermark)] in order, how they reached the bus (for the oracle).
    masks: uint32 [n] code masks; pair_shapes / shape_of (optional): uint32 [S, 16, 2] exact {code, source} cases (unused
        rows 0xFFFFFFFF) and the shape index of each subscriber.
    timers: one dict per timer slot, in slot order: period (uint64 [n]), source (uint32 [n]), oneshot (bool); every timer
        armed at clock 0 on every subscriber."""

    def __init__(self, n_subs, ring_cap, records, batches, masks, pair_shapes=None, shape_of=None, timers=(), sub_id_base=0):
        self.n, self.R, self.base = n_subs, ring_cap, sub_id_base
        self.records, self.batches = np.ascontiguousarray(records), list(batches)
        assert (np.diff(self.records["ts_ns"].astype(np.int64)) >= 0).all(), "records must be in clock order"
        self.watermark = max([int(w) for _, _, w in self.batches] + [int(self.records["ts_ns"].max(initial=0))])
        self.masks = np.asarray(masks, dtype=np.uint32) & np.uint32(MASK_ALL)
        self.pair_shapes, self.shape_of = pair_shapes, shape_of
        self.timers = list(timers)
        self._dev = {}

    def _on(self, device):
        if device not in self._dev:
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
            rec = t(self.records.view(np.int64).reshape(-1, 4))
            d = {"rec": rec, "masks": t(self.masks.astype(np.int64)),
                 "timers": [(t(tm["period"].astype(np.int64)), t(tm["source"].astype(np.int64)), bool(tm["oneshot"]))
                            for tm in self.timers]}
            code, src, target = rec[:, 2] & 0xFFFFFFFF, rec[:, 2] >> 32, rec[:, 3] & 0xFFFFFFFF
            d["bcast"] = target == TARGET_ALL
            d["mask_bit"] = code.clamp(max=N_CODES)   # a code past the enum is matched by no mask bit (bit 17 is never set)
            d["target"] = torch.where(d["bcast"], torch.full_like(target, -1), target)
            if self.pair_shapes is not None:
                sh = t(self.pair_shapes.astype(np.int64))                                        # [S, 16, 2]
                hit = (sh[:, :, None, 0] == code[None, None, :]) & (sh[:, :, None, 1] == src[None, None, :])
                d["shape_match"] = hit.any(1) & d["bcast"][None, :]                              # [S, E]
                d["shape_of"] = t(np.asarray(self.shape_of, dtype=np.int64))
            self._dev[device] = d
        return self._dev[device]

    def chunk(self) -> int:
        """mailboxes per reference chunk: about 2^25 (mailbox, record) pairs"""
        return max(1, min(self.n, 1 << max(0, (2 ** 25 // max(1, len(self.records))).bit_length() - 1)))

    def expected(self, g0: int, g1: int, device):
        """(count [C], image int64 [C * R, 4], written bool [C * R]) of mailboxes [g0, g1) (indices, not global ids)"""
        d, R, C = self._on(device), self.R, g1 - g0
        rec, E = d["rec"], len(self.records)
        gid = torch.arange(self.base + g0, self.base + g1, device=device, dtype=torch.int64)
        ts = rec[:, 1].contiguous()
        match = (((d["masks"][g0:g1, None] >> d["mask_bit"][None, :]) & 1) != 0) & d["bcast"][None, :]
        if "shape_match" in d:
            match |= d["shape_match"][d["shape_of"][g0:g1]]
        match |= d["target"][None, :] == gid[:, None]                       # unicast records bypass both filter levels
        cum = torch.cumsum(match, 1, dtype=torch.int64)                       # matches up to and including record i
        n_rec = cum[:, -1] if E else torch.zeros(C, dtype=torch.int64, device=device)
        # ticks: slot-major columns, then a stable sort by due time = order by (due, slot)
        dues, seqs, srcs = [], [], []
        for period, source, oneshot in d["timers"]:
            p = period[g0:g1]
            fires = torch.div(self.watermark, p, rounding_mode="floor")
            if oneshot:
                fires = fires.clamp(max=1)
            f = torch.arange(1, int(fires.max()) + 1 if C else 1, device=device, dtype=torch.int64)
            due = p[:, None] * f[None, :]
            dues.append(torch.where(f[None, :] <= fires[:, None], due, torch.iinfo(torch.int64).max))
            seqs.append((f - 1)[None, :].expand(C, -1)); srcs.append(source[g0:g1, None].expand(-1, len(f)))
        if dues and sum(x.shape[1] for x in dues):
            due, order = torch.sort(torch.cat(dues, 1), dim=1, stable=True)
            seq, tsrc = torch.cat(seqs, 1).gather(1, order), torch.cat(srcs, 1).gather(1, order)
            live = due != torch.iinfo(torch.int64).max
            n_tick = live.sum(1)
            ticks_before = torch.searchsorted(due, ts[None, :].expand(C, -1).contiguous(), right=True)   # due <= ts
            rec_pos = cum - match.long() + ticks_before
            cum0 = torch.cat([torch.zeros(C, 1, dtype=torch.int64, device=device), cum], 1)
            tick_pos = cum0.gather(1, torch.searchsorted(ts, due)) + torch.arange(due.shape[1], device=device)[None, :]
        else:
            live = None
            n_tick = torch.zeros(C, dtype=torch.int64, device=device)
            rec_pos = cum - match.long()
        count = n_rec + n_tick
        first = (count - R)[:, None]                                          # older positions were overwritten
        image = torch.zeros(C * R, 4, dtype=torch.int64, device=device)
        written = torch.zeros(C * R, dtype=torch.bool, device=device)
        ci, ei = (match & (rec_pos >= first)).nonzero(as_tuple=True)
        at = ci * R + (rec_pos[ci, ei] & (R - 1))
        image[at] = rec[ei]; written[at] = True
        if live is not None:
            ci, ti = (live & (tick_pos >= first)).nonzero(as_tuple=True)
            at = ci * R + (tick_pos[ci, ti] & (R - 1))
            image[at] = torch.stack([seq[ci, ti], due[ci, ti], TIMER_EXPIRED | (tsrc[ci, ti] << 32), gid[ci] | (F_TICK << 32)], 1)
            written[at] = True
        return count, image, written

    def window(self, i: int, device="cpu") -> np.ndarray:
        """the reference's last min(count, R) records of mailbox i, oldest first"""
        count, image, _ = self.expected(i, i + 1, device)
        c = int(count[0])
        slots = torch.arange(max(0, c - self.R), c, device=device) & (self.R - 1)
        return image[slots].cpu().numpy().view(ob.EVENT_DTYPE).reshape(-1)

    def oracle_for_one(self, i: int) -> ob.Oracle:
        """the C oracle's view of mailbox i alone: a 1-subscriber oracle at sub_id_base = its global id, fed the same
        batches"""
        gid = self.base + i
        orc = ob.Oracle(1, timers_per_sub=len(self.timers), keep_window=self.R, sub_id_base=gid)
        pairs = None
        if self.pair_shapes is not None:
            rows = self.pair_shapes[self.shape_of[i]]
            pairs = [(int(c), int(s)) for c, s in rows if c != 0xFFFFFFFF]
        orc.subscribe(int(self.masks[i]), pairs)
        for tm in self.timers:
            orc.timer_add(gid, int(tm["period"][i]), int(tm["source"][i]), bool(tm["oneshot"]))
        for a, b, w in self.batches:
            assert orc.publish_records(self.records[a:b], int(w)) == 0
        return orc

    def pin(self, mailboxes):
        """the reference against the C oracle on sampled mailboxes (indices): it is not a second unchecked implementation"""
        for i in mailboxes:
            i, gid = int(i), self.base + int(i)
            orc = self.oracle_for_one(i)
            want = orc.mailbox(gid)
            got = self.window(i)
            assert len(got) == min(orc.count(gid), self.R), f"reference count at mailbox {gid}"
            assert got.tobytes() == want.tobytes(), f"reference window differs from the oracle at mailbox {gid}"


def check(views, model: FleetModel) -> int:
    """Every mailbox: tail == expected count, and every slot the reference writes equals the ring word for word.
    Raises AssertionError naming the first mailbox (by global id), slot and word that differ.  Returns the slots compared."""
    ring, ctl = views
    R, C, compared = model.R, model.chunk(), 0
    for g0 in range(0, model.n, C):
        g1 = min(model.n, g0 + C)
        count, image, written = model.expected(g0, g1, ring.device)
        tail = ctl[g0:g1, 0]
        bad = (tail != count).nonzero()
        if len(bad):
            i = int(bad[0])
            raise AssertionError(f"mailbox {model.base + g0 + i}: tail {int(tail[i])}, expected count {int(count[i])}")
        diff = (ring[g0:g1].reshape(-1, 4) != image) & written[:, None]
        if bool(diff.any()):
            at, w = (int(x) for x in diff.nonzero()[0])
            got = int(ring[g0:g1].reshape(-1, 4)[at, w])
            raise AssertionError(f"mailbox {model.base + g0 + at // R} slot {at % R} word {w}: ring {got & (2**64 - 1):#018x}, "
                                 f"expected {int(image[at, w]) & (2**64 - 1):#018x}")
        compared += int(written.sum())
        free = torch.cuda.mem_get_info()[0]
        if low_water["free_bytes"] is None or free < low_water["free_bytes"]:
            low_water["free_bytes"] = free
    return compared
