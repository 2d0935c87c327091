"""Consumer-side parity: what every consumer call must return, computed from a snapshot of the bus's own memory.  Test
infrastructure, the consumer half of `tests/ring_check.py`.

The consumer calls never write a ring, so an exact answer follows from the control blocks and rings as they stand just
before a call, plus what the test itself knows: each mailbox's take cursor T, which mailboxes are subscribed, the timers it
armed and the record it staged.  The producer is not modelled (`ring_check.check` pins it).  The reference is plain torch
on the views' device and shares no code with the kernels: cursors, a boolean ready mask, the walk as a rolled index,
`cumsum`, and one gather of ring slots (cur + j) & (R - 1).  `tests/test_drain_reference.py` pins it to the C oracle.

A `Fleet` is (ring int64 [n, R, 4], ctl int64 [n, 4] = {tail, head, digest, mask|pad}) of one shard whose mailbox i is
global id base + i; both may be live views (`ring_check.fleet_views`) or CPU tensors.  Calls take `ctl` separately, a
snapshot (`ctl.clone()`) taken before the call, so that the answer is the one for that point in stream order."""
from __future__ import annotations

import numpy as np
import torch

from containerpilot_b200.bus import READY_DTYPE
from containerpilot_b200 import _native as nat
from test_oracle_semantics import py_record_hash

ACTIVE_BIT = 1 << 31
TILE = 1024                       # positions per tile of the device scans (kThreads * kReadyItems)


class Fleet:
    """sync: for views of a live bus, its `sync` (the bus runs on a stream of its own, which torch's stream does not wait
    for); every Snapshot calls it first, so no snapshot can read the memory while a launch still writes it"""

    def __init__(self, ring, ctl, base: int, lossless: bool, sync=None):
        self.ring, self.ctl, self.base, self.lossless = ring, ctl, int(base), bool(lossless)
        self.sync = sync
        self.n, self.R = ring.shape[0], ring.shape[1]
        self.dev = ring.device
        self.taken = torch.zeros(self.n, dtype=torch.int64, device=self.dev)   # take cursors T (0 at subscribe)

    # -- cursors ------------------------------------------------------------------------------------------------------
    def walk(self, first: int, n: int, start: int):
        """local mailbox at each walk position: [first, first + n) in cyclic id order from start"""
        l0, rot = first - self.base, start - first
        assert 0 <= l0 and l0 + n <= self.n and 0 <= rot < n
        return l0 + (torch.arange(n, device=self.dev, dtype=torch.int64) + rot) % n

    def cursor(self, ctl, loc, mode: str):
        """(tail, head, cur) of mailboxes loc; mode 'drain' (head, or max(head, tail - R) in throughput mode) or 'take'
        (max(T, head)); 'lag': the drain cursor"""
        tail, head = ctl[loc, 0], ctl[loc, 1]
        if mode == "take":
            cur = torch.maximum(self.taken[loc], head)
        elif not self.lossless:
            cur = torch.maximum(head, tail - self.R)
        else:
            cur = head
        return tail, head, cur

    # -- drain_ready / take_ready / their tickets ---------------------------------------------------------------------
    def expected_ready(self, ctl, first: int, n: int, start: int, cap: int, ready_cap: int, mode: str = "drain") -> dict:
        """cpbus_drain_ready (mode 'drain') or cpbus_take_ready ('take'): ready mailboxes in walk order while their whole run
        fits into cap records and ready_cap entries; the first that does not fit ends the call.  Returns out (int64
        [total, 4] on the device), ready (READY_DTYPE), total, next_sub, cut (walk position of the mailbox that ended the
        call, None when all were taken), pos (walk position of every entry), loc (their local ids) and tail."""
        loc = self.walk(first, n, start)
        tail, head, cur = self.cursor(ctl, loc, mode)
        cnt = tail - cur
        rp = (cnt > 0).nonzero().squeeze(1)                    # ready positions, ascending
        csum = torch.cumsum(cnt[rp], 0)
        fits = (torch.arange(len(rp), device=self.dev) < ready_cap) & (csum <= cap)
        k = int(fits.sum())                                    # both conditions are monotone: a prefix fits
        assert bool(fits[:k].all())
        cut = int(rp[k]) if k < len(rp) else None
        p = rp[:k]
        count, lp = cnt[p], loc[p]
        offset = csum[:k] - count
        total = int(csum[k - 1]) if k else 0
        lost = (cur - head)[p] if mode == "drain" and not self.lossless else torch.zeros_like(count)
        ready = np.zeros(k, dtype=READY_DTYPE)
        ready["sub_id"], ready["count"] = (lp + self.base).cpu().numpy(), count.cpu().numpy()
        ready["offset"], ready["lost"] = offset.cpu().numpy(), lost.cpu().numpy()
        e = torch.repeat_interleave(torch.arange(k, device=self.dev), count)
        j = torch.arange(total, device=self.dev) - offset[e]
        out = self.ring[lp[e], (cur[p][e] + j) & (self.R - 1)]
        next_sub = start if cut is None else first + (start - first + cut) % n
        return {"out": out, "ready": ready, "total": total, "next_sub": next_sub, "cut": cut, "pos": p, "loc": lp,
                "tail": tail[p], "n_ready_all": len(rp), "csum": csum, "rp": rp}

    def took(self, want: dict, mode: str):
        """after a take: T = tail of every mailbox it took (a drain moves head, which the control blocks show)"""
        if mode == "take":
            self.taken[want["loc"]] = want["tail"]

    # -- lagging ------------------------------------------------------------------------------------------------------
    def expected_lagging(self, ctl, subscribed, first: int, n: int, start: int, min_backlog: int, cap: int) -> dict:
        """cpbus_lagging: the first cap subscribed mailboxes in walk order with backlog >= min_backlog (LAG_DTYPE), next_sub
        and the summary over every subscribed mailbox of the range (hist[0]: backlog 0, hist[k]: [2^(k-1), 2^k))"""
        loc = self.walk(first, n, start)
        tail, head, cur = self.cursor(ctl, loc, "lag")
        act = subscribed[loc]
        backlog, lost = tail - cur, cur - head
        sel = act & (backlog >= min_backlog)
        sp = sel.nonzero().squeeze(1)
        taken = sp[:cap]
        out = np.zeros(len(taken), dtype=nat.LAG_DTYPE)
        out["sub_id"] = (loc[taken] + self.base).cpu().numpy()
        out["backlog"], out["lost"] = backlog[taken].cpu().numpy(), lost[taken].cpu().numpy()
        next_sub = start if len(sp) <= cap else first + (start - first + int(sp[cap])) % n
        b = backlog[act]
        bucket = (b[:, None] >= (1 << torch.arange(32, device=self.dev, dtype=torch.int64))[None, :]).sum(1)   # bit length
        hist = torch.bincount(bucket, minlength=33)
        summary = {"active": int(act.sum()), "lagging": int(sel.sum()), "backlog_total": int(b.sum()),
                   "backlog_max": int(b.max()) if len(b) else 0, "lost_total": int(lost[act].sum()),
                   "hist": [int(x) for x in hist.cpu()]}
        return {"out": out, "next_sub": next_sub, "summary": summary}

    # -- ack_many -----------------------------------------------------------------------------------------------------
    def expected_acks(self, ctl, ids, counts, known) -> dict:
        """cpbus_ack_many, element by element: ENOENT for an id outside the shard or not handed out (known[l] False: never
        subscribed, or released), OK for count 0, else OK when count <= held = max(T, head) - head after the earlier
        elements of the same call (head += count), EINVAL otherwise.  Returns status (int32), applied, heads {local: head}."""
        head = {}
        tk = self.taken.cpu().numpy()
        hd = ctl[:, 1].cpu().numpy()
        known = known.cpu().numpy()
        status = np.zeros(len(ids), dtype=np.int32)
        for i, (g, c) in enumerate(zip(np.asarray(ids, dtype=np.int64), np.asarray(counts, dtype=np.int64))):
            l = int(g) - self.base
            if l < 0 or l >= self.n or not known[l]:
                status[i] = nat.ENOENT
                continue
            if c == 0:
                continue
            h = head.get(l, int(hd[l]))
            if c <= max(int(tk[l]), h) - h:
                head[l] = h + int(c)
            else:
                status[i] = nat.EINVAL
        return {"status": status, "applied": int((status == nat.OK).sum()), "heads": head}

    # -- blockers -----------------------------------------------------------------------------------------------------
    def expected_blockers(self, ctl, subscribed, takes_record, clock: int, timers=()) -> np.ndarray:
        """cpbus_blockers of a lossless bus: a subscribed mailbox blocks when its share of the next unit U exceeds its room
        R - (tail - head).  takes_record: bool [n], whether it takes U's staged record (None: nothing staged); timers: one
        (first due int64 [n], period int64 [n], armed bool [n]) per slot, periodic; its ticks due by clock count."""
        share = torch.zeros(self.n, dtype=torch.int64, device=self.dev)
        for due, period, armed in timers:
            fire = armed & (due <= clock)
            share += torch.where(fire, torch.div(clock - due, period, rounding_mode="floor") + 1, torch.zeros_like(due))
        if takes_record is not None:
            share += takes_record.long()
        room = self.R - torch.clamp(ctl[:, 0] - ctl[:, 1], max=self.R)
        block = subscribed & (share > room)
        return (block.nonzero().squeeze(1) + self.base).cpu().numpy().astype(np.uint32)

    # -- digest_fold --------------------------------------------------------------------------------------------------
    def expected_fold(self, ctl, first: int, n: int) -> tuple:
        """(sum of tails, sum of digests, XOR of H(digest, count, id), n) mod 2^64, H = the record hash of {seq = digest,
        ts = count, code = id, 0...}"""
        l0 = first - self.base
        c = ctl[l0:l0 + n].cpu().numpy().view(np.uint64)
        tail, dig = c[:, 0].copy(), c[:, 2].copy()
        gid = np.arange(first, first + n, dtype=np.uint64)
        z = np.zeros(n, dtype=np.uint64)
        h = py_record_hash(dig, tail, gid, z, z, z)
        return (int(tail.sum(dtype=np.uint64)), int(dig.sum(dtype=np.uint64)), int(np.bitwise_xor.reduce(h)), n)


# -- comparison -------------------------------------------------------------------------------------------------------
def assert_ready_equal(got, want: dict, what: str = ""):
    """(records, ready, next_sub) of a ready call against expected_ready: names the first entry, mailbox and record that
    differ"""
    rec, rdy, nxt = got
    wr = want["ready"]
    if len(rdy) != len(wr) or rdy.tobytes() != wr.tobytes():
        k = min(len(rdy), len(wr))
        bad = np.flatnonzero(rdy[:k].view(np.uint8).reshape(k, -1) != wr[:k].view(np.uint8).reshape(k, -1))
        i = int(bad[0]) // READY_DTYPE.itemsize if len(bad) else k
        g = rdy[i] if i < len(rdy) else None
        w = wr[i] if i < len(wr) else None
        raise AssertionError(f"{what} entry {i} of {len(wr)}: got {g}, expected {w} (mailbox "
                             f"{int((w if w is not None else g)['sub_id'])})")
    wo = want["out"].cpu().numpy()
    go = rec.view(np.int64).reshape(-1, 4)
    if go.shape != wo.shape or not np.array_equal(go, wo):
        k = min(len(go), len(wo))
        rows = np.flatnonzero((go[:k] != wo[:k]).any(1))
        r = int(rows[0]) if len(rows) else k
        e = int(np.searchsorted(wr["offset"].astype(np.int64), r, side="right")) - 1
        raise AssertionError(f"{what} record {r} (entry {e}, mailbox {int(wr[e]['sub_id'])}, run record "
                             f"{r - int(wr[e]['offset'])}): got {go[r] if r < len(go) else None}, "
                             f"expected {wo[r] if r < len(wo) else None}")
    assert nxt == want["next_sub"], f"{what} next_sub {nxt}, expected {want['next_sub']}"


class Snapshot:
    """Control blocks (a copy) and a chunked, position-weighted checksum of the rings (they are 2 GiB at 1M x 64), taken
    in stream order: after every launch the bus has queued (fleet.sync), and complete before its next one"""
    CHUNK = 1 << 14

    def __init__(self, fleet: Fleet):
        if fleet.sync is not None:
            fleet.sync()
        self.ctl = fleet.ctl.clone()
        self.ring = ring_sums(fleet.ring, self.CHUNK)
        if self.ring.is_cuda:
            torch.cuda.synchronize()         # complete before the bus's next launch, which runs on a stream of its own


_weights = {}


def ring_sums(ring, chunk: int) -> torch.Tensor:
    n, R = ring.shape[0], ring.shape[1]
    key = (ring.device, chunk * R * 4)
    if key not in _weights:
        g = torch.Generator().manual_seed(0x5EED)
        _weights[key] = (torch.randint(0, 1 << 62, (chunk * R * 4,), generator=g, dtype=torch.int64) | 1).to(ring.device)
    w = _weights[key]
    sums = []
    for g0 in range(0, n, chunk):
        x = ring[g0:g0 + chunk].reshape(-1)
        sums.append((x * w[:len(x)]).sum())
    return torch.stack(sums)


def assert_unchanged(before: Snapshot, after: Snapshot, base: int, heads=None):
    """Control blocks byte-identical but for the heads a call may move (heads: {local: new head}, or a (loc, head) pair of
    tensors), and every ring chunk's checksum unchanged.  Names the first mailbox and word that differ."""
    a, b = before.ctl, after.ctl.clone()
    if heads is not None:
        loc, h = heads if isinstance(heads, tuple) else (
            torch.tensor(list(heads.keys()), dtype=torch.int64), torch.tensor(list(heads.values()), dtype=torch.int64))
        loc, h = loc.to(b.device), h.to(b.device)
        moved = b[loc, 1]
        bad = (moved != h).nonzero()
        if len(bad):
            i = int(bad[0])
            raise AssertionError(f"mailbox {base + int(loc[i])}: head {int(moved[i])}, expected {int(h[i])}")
        b[loc, 1] = a[loc, 1]
    diff = (a != b).nonzero()
    if len(diff):
        i, w = (int(x) for x in diff[0])
        raise AssertionError(f"mailbox {base + i} control word {w} changed: {int(a[i, w])} -> {int(b[i, w])}")
    bad = (before.ring != after.ring).nonzero()
    if len(bad):
        c = int(bad[0])
        raise AssertionError(f"ring memory of mailboxes {base + c * Snapshot.CHUNK} .. {base + (c + 1) * Snapshot.CHUNK - 1} "
                             "changed")


# -- geometry: what a cell claims to reach ----------------------------------------------------------------------------
def chunk_geometry(ready) -> dict:
    """Where the ticket gather's 16-record chunks fall on the runs of a ready list"""
    off, cnt = ready["offset"].astype(np.int64), ready["count"].astype(np.int64)
    end = off + cnt
    total = int(end[-1]) if len(end) else 0
    ones = np.bincount(off[cnt == 1] // 16, minlength=1) if (cnt == 1).any() else np.zeros(1, dtype=np.int64)
    return {"inside": bool(((off // 16) < ((end - 1) // 16)).any()),            # a boundary 16c inside a run
            "at_start": bool(((off % 16 == 0) & (off > 0)).any()),              # ... at a run's first record
            "at_end": bool(((end % 16 == 0) & (end < total)).any()),            # ... just past a run's last record
            "ones_chunk": bool((ones >= 16).any()),                             # a chunk of 16 runs of one record
            "long_run": bool((((end - 1) // 16 - off // 16) >= 3).any()),       # a run over four or more chunks
            "total_mod_16": total % 16}
