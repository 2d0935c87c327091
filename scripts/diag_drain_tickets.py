"""Drain tickets against the synchronous drain: what a pump step costs when its drain is begun after the flush and ended
one step later (cpbus_drain_ready_begin / cpbus_drain_ready_end), against cpbus_drain_ready at the same place.

Fleets: the Job-shaped fleet of scripts/bridge_sparse.py at each size of --subs, 512-event batches from host buffers on
twin buses.  A pump step is publish + flush + one drain call from the previous call's next_sub + handing each run to its
channel (a copy of the run).  The synchronous twin drains with cpbus_drain_ready; the pipelined twin begins its ticket
after the flush and ends the previous step's ticket before handing its runs on.  The two paths alternate in blocks of
--block steps; the pipelined twin ends its last ticket inside the block, so each block does the same work on both.
Reported: the median over blocks of the mean step time, and the range.  Parity: every subscriber's records are the same on
both twins.  Also the dense bridge shape (8,192 mailboxes x 512 records into pinned host memory): cpbus_drain_ready
against _begin + _end, in records/s, alternating.  Prints one JSON line with the card's name and power limit; exits 3
when a parity check fails.  Writes nothing.

  python scripts/diag_drain_tickets.py [--blocks 20 --block 10 --subs 32768 1048576]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np
import torch

from bridge_sparse import card, job_fleet
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE, READY_DTYPE


def pinned(n_rec, dtype):
    t = torch.empty((n_rec * dtype.itemsize,), dtype=torch.uint8).pin_memory()
    return t, t.numpy().view(dtype)


def stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))}


class Pump:
    """One bus and its pump: sync (cpbus_drain_ready) or pipelined (ticket begun after the flush, ended a step later)."""

    def __init__(self, lib, bus, n_subs, cap, ready_cap, pipelined):
        self.lib, self.bus, self.n, self.cap, self.ready_cap, self.pipelined = lib, bus, n_subs, cap, ready_cap, pipelined
        self.t_out, self.out = pinned(cap, EVENT_DTYPE)
        self.t_rdy, self.rdy = pinned(ready_cap, READY_DTYPE)
        self.n_ready, self.total, self.nxt, self.ticket = C.c_size_t(), C.c_size_t(), C.c_uint32(), C.c_uint32()
        self.start, self.pending, self.got = 0, False, {}

    def _hand(self):
        for e in self.rdy[:self.n_ready.value]:
            o = int(e["offset"])
            self.got.setdefault(int(e["sub_id"]), []).append(self.out[o:o + int(e["count"])].copy())
        self.start = self.nxt.value

    def _end(self, ticket):
        nat.check(self.lib.cpbus_drain_ready_end(self.bus._h, ticket, self.out.ctypes.data, self.cap, self.rdy.ctypes.data,
                                                 self.ready_cap, C.byref(self.n_ready), C.byref(self.total),
                                                 C.byref(self.nxt)), "cpbus_drain_ready_end")
        self._hand()

    def step(self, batch):
        nat.check(self.bus.publish_many(batch), "cpbus_publish"); nat.check(self.bus.flush(), "cpbus_flush")
        if not self.pipelined:
            nat.check(self.lib.cpbus_drain_ready(self.bus._h, 0, self.n, self.start, self.out.ctypes.data, self.cap,
                                                 self.rdy.ctypes.data, self.ready_cap, C.byref(self.n_ready),
                                                 C.byref(self.total), C.byref(self.nxt)), "cpbus_drain_ready")
            self._hand()
            return
        # the ticket starts where the last one ended stopped (every record is taken once whatever the start)
        prev, had = self.ticket.value, self.pending
        nat.check(self.lib.cpbus_drain_ready_begin(self.bus._h, 0, self.n, self.start, self.cap, self.ready_cap,
                                                   C.byref(self.ticket)), "cpbus_drain_ready_begin")
        if had:
            self._end(prev)
        self.pending = True

    def finish(self):
        if self.pending:
            self._end(self.ticket.value)
            self.pending = False


def fleet_leg(lib, n_subs, args):
    B, R = 512, 512
    masks, rows, cnt, n_src = job_fleet(n_subs)
    rng = np.random.default_rng(0xD7A1 + n_subs)
    n_steps = (args.blocks + 1) * args.block
    host = np.zeros(2 * n_steps * B, dtype=EVENT_DTYPE)
    host["code"] = rng.integers(1, 17, len(host)); host["source_id"] = rng.integers(0, n_src, len(host))
    pumps = []
    for pipelined in (False, True):
        bus = Bus(n_subs, ring_cap=R, batch_cap=R // 2, digest=False, device=args.device)
        first = C.c_uint32()
        nat.check(lib.cpbus_subscribe_pairs_many(bus._h, masks.ctypes.data, rows.ctypes.data, cnt.ctypes.data, n_subs,
                                                 C.byref(first)), "cpbus_subscribe_pairs_many")
        pumps.append(Pump(lib, bus, n_subs, 1 << 16, 4096, pipelined))
    times = [[], []]
    step = [0, 0]
    for blk in range(args.blocks + 1):                     # block 0 of each path is warm-up
        for leg in ((0, 1) if blk % 2 == 0 else (1, 0)):
            p = pumps[leg]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.block):
                i = step[leg]; step[leg] += 1
                p.step(host[i * B:(i + 1) * B])
            p.finish()
            dt = (time.perf_counter() - t0) / args.block
            if blk:
                times[leg].append(dt * 1e6)
    for p in pumps:   # the rest of what arrived, so that both have every record
        while True:
            nat.check(lib.cpbus_drain_ready(p.bus._h, 0, n_subs, 0, p.out.ctypes.data, p.cap, p.rdy.ctypes.data,
                                            p.ready_cap, C.byref(p.n_ready), C.byref(p.total), C.byref(p.nxt)), "drain")
            if not p.n_ready.value:
                break
            p._hand()
    same = pumps[0].got.keys() == pumps[1].got.keys() and all(
        np.concatenate(pumps[0].got[s]).tobytes() == np.concatenate(pumps[1].got[s]).tobytes() for s in pumps[0].got)
    recs = sum(len(r) for parts in pumps[1].got.values() for r in parts)
    for p in pumps:
        p.bus.close()
    return {"subscribers": n_subs, "us_per_step_sync": stats(times[0]), "us_per_step_pipelined": stats(times[1]),
            "records_per_step": recs / step[1], "identical_per_subscriber": bool(same)}


def dense_leg(lib, args):
    n_drain, R2 = 8192, 1024
    bus = Bus(n_drain, ring_cap=R2, batch_cap=512, digest=False, device=args.device)
    bus.subscribe_many(np.full(n_drain, nat.MASK_ALL, dtype=np.uint32))
    cap = n_drain * 512
    t_out, out = pinned(cap, EVENT_DTYPE)
    t_rdy, rdy = pinned(n_drain, READY_DTYPE)
    n_ready, total, nxt, ticket = C.c_size_t(), C.c_size_t(), C.c_uint32(), C.c_uint32()
    host = np.zeros(512, dtype=EVENT_DTYPE)
    host["code"] = np.arange(512) % 16 + 1
    times, ok, split = [[], []], True, [[], []]
    for rep in range(2 * args.dense_reps + 4):
        for leg in ((0, 1) if rep % 2 == 0 else (1, 0)):
            host["source_id"] = rep * 2 + leg
            nat.check(bus.publish_many(host), "cpbus_publish"); nat.check(bus.flush(), "cpbus_flush"); bus.sync()
            t0 = time.perf_counter()
            if leg == 0:
                nat.check(lib.cpbus_drain_ready(bus._h, 0, n_drain, 0, out.ctypes.data, cap, rdy.ctypes.data, n_drain,
                                                C.byref(n_ready), C.byref(total), C.byref(nxt)), "cpbus_drain_ready")
            else:
                nat.check(lib.cpbus_drain_ready_begin(bus._h, 0, n_drain, 0, cap, n_drain, C.byref(ticket)), "begin")
                torch.cuda.synchronize()   # the gather into the ticket's buffer is done ...
                t1 = time.perf_counter()   # ... and _end is the host copy alone
                nat.check(lib.cpbus_drain_ready_end(bus._h, ticket.value, out.ctypes.data, cap, rdy.ctypes.data, n_drain,
                                                    C.byref(n_ready), C.byref(total), C.byref(nxt)), "end")
                if rep >= 4:
                    split[0].append((t1 - t0) * 1e3); split[1].append((time.perf_counter() - t1) * 1e3)
            dt = time.perf_counter() - t0
            ok = ok and n_ready.value == n_drain and total.value == n_drain * 512
            ok = ok and bool((out["source_id"][:total.value] == rep * 2 + leg).all())
            if rep >= 4:                                           # the first calls allocate staging and ticket buffers
                times[leg].append(n_drain * 512 / dt)
    bus.close()
    del t_out, t_rdy
    return {"workload": f"{n_drain} mailboxes x 512 records -> pinned host memory, one call",
            "records_per_s_sync": stats(times[0]), "records_per_s_ticket": stats(times[1]),
            "ticket_ms_begin_to_gather_done": stats(split[0]), "ticket_ms_end_host_copy": stats(split[1]), "ok": ok}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=20, help="timed blocks per path and fleet size")
    ap.add_argument("--block", type=int, default=10, help="steps per block")
    ap.add_argument("--dense-reps", type=int, default=10)
    ap.add_argument("--subs", type=int, nargs="+", default=[32_768, 1_048_576])
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("diag_drain_tickets.py: no CUDA device; cpbus has no CPU fallback")
    torch.cuda.set_device(args.device)
    lib = nat.load()
    legs = [fleet_leg(lib, n, args) for n in args.subs]
    dense = dense_leg(lib, args)
    ok = dense["ok"] and all(l["identical_per_subscriber"] for l in legs)
    res = {"name": "drain-tickets", "unit": "us per pump step (publish + flush + drain + hand-off), host clock",
           "legs": legs, "dense": dense, "parity_checked": bool(ok), "gpu": card(args.device)}
    print(json.dumps(res), flush=True)
    if not ok:
        sys.exit(3)


if __name__ == "__main__":
    main()
