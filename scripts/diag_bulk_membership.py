"""Host ms of a membership change over many ids: the loop of single calls (cpbus_unsubscribe / cpbus_set_mask /
cpbus_timer_cancel, one flush + copy + synchronise each) against one bulk call (cpbus_*_many: one flush, one copy, one
membership_kernel launch, one synchronise), alternated in blocks in one run.

Fleet: 1,048,576 subscribers (mask all codes, 64-record rings), one periodic 1 s timer each, throughput mode, dense and with
CPBUS_CFG_SPARSE_TICKS | CPBUS_CFG_SPARSE_RECORDS.  Shapes: unsubscribe 10^3 / 10^4 / 10^5 scattered ids, re-mask 10^5
scattered ids, cancel 10^5 scattered timers.  Each call kind runs on a fleet of its own, and every unsubscribe and cancel takes ids no
earlier one touched (a re-mask sets the same mask again on the same ids).  Each round measures the loop, then the bulk call.  Rows give the median and the
min..max over the rounds, and name the card and its power limit.  A run without a GPU stops.
Usage: python scripts/diag_bulk_membership.py [--subs 1048576] [--rounds 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from containerpilot_b200 import _native as nat  # noqa: E402
from containerpilot_b200.bus import Bus  # noqa: E402

R, B, PERIOD = 64, 32, 1_000_000_000
SHAPES = [("unsubscribe", 1_000), ("unsubscribe", 10_000), ("unsubscribe", 100_000), ("set_mask", 100_000),
          ("timer_cancel", 100_000)]


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else "unknown card"


def _fleet(N, sparse):
    bus = Bus(N, ring_cap=R, batch_cap=B, timers_per_sub=1, digest=True, device=0, sparse_records=sparse)
    bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
    bus.timer_add_many(0, N, PERIOD, source_id0=1)   # timer id of subscriber s = s (K = 1, first arming)
    nat.check(bus.flush(), "flush")
    return bus


def _loop(bus, kind, ids):
    if kind == "unsubscribe":
        for i in ids:
            bus.unsubscribe(int(i))
    elif kind == "set_mask":
        for i in ids:
            bus.set_mask(int(i), 0x3FF)
    else:
        for i in ids:
            bus.timer_cancel(int(i))


def _bulk(bus, kind, ids):
    if kind == "unsubscribe":
        st = bus.unsubscribe_many(ids)
    elif kind == "set_mask":
        st = bus.set_mask_many(ids, np.full(ids.size, 0x3FF, dtype=np.uint32))
    else:
        st = bus.timer_cancel_many(ids)
    assert (st == nat.OK).all()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subs", type=int, default=1 << 20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no GPU: nothing is measured")
    card, N = _card(), args.subs
    rows = []
    for sparse in (False, True):
        mode = "sparse_ticks|sparse_records" if sparse else "dense"
        fleets = {kind: _fleet(N, sparse) for kind in ("unsubscribe", "set_mask", "timer_cancel")}
        perm = np.random.default_rng(7).permutation(N).astype(np.uint32)
        used = {"unsubscribe": 0, "timer_cancel": 0}
        times = {(k, n): {"loop": [], "bulk": []} for k, n in SHAPES}
        for _ in range(args.rounds):
            for kind, n in SHAPES:
                for how in ("loop", "bulk"):
                    bus = fleets[kind]
                    if kind == "set_mask":
                        ids = perm[:n] if how == "bulk" else perm[n:2 * n]
                    else:
                        ids = perm[used[kind]:used[kind] + n]
                        used[kind] += n
                    t0 = time.perf_counter()
                    (_loop if how == "loop" else _bulk)(bus, kind, ids)
                    times[(kind, n)][how].append((time.perf_counter() - t0) * 1e3)
        for bus in fleets.values():
            bus.close()
        for kind, n in SHAPES:
            t = times[(kind, n)]
            row = {"mode": mode, "call": kind, "ids": n, "subs": N, "rounds": args.rounds, "card": card,
                   "loop_ms": float(np.median(t["loop"])), "loop_range": [min(t["loop"]), max(t["loop"])],
                   "bulk_ms": float(np.median(t["bulk"])), "bulk_range": [min(t["bulk"]), max(t["bulk"])]}
            rows.append(row)
            print(f"{mode:28s} {kind:13s} {n:>7d} ids: loop {row['loop_ms']:9.2f} ms [{row['loop_range'][0]:.2f}..."
                  f"{row['loop_range'][1]:.2f}]  bulk {row['bulk_ms']:7.3f} ms [{row['bulk_range'][0]:.3f}..."
                  f"{row['bulk_range'][1]:.3f}]  ({card})", flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
