"""Host ms of arming many timers: the loop of cpbus_timer_add (a flush and two synchronised copies each) against one
cpbus_timer_add_list (one flush, one copy, one timer_arm_kernel launch, one synchronise), alternated in one run.

Fleet: 1,048,576 subscribers (mask all codes, 64-record rings, one timer slot each), throughput mode, dense and with
CPBUS_CFG_SPARSE_TICKS | CPBUS_CFG_SPARSE_RECORDS.  Shapes: 10^3, 10^4 and 10^5 timers on scattered owners that no earlier
arming touched, periods of 1-10 s, one in seven one-shot.  Each round measures the loop, then the list call.  Then the whole
fleet: 2^20 timers, one per subscriber in shuffled order, in one list call on a fresh bus, once per round.  Rows give the
median and the min..max over the rounds, and name the card and its power limit.  A run without a GPU stops.
Usage: python scripts/diag_timer_add_list.py [--subs 1048576] [--rounds 3] [--out FILE]
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

R, B = 64, 32
SHAPES = [1_000, 10_000, 100_000]


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else "unknown card"


def _fleet(N, sparse):
    bus = Bus(N, ring_cap=R, batch_cap=B, timers_per_sub=1, digest=True, device=0, sparse_records=sparse)
    bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
    nat.check(bus.flush(), "flush")
    return bus


def _timers(rng, owners):
    periods = rng.integers(1, 11, owners.size).astype(np.uint64) * 1_000_000_000
    return owners, periods, (1000 + owners).astype(np.uint32), rng.random(owners.size) < 1 / 7


def _loop(bus, owners, periods, sources, oneshot):
    for s, p, src, one in zip(owners.tolist(), periods.tolist(), sources.tolist(), oneshot.tolist()):
        bus.timer_add(s, p, src, one)


def _list(bus, owners, periods, sources, oneshot):
    _, st = bus.timer_add_list(owners, periods, sources, oneshot)
    assert (st == nat.OK).all()


def _row(mode, what, n, N, t, card, rounds):
    row = {"mode": mode, "timers": n, "subs": N, "rounds": rounds, "card": card}
    for how, v in t.items():
        row[how + "_ms"], row[how + "_range"] = float(np.median(v)), [min(v), max(v)]
    text = "  ".join(f"{how} {row[how + '_ms']:9.3f} ms [{row[how + '_range'][0]:.3f}...{row[how + '_range'][1]:.3f}]"
                     for how in t)
    print(f"{mode:28s} {what:11s} {n:>8d} timers: {text}  ({card})", flush=True)
    return row


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
    if 2 * sum(SHAPES) * args.rounds > N:
        sys.exit("too few subscribers for fresh owners in every round")
    rows = []
    for sparse in (False, True):
        mode = "sparse_ticks|sparse_records" if sparse else "dense"
        rng = np.random.default_rng(7)
        perm = rng.permutation(N).astype(np.uint32)
        used = 0
        times = {n: {"loop": [], "list": []} for n in SHAPES}
        with _fleet(N, sparse) as bus:
            for _ in range(args.rounds):
                for n in SHAPES:
                    for how in ("loop", "list"):
                        arm = _timers(rng, perm[used:used + n])
                        used += n
                        t0 = time.perf_counter()
                        (_loop if how == "loop" else _list)(bus, *arm)
                        times[n][how].append((time.perf_counter() - t0) * 1e3)
        for n in SHAPES:
            rows.append(_row(mode, "scattered", n, N, times[n], card, args.rounds))
        whole = {"list": []}
        for _ in range(args.rounds):
            with _fleet(N, sparse) as bus:
                arm = _timers(rng, rng.permutation(N).astype(np.uint32))
                t0 = time.perf_counter()
                _list(bus, *arm)
                whole["list"].append((time.perf_counter() - t0) * 1e3)
        rows.append(_row(mode, "whole fleet", N, N, whole, card, args.rounds))
    if args.out:
        with open(args.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
