"""Host µs per pump step (cpbus_advance by 1 ms + cpbus_flush + cpbus_drain_ready, which ends in a device synchronise) on a
bus with sparse timer delivery (CPBUS_CFG_SPARSE_TICKS) and on an unflagged twin, alternated in blocks in one run.

Shapes (throughput mode, one timer per subscriber, 512-record rings, 256-event batches):
  sparse     periods spread over 1-10 s (1,024 distinct periods), the clock past 10 s: ~N/5,500 ticks due per step
  sparse+pub the same with one 512-event publish every 100 steps
  density    period 1,024 / 128 / 32 ms with phases staggered over the period: exactly N/1,024, N/128 or N/32 due slots per
             step (past max(32, N/1,024) due slots the flagged bus runs the full fan-out, like its twin)
  dense      a 1 kHz timer each (the config-3 shape): every slot due every step, the full fan-out plus the host index's pass
Medians over the timed steps of each bus; every row names the card and its power limit.  A run without a GPU stops.
Usage: python scripts/diag_sparse_ticks.py [--subs 65536,1048576] [--steps 300] [--rounds 4] [--out FILE]
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
from containerpilot_b200.bus import Bus, EVENT_DTYPE  # noqa: E402

R, B, MS = 512, 256, 1_000_000


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else "unknown card"


def _fleet(N, sparse, shape):
    bus = Bus(N, ring_cap=R, batch_cap=B, timers_per_sub=1, digest=True, device=0, sparse_ticks=sparse)
    bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
    if shape in ("sparse", "sparse+pub"):
        chunk = N // 1024
        for c in range(1024):
            bus.timer_add_many(c * chunk, chunk, MS * 1000 + c * (9000 * MS // 1023), source_id0=c * chunk)
        now = 10_000 * MS
        nat.check(bus.advance(now), "advance"); nat.check(bus.flush(), "flush")
    elif shape.startswith("density"):
        P = int(shape.split("/")[1])            # period in steps; N/P slots due per step
        chunk = N // P
        for c in range(P):                      # chunk c armed at step c: due at c + P, c + 2P, ...
            nat.check(bus.advance(c * MS), "advance")
            bus.timer_add_many(c * chunk, chunk, P * MS, source_id0=c * chunk)
        now = 2 * P * MS
        nat.check(bus.advance(now), "advance"); nat.check(bus.flush(), "flush")
    else:                                       # dense: 1 kHz each
        bus.timer_add_many(0, N, MS, source_id0=0)
        now = 0
    bus.consume_all(); bus.sync()
    return bus, now


def _steps(bus, st, n, pub_every, out, ready_cap):
    ev = np.zeros(512, dtype=EVENT_DTYPE)
    ev["code"] = 5
    t = []
    for i in range(n):
        t0 = time.perf_counter()
        st["now"] += MS
        nat.check(bus.advance(st["now"]), "advance")
        if pub_every and st["i"] % pub_every == 0:
            nat.check(bus.publish_many(ev), "publish")
        nat.check(bus.flush(), "flush")
        rec, ready, st["next"] = bus.drain_ready(0, bus.N, st["next"], len(out), ready_cap, out=out)
        t.append(time.perf_counter() - t0)
        st["i"] += 1
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subs", default="65536,1048576")
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--shapes", default="sparse,sparse+pub,density/1024,density/128,density/32,dense")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = _card()
    rows = []
    for N in [int(x) for x in a.subs.split(",")]:
        for shape in a.shapes.split(","):
            buses = {}
            for sparse in (True, False):
                bus, now = _fleet(N, sparse, shape)
                bus.N = N
                buses[sparse] = (bus, {"now": now, "i": 0, "next": 0})
            out = np.zeros(max(4 * R, 2 * N if shape == "dense" else 64 * 1024), dtype=EVENT_DTYPE)
            pub_every = 100 if shape == "sparse+pub" else 0
            times = {True: [], False: []}
            launches = {}
            ready_cap = N if shape == "dense" else min(N, 65536)
            for sparse in (True, False):   # warm-up
                _steps(buses[sparse][0], buses[sparse][1], 20, pub_every, out, ready_cap)
            for r in range(a.rounds):
                for sparse in ((True, False) if r % 2 == 0 else (False, True)):
                    bus, st = buses[sparse]
                    k0 = bus.stats()["kernel_launches"]
                    times[sparse] += _steps(bus, st, a.steps // a.rounds, pub_every, out, ready_cap)
                    launches[sparse] = launches.get(sparse, 0) + bus.stats()["kernel_launches"] - k0
            row = {"card": card, "subs": N, "shape": shape,
                   "sparse_us": round(float(np.median(times[True])) * 1e6, 1),
                   "plain_us": round(float(np.median(times[False])) * 1e6, 1),
                   "sparse_p90_us": round(float(np.percentile(times[True], 90)) * 1e6, 1),
                   "plain_p90_us": round(float(np.percentile(times[False], 90)) * 1e6, 1),
                   "sparse_launches_per_step": round(launches[True] / len(times[True]), 3),
                   "plain_launches_per_step": round(launches[False] / len(times[False]), 3),
                   "ticks_equal": buses[True][0].stats()["ticks"] == buses[False][0].stats()["ticks"]}
            print(json.dumps(row), flush=True)
            rows.append(row)
            for bus, _ in buses.values():
                bus.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
