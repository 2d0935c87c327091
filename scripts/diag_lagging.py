"""µs per call of the consumer backlog queries: `cpbus_lagging` (summary only, and with every lagging entry) and
`cpbus_blockers`, beside `cpbus_drain_ready` with nothing ready, which reads the same control blocks.

Lossless buses of 65,536 and 1,048,576 subscribers with 1,024-record rings (2 GiB and 32 GiB), with and without one armed
timer per subscriber (due far in the future: the scans read the timer slots, nothing fires).  A fraction of 0 %, 0.1 % or
100 % of the mailboxes is filled to the brim (1,024 records): those are lagging, and they block the staged event that every
blockers call evaluates.  Each timing is host time around one library call, which ends in a device synchronise; medians
over --reps calls after --warmup untimed ones, every case in one run.  Every row names the card and its power limit; a run
without a GPU prints "not measured".  Usage: python scripts/diag_lagging.py [--reps 50] [--warmup 5] [--out FILE]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from containerpilot_b200 import _native as nat  # noqa: E402
from containerpilot_b200.bus import Bus, EVENT_DTYPE, READY_DTYPE  # noqa: E402

R, BATCH = 1024, 512


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown card"
    except Exception:
        return "unknown card"


def _median_us(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return round(float(np.median(t)) * 1e6, 1)


def _case(n, frac, timers, reps, warmup):
    bus = Bus(n, ring_cap=R, batch_cap=BATCH, timers_per_sub=1 if timers else 0, lossless=True, digest=False, device=0)
    try:
        lib, h = bus._lib, bus._h
        n_lag = int(round(n * frac))
        masks = np.zeros(n, dtype=np.uint32)
        masks[np.linspace(0, n - 1, n_lag).astype(np.int64) if n_lag else []] = nat.MASK_ALL
        bus.subscribe_many(masks)
        if timers:
            bus.timer_add_many(0, n, 1 << 60, source_id0=1)
        ready = np.zeros(1024, dtype=READY_DTYPE)
        recs = np.zeros(R, dtype=EVENT_DTYPE)
        n_ready, total, nxt = C.c_size_t(), C.c_size_t(), C.c_uint32()
        # baseline before any record exists: drain_ready finds nothing ready and reads every control block
        base = _median_us(lambda: nat.check(lib.cpbus_drain_ready(h, 0, n, 0, recs.ctypes.data, R, ready.ctypes.data, 1024,
                                                                   C.byref(n_ready), C.byref(total), C.byref(nxt)),
                                            "cpbus_drain_ready"), reps, warmup)
        ev = np.zeros(BATCH, dtype=EVENT_DTYPE)
        ev["code"] = 1
        for _ in range(R // BATCH):                 # fill the lagging mailboxes to the brim
            nat.check(bus.publish_many(ev), "publish")
            nat.check(bus.flush(), "flush")
        nat.check(bus.publish(1, 0), "publish")     # staged: the unit every blockers call evaluates
        bus.sync()
        lag = np.zeros(max(1, n_lag), dtype=nat.LAG_DTYPE)
        blk = np.zeros(max(1, n_lag), dtype=np.uint32)
        n_out, summ = C.c_size_t(), nat.LagSummary()
        summary_only = _median_us(lambda: nat.check(lib.cpbus_lagging(h, 0, n, 0, 1, None, 0, C.byref(n_out), C.byref(nxt),
                                                                      C.byref(summ)), "cpbus_lagging"), reps, warmup)
        assert summ.lagging == n_lag and summ.backlog_max == (R if n_lag else 0)
        entries = _median_us(lambda: nat.check(lib.cpbus_lagging(h, 0, n, 0, 1, lag.ctypes.data, n_lag, C.byref(n_out),
                                                                 C.byref(nxt), C.byref(summ)), "cpbus_lagging"), reps, warmup)
        assert n_out.value == n_lag
        k0 = bus.stats()["kernel_launches"]
        blockers = _median_us(lambda: nat.check(lib.cpbus_blockers(h, blk.ctypes.data, n_lag, C.byref(n_out)),
                                                "cpbus_blockers"), reps, warmup)
        assert n_out.value == n_lag
        launched = bus.stats()["kernel_launches"] > k0
        return {"us_drain_ready_nothing_ready": base, "us_lagging_summary": summary_only, "us_lagging_entries": entries,
                "us_blockers": blockers, "blockers_kernel": launched, "lagging": n_lag}
    finally:
        bus.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sizes", default="65536,1048576")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    gpu = torch.cuda.is_available() and torch.cuda.device_count() > 0
    card = _card() if gpu else "no GPU"
    rows = []
    for n in [int(x) for x in a.sizes.split(",")]:
        for timers in (False, True):
            for frac in (0.0, 0.001, 1.0):
                row = {"subscribers": n, "ring_cap": R, "timers": timers, "lagging_fraction": frac, "card": card}
                if not gpu:
                    row["result"] = "not measured"
                else:
                    row.update(_case(n, frac, timers, a.reps, a.warmup))
                rows.append(row)
                print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
