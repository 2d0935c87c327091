"""Host µs per publish + flush ending in a device synchronise, on a bus with sparse record delivery
(CPBUS_CFG_SPARSE_RECORDS) and on a twin with sparse timer delivery only (CPBUS_CFG_SPARSE_TICKS), alternated in blocks in
one run.  Throughput mode, 1,024-record rings, 512-event batches.

Shapes:
  job       a Job-shaped fleet (masks.JobSwitch.cases(): the switch's code mask and exact cases, the diag_pairs.py shape)
            with random events over the fleet's sources: 1-event publishes (the Go shim flushes inside every Publish) and
            512-event batches
  sweep     a fleet whose code k (k = 1..) is subscribed by exactly 4^(k-1) mailboxes, up to N/32, the rest on a code that is
            never published: one event of code k per flush reaches exactly that many mailboxes (1-event rows) and a 512-event
            batch of it 512 times as many records (past the caps the flagged bus runs the full fan-out, like its twin)
  allones   every mailbox all-ones: a broadcast code's count is past the cap, so planning ends at the first record
Medians over the timed steps of each bus; every row names the card and its power limit.  A run without a GPU stops.
Usage: python scripts/diag_sparse_records.py [--jobs 32768,1048576] [--steps 200] [--rounds 3] [--out FILE]
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
from containerpilot_b200 import events as ev  # noqa: E402
from containerpilot_b200 import masks as mk  # noqa: E402
from containerpilot_b200.bus import Bus, EVENT_DTYPE  # noqa: E402

R, B = 1024, 512
FIXED = {"": 0, "global": 1, "closed": 2, "SIGHUP": 3, "SIGUSR2": 4}


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else "unknown card"


def _sid(name):
    if name in FIXED:
        return FIXED[name]
    base, _, suffix = name.partition(".")
    if base == "check":
        return 5 + 5 * int(suffix[3:]) + 1
    return 5 + 5 * int(base[3:]) + {"": 0, "heartbeat": 2, "run-every": 3, "wait-timeout": 4}[suffix]


def _job_fleet(N):
    rng = np.random.default_rng(7)
    ms, cases = [], []
    for j in range(N):
        dep = int(rng.integers(0, N))
        sw = mk.JobSwitch(f"job{j}", start_event=ev.Event(ev.ExitSuccess, f"job{dep}") if j % 3 else ev.GlobalStartup)
        m, cs = sw.cases()
        ms.append(m)
        cases.append([(e.Code, _sid(e.Source)) for e in cs])
    return ms, cases


def _bus(N, flagged):
    return Bus(N, ring_cap=R, batch_cap=B, digest=True, device=0, sparse_ticks=True, sparse_records=flagged)


def _time(buses, batches, steps, rounds):
    """median host µs per publish + flush + sync of each bus, the buses alternated in blocks of `steps`"""
    t = {k: [] for k in buses}
    i = 0
    for _ in range(rounds):
        for k, bus in buses.items():
            for _ in range(steps):
                e = batches[i % len(batches)]
                i += 1
                t0 = time.perf_counter()
                nat.check(bus.publish_many(e), "publish"); nat.check(bus.flush(), "flush"); bus.sync()
                t[k].append(time.perf_counter() - t0)
            bus.consume_all()
    return {k: float(np.median(v)) * 1e6 for k, v in t.items()}


def _launch_share(bus, batches):
    st0 = bus.stats()
    for e in batches:
        nat.check(bus.publish_many(e), "publish"); nat.check(bus.flush(), "flush")
    bus.sync()
    st1 = bus.stats()
    n = len(batches)
    return {"fanouts_per_flush": (st1["batches"] - st0["batches"]) / n,
            "deliveries_per_flush": (st1["deliveries"] - st0["deliveries"]) / n}


def _events(rng, n, codes, n_src, k):
    out = []
    for _ in range(k):
        e = np.zeros(n, dtype=EVENT_DTYPE)
        e["code"] = rng.choice(codes, n) if isinstance(codes, list) else codes
        e["source_id"] = rng.integers(0, n_src, n)
        out.append(e)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", default="32768,1048576")
    ap.add_argument("--sweep", type=int, default=1048576)
    ap.add_argument("--allones", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = _card()
    rows = []

    def emit(row):
        row["card"] = card
        rows.append(row)
        print(json.dumps(row), flush=True)

    rng = np.random.default_rng(11)
    for N in [int(x) for x in a.jobs.split(",") if x]:
        ms, cases = _job_fleet(N)
        buses = {"flagged": _bus(N, True), "twin": _bus(N, False)}
        for bus in buses.values():
            bus.subscribe_pairs_many(ms, cases)
        for n in (1, B):
            batches = _events(rng, n, list(range(1, 17)), 5 + 5 * N, 64)
            us = _time(buses, batches, a.steps, a.rounds)
            emit({"shape": "job", "subscribers": N, "events_per_flush": n, "us_flagged": round(us["flagged"], 1),
                  "us_twin": round(us["twin"], 1), **_launch_share(buses["flagged"], batches[:16])})
        for bus in buses.values():
            bus.close()

    N = a.sweep
    sizes, masks, lo = [], np.full(N, 1 << 16, dtype=np.uint32), 0
    k = 1
    while 4 ** (k - 1) <= N // 32 and k < 16:
        masks[lo: lo + 4 ** (k - 1)] = 1 << k
        sizes.append((k, 4 ** (k - 1)))
        lo += 4 ** (k - 1)
        k += 1
    buses = {"flagged": _bus(N, True), "twin": _bus(N, False)}
    for bus in buses.values():
        bus.subscribe_many(masks)
    for code, size in sizes:
        for n in (1, B):
            batches = _events(rng, n, code, 64, 4)
            us = _time(buses, batches, a.steps // 2, a.rounds)
            emit({"shape": "sweep", "subscribers": N, "mailboxes_per_flush": size, "events_per_flush": n,
                  "us_flagged": round(us["flagged"], 1), "us_twin": round(us["twin"], 1),
                  **_launch_share(buses["flagged"], batches)})
    for bus in buses.values():
        bus.close()

    N = a.allones
    buses = {"flagged": _bus(N, True), "twin": _bus(N, False)}
    for bus in buses.values():
        bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
    for n in (1, B):
        batches = _events(rng, n, list(range(1, 17)), 64, 16)
        us = _time(buses, batches, a.steps, a.rounds)
        emit({"shape": "allones", "subscribers": N, "events_per_flush": n, "us_flagged": round(us["flagged"], 1),
              "us_twin": round(us["twin"], 1), **_launch_share(buses["flagged"], batches)})
    for bus in buses.values():
        bus.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
