"""What subscriber id reuse costs and saves, on one GPU.

1. Host ms of a churn of k scattered ids (k = 10^3, 10^4, 10^5) on a fleet of 1,048,576 subscribers (mask all codes,
   64-record rings, throughput mode), dense and with CPBUS_CFG_SPARSE_TICKS | CPBUS_CFG_SPARSE_RECORDS:
   cpbus_unsubscribe_many + cpbus_release_many + cpbus_subscribe_list (the ids come back), against cpbus_unsubscribe_many +
   cpbus_subscribe_many into spare fresh capacity (a bus of 2^20 + 3 * 10^5 slots).  Every churn takes ids no earlier one
   of its round touched.  Each round measures both, alternated.
2. us per full fan-out (one broadcast record: publish + flush, 200 steps timed on the host clock with one synchronise at the
   end) on a fleet of N live subscribers
   after each has been churned once: with reuse the ids stay [0, N) (n_next = N); without it the live ids are [N, 2N) on a
   bus of 2N slots, and every fan-out walks the N dead slots too.
Rows give the median and min..max over the rounds and name the card and its power limit.  A run without a GPU stops.
Usage: python scripts/diag_subscriber_reuse.py [--subs 1048576] [--rounds 3] [--out FILE]
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

R, B = 64, 32
SIZES = (1_000, 10_000, 100_000)


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else "unknown card"


def _ms(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def churn(N, rounds, sparse):
    spare = 3 * max(SIZES)
    rows = {k: {"reuse": [], "fresh": []} for k in SIZES}
    rng = np.random.default_rng(1)
    for _ in range(rounds):
        with Bus(N, ring_cap=R, batch_cap=B, device=0, sparse_records=sparse) as a, \
                Bus(N + spare, ring_cap=R, batch_cap=B, device=0, sparse_records=sparse) as b:
            for bus in (a, b):
                bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
                bus.sync()
            order = rng.permutation(N).astype(np.uint32)
            at = 0
            for k in SIZES:
                ids = np.sort(order[at:at + k]); at += k
                m = np.full(k, nat.MASK_ALL, dtype=np.uint32)
                rows[k]["reuse"].append(_ms(lambda: (a.unsubscribe_many(ids), a.release_many(ids), a.subscribe_list(m))))
                rows[k]["fresh"].append(_ms(lambda: (b.unsubscribe_many(ids), b.subscribe_many(m))))
    return rows


def fanout_us(N, rounds, reuse, reps=200):
    cap = N if reuse else 2 * N
    out = []
    with Bus(cap, ring_cap=R, batch_cap=B, device=0) as bus:
        m = np.full(N, nat.MASK_ALL, dtype=np.uint32)
        bus.subscribe_many(m)
        ids = np.arange(N, dtype=np.uint32)
        bus.unsubscribe_many(ids)
        if reuse:
            bus.release_many(ids)
            assert (bus.subscribe_list(m) == ids).all()
        else:
            bus.subscribe_many(m)
        ev = np.zeros(1, dtype=EVENT_DTYPE)
        ev["code"] = 3
        for _ in range(20):
            bus.publish_many(ev); bus.flush()
        bus.sync()
        for _ in range(rounds):
            t0 = time.perf_counter()
            for _ in range(reps):
                bus.publish_many(ev); bus.flush()
            bus.sync()
            out.append((time.perf_counter() - t0) * 1e6 / reps)
    return out


def _row(v):
    v = sorted(v)
    return {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subs", type=int, default=1 << 20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": _card(), "subs": a.subs}
    for sparse in (False, True):
        key = "sparse" if sparse else "dense"
        rows = churn(a.subs, a.rounds, sparse)
        res[key] = {str(k): {w: _row(v) for w, v in r.items()} for k, r in rows.items()}
        for k, r in rows.items():
            print(f"{key:6s} churn of {k:>6d} ids: reuse {_row(r['reuse'])['median']:8.2f} ms   "
                  f"fresh {_row(r['fresh'])['median']:8.2f} ms   (host ms, median of {a.rounds})")
    for reuse in (True, False):
        v = fanout_us(a.subs, a.rounds, reuse)
        res["fanout_reuse" if reuse else "fanout_no_reuse"] = _row(v)
        print(f"full fan-out after one churn, {'reuse (n_next = N) ' if reuse else 'no reuse (n_next = 2N)'}: "
              f"{_row(v)['median']:8.2f} us per publish + flush (host clock around {200} synchronised-at-end steps)")
    print(res["card"])
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
