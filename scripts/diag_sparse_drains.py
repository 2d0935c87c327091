"""Host µs and kernel launches per operation on a bus with sparse drains (CPBUS_CFG_SPARSE_DRAINS) and on a twin with
CPBUS_CFG_SPARSE_TICKS | CPBUS_CFG_SPARSE_RECORDS only, alternated in blocks in one run.  Lossless mode, 1,024-record rings,
512-event batches.

Shapes:
  pump      the Go shim's 1 ms pump step: cpbus_advance by 1 ms + cpbus_flush + cpbus_take_ready over every mailbox +
            cpbus_ack_many of what it took.  One periodic timer per mailbox (timers=all: 1,024 distinct periods over 1-10 s,
            ~N/5,500 due per step) or on one mailbox in 1,024 (timers=1/1024: most steps have nothing due).  pub512: a
            512-event publish every 100 steps whose code 1/1,024 of the fleet takes (past the record cap: a full fan-out)
  publish   the shim's Publish on a Job-shaped fleet (masks.JobSwitch.cases(), the diag_sparse_records.py shape):
            publish(1) + flush + take_ready + ack_many
  sweep     cpbus_drain_ready alone (timed from a synchronised bus) after unicast sends to k distinct mailboxes, k = 1 ..
            N/16 (sparse launches of up to 512 mailboxes each), and after a full fan-out to k mailboxes: candidates in the
            range against the dense scan, to place the list cap
Medians over the timed operations of each bus and the spread of the per-round medians; every row names the card and its
power limit.  A run without a GPU stops.
Usage: python scripts/diag_sparse_drains.py [--pump 1048576,32768] [--jobs 32768,1048576] [--sweep 1048576] [--out FILE]
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
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
from containerpilot_b200 import _native as nat  # noqa: E402
from containerpilot_b200.bus import Bus, EVENT_DTYPE, READY_DTYPE  # noqa: E402
from diag_sparse_records import _job_fleet  # noqa: E402

R, B, MS = 1024, 512, 1_000_000


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else "unknown card"


def _bus(N, flagged, lossless=True, K=1):
    return Bus(N, ring_cap=R, batch_cap=B, timers_per_sub=K, lossless=lossless, digest=True, device=0, sparse_records=True,
               sparse_drains=flagged)


class Pump:
    """one bus and its consumer: take_ready over [0, N) into buffers allocated once (as the Go shim keeps them), and ack
    what it took"""

    def __init__(self, bus, N, cap, ready_cap=65536):
        self.bus, self.N, self.cap, self.now = bus, N, cap, 0
        self.out = np.zeros(cap, dtype=EVENT_DTYPE)
        self.ready_cap = min(N, ready_cap)
        self.ready = np.zeros(self.ready_cap, dtype=READY_DTYPE)
        self.nr, self.tot, self.next = C.c_size_t(), C.c_size_t(), C.c_uint32()
        self.start = 0

    def drain(self):
        b = self.bus
        nat.check(b._lib.cpbus_take_ready(b._h, 0, self.N, self.start, self.out.ctypes.data, self.cap, self.ready.ctypes.data,
                                          self.ready_cap, C.byref(self.nr), C.byref(self.tot), C.byref(self.next)),
                  "cpbus_take_ready")
        self.start = self.next.value
        ready = self.ready[: self.nr.value]
        if len(ready):
            st = self.bus.ack_many(ready["sub_id"], ready["count"])
            assert (st == nat.OK).all()
        return len(ready)

    def step(self, events=None):
        self.now += MS
        nat.check(self.bus.advance(self.now), "advance")
        if events is not None:
            nat.check(self.bus.publish_many(events), "publish")
        nat.check(self.bus.flush(), "flush")
        self.drain()


def _time(pumps, steps, rounds, make_events):
    """per pump: (median µs per step, spread of the per-round medians in µs, kernels per step); blocks alternate"""
    t = {k: [] for k in pumps}
    k0 = {k: p.bus.stats()["kernel_launches"] for k, p in pumps.items()}
    n = {k: 0 for k in pumps}
    for rnd in range(rounds + 1):                       # round 0 warms every path up
        for k, p in pumps.items():
            times = []
            if rnd == 1:
                k0[k] = p.bus.stats()["kernel_launches"]
            for i in range(steps):
                e = make_events(n[k])
                n[k] += 1
                t0 = time.perf_counter()
                p.step(e)
                times.append(time.perf_counter() - t0)
            if rnd:
                t[k].append(times)
    res = {}
    for k, p in pumps.items():
        med = [float(np.median(v)) * 1e6 for v in t[k]]
        res[k] = (float(np.median(np.concatenate(t[k]))) * 1e6, max(med) - min(med),
                  (p.bus.stats()["kernel_launches"] - k0[k]) / (rounds * steps))
    return res


def _row(res):
    f, w = res["flagged"], res["twin"]
    return {"us_flagged": round(f[0], 1), "us_twin": round(w[0], 1), "spread_us_flagged": round(f[1], 1),
            "spread_us_twin": round(w[1], 1), "kernels_flagged": round(f[2], 3), "kernels_twin": round(w[2], 3)}


def _pump_fleet(N, flagged, timers):
    bus = _bus(N, flagged)
    masks = np.full(N, 1 << 2, dtype=np.uint32)          # code 2 is never published
    masks[::1024] = 1 << 1                               # code 1: one mailbox in 1,024
    bus.subscribe_many(masks)
    chunk = max(1, N // 1024)
    if timers == "all":
        for c in range(1024):
            bus.timer_add_many(c * chunk, chunk, MS * 1000 + c * (9000 * MS // 1023), source_id0=c * chunk)
    else:
        ids = np.arange(0, N, 1024, dtype=np.uint32)
        bus.timer_add_list(ids, MS * 1000 + (np.arange(len(ids)) % 1024) * (9000 * MS // 1023), ids)
    p = Pump(bus, N, max(R, 2 * B * (N // 1024 + 1)))
    p.now = 10_000 * MS                                  # past the longest period: the phases are spread
    nat.check(bus.advance(p.now), "advance"); nat.check(bus.flush(), "flush")
    while p.drain():
        pass
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pump", default="1048576,32768")
    ap.add_argument("--jobs", default="32768,1048576")
    ap.add_argument("--sweep", type=int, default=1048576)
    ap.add_argument("--steps", type=int, default=300)
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
    for N in [int(x) for x in a.pump.split(",") if x]:
        for timers in ("all", "1/1024"):
            pumps = {"flagged": _pump_fleet(N, True, timers), "twin": _pump_fleet(N, False, timers)}
            batch = np.zeros(B, dtype=EVENT_DTYPE)
            batch["code"] = 1
            for pub in (False, True) if timers == "all" else (False,):
                res = _time(pumps, a.steps, a.rounds, lambda i: batch if pub and i % 100 == 99 else None)
                emit({"shape": "pump", "subscribers": N, "timers": timers, "pub512_every": 100 if pub else 0, **_row(res)})
            for p in pumps.values():
                p.bus.close()

    for N in [int(x) for x in a.jobs.split(",") if x]:
        ms, cases = _job_fleet(N)
        pumps = {}
        for k, flagged in (("flagged", True), ("twin", False)):
            bus = _bus(N, flagged, K=0)
            bus.subscribe_pairs_many(ms, cases)
            pumps[k] = Pump(bus, N, 1 << 16)
        evs = []
        for _ in range(64):
            e = np.zeros(1, dtype=EVENT_DTYPE)
            e["code"], e["source_id"] = rng.integers(1, 17), rng.integers(0, 5 + 5 * N)
            evs.append(e)
        res = _time(pumps, a.steps, a.rounds, lambda i: evs[i % len(evs)])
        emit({"shape": "publish", "subscribers": N, "events": 1, **_row(res)})
        for p in pumps.values():
            p.bus.close()

    N = a.sweep
    buses = {"flagged": _bus(N, True, lossless=False, K=0), "twin": _bus(N, False, lossless=False, K=0)}
    masks = np.full(N, 1 << 2, dtype=np.uint32)
    for bus in buses.values():
        bus.subscribe_many(masks)
    out = np.zeros(max(R, N // 16), dtype=EVENT_DTYPE)
    one = np.zeros(1, dtype=EVENT_DTYPE)
    one["code"], one["target"] = 3, nat.TARGET_ALL
    dev = torch.from_numpy(one.view(np.uint8).reshape(-1, 32).copy()).cuda()
    torch.cuda.synchronize()
    perm = rng.permutation(N)
    ks, k = [], 1
    while k <= N // 16:
        ks.append(k)
        k *= 4
    for fanout in (False, True):
        for k in ks:
            targets = np.sort(perm[:k]).astype(np.uint32)
            t = {name: [] for name in buses}
            launches = {name: 0 for name in buses}
            for rnd in range(a.rounds + 1):
                for name, bus in buses.items():
                    times = []
                    for _ in range(20 if k <= 4096 else 4):
                        if fanout:                   # one device record of the k targets' code: a full fan-out
                            bus.set_mask_many(targets, np.full(k, 1 << 3, dtype=np.uint32))
                            nat.check(bus.publish_device(dev.data_ptr(), 1, bus.stats()["now_ns"]), "publish_device")
                        else:
                            for s in targets:
                                nat.check(bus.send(int(s), 4, 1), "send")
                        nat.check(bus.flush(), "flush")
                        bus.sync()
                        k0 = bus.stats()["kernel_launches"]
                        t0 = time.perf_counter()
                        _, ready, _ = bus.drain_ready(0, N, 0, len(out), k, out=out)
                        times.append(time.perf_counter() - t0)
                        launches[name] = bus.stats()["kernel_launches"] - k0
                        assert len(ready) == k
                        if fanout:
                            bus.set_mask_many(targets, np.full(k, 1 << 2, dtype=np.uint32))
                    if rnd:
                        t[name].append(times)
            med = {n_: [float(np.median(v)) * 1e6 for v in t[n_]] for n_ in buses}
            emit({"shape": "sweep", "subscribers": N, "candidates": k, "after": "fan-out" if fanout else "sparse sends",
                  "drain_us_flagged": round(float(np.median(np.concatenate(t["flagged"]))) * 1e6, 1),
                  "drain_us_twin": round(float(np.median(np.concatenate(t["twin"]))) * 1e6, 1),
                  "spread_us_flagged": round(max(med["flagged"]) - min(med["flagged"]), 1),
                  "spread_us_twin": round(max(med["twin"]) - min(med["twin"]), 1),
                  "drain_kernels_flagged": launches["flagged"], "drain_kernels_twin": launches["twin"]})
    for bus in buses.values():
        bus.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
