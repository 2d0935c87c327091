"""What dropping missed ticks (CPBUS_CFG_DROP_MISSED_TICKS) costs and saves, on a bus flagged with it and an unflagged twin,
alternated in one run.

Fleet: N subscribers (default 1,048,576), one 1 s heartbeat each (K = 1), 1,024-record rings, 256-event batches.
  jump      host µs and kernel launches of one `advance` by 1,000 s + `flush` + sync, dense and sparse (CPBUS_CFG_SPARSE_TICKS)
            buses, throughput and lossless mode; each bus drains everything (consume_all) between its jumps
  pump      host µs per 1 ms pump step (`advance` + `flush`, a sync every step) in steady state: no step crosses a period
  kernel    the catch-up kernel's duration (torch.profiler, CUDA activities) on the dense throughput bus
Medians over the rounds; the card and its power limit head the output.  A run without a GPU stops.
Usage: python scripts/diag_drop_missed_ticks.py [--subs 1048576] [--rounds 5] [--pump-steps 2000] [--out FILE]
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

R, B, MS, SEC = 1024, 256, 1_000_000, 1_000_000_000


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else "unknown card"


def _fleet(N, flagged, sparse, lossless):
    bus = Bus(N, ring_cap=R, batch_cap=B, timers_per_sub=1, lossless=lossless, digest=True, device=0, sparse_ticks=sparse,
              drop_missed_ticks=flagged)
    bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
    bus.timer_add_many(0, N, SEC, source_id0=0)
    bus.sync()
    return bus


def _jump(bus, st):
    bus.consume_all(); bus.sync()
    k0 = bus.stats()["kernel_launches"]
    t0 = time.perf_counter()
    st["now"] += 1000 * SEC
    nat.check(bus.advance(st["now"]), "advance")
    nat.check(bus.flush(), "flush")
    bus.sync()
    return (time.perf_counter() - t0) * 1e6, bus.stats()["kernel_launches"] - k0


def _pump(bus, st, n):
    bus.consume_all(); bus.sync()
    t0 = time.perf_counter()
    for _ in range(n):
        st["now"] += MS
        nat.check(bus.advance(st["now"]), "advance")
        nat.check(bus.flush(), "flush")
        bus.sync()
    return (time.perf_counter() - t0) * 1e6 / n


def _kernel_us(bus, st):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _jump(bus, st)
        torch.cuda.synchronize()
    ds = [e.device_time for e in prof.events() if "timer_catchup_kernel" in e.name]
    return ds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subs", type=int, default=1 << 20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--pump-steps", type=int, default=2000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    lines = [f"# {_card()}  N={a.subs}  1 s heartbeat, K=1, R={R}"]
    res = {}
    for lossless in (False, True):
        for sparse in (False, True):
            buses = {f: _fleet(a.subs, f, sparse, lossless) for f in (True, False)}
            st = {f: {"now": 0} for f in buses}
            jump = {f: [] for f in buses}
            pump = {f: [] for f in buses}
            for f in buses:                                   # warm-up: one jump and a few pump steps each
                _jump(buses[f], st[f]); _pump(buses[f], st[f], 20)
            for _ in range(a.rounds):
                for f in (True, False):
                    jump[f].append(_jump(buses[f], st[f]))
                    pump[f].append(_pump(buses[f], st[f], a.pump_steps))
            mode = ("lossless" if lossless else "throughput") + ("/sparse" if sparse else "/dense")
            for f in (True, False):
                us = [j[0] for j in jump[f]]
                row = {"jump_us_median": float(np.median(us)), "jump_us_min": float(min(us)), "jump_us_max": float(max(us)),
                       "jump_launches": int(jump[f][-1][1]), "pump_us_median": float(np.median(pump[f])),
                       "pump_us_min": float(min(pump[f])), "pump_us_max": float(max(pump[f]))}
                res[f"{mode}/{'flagged' if f else 'unflagged'}"] = row
                lines.append(f"{mode:20s} {'flagged' if f else 'unflagged':9s} jump {row['jump_us_median']:10.1f} us "
                             f"[{row['jump_us_min']:.1f}-{row['jump_us_max']:.1f}] launches {row['jump_launches']:3d}   "
                             f"pump {row['pump_us_median']:7.2f} us/step [{row['pump_us_min']:.2f}-{row['pump_us_max']:.2f}]")
            if not lossless and not sparse:
                ds = _kernel_us(buses[True], st[True])
                res["catchup_kernel_us"] = ds
                lines.append(f"catch-up kernel (dense, {a.subs} slots): {', '.join(f'{d:.1f}' for d in ds)} us")
            for b in buses.values():
                b.close()
    try:
        lib = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "containerpilot_b200", "libcpbus.so")
        ru = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True, timeout=60).stdout.splitlines()
        for i, l in enumerate(ru):
            if "timer_catchup_kernel" in l and i + 1 < len(ru):
                lines.append("catch-up kernel resources: " + ru[i + 1].strip())
    except (OSError, subprocess.SubprocessError):
        lines.append("catch-up kernel resources: cuobjdump not available")
    print("\n".join(lines))
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": lines[0], "rows": res}, f, indent=1)


if __name__ == "__main__":
    main()
