"""Deliveries/s of device-resident batches on a group (`cpbus_group_publish_device`) against one bus with the same config.

Shapes: BASELINE config 2 (65,536 subscribers, all-ones masks) and config 3 (1,048,576 subscribers, a 1 kHz timer each),
512-event batches already in HBM, 10 us of virtual time per record, ring_cap 1024.  Rows: one bus; groups of 1, 2 and 4
shards on one GPU; groups over 2, 4 and 8 GPUs where the box has them (the batches on GPU 0).  The one bus and the groups
of a shape alternate within this run (`--rounds` times), each with its own warm-up; a timed window ends in a synchronise.
Only one bus or group is alive at a time (config 3 takes 32 GiB of mailboxes).  A row the run cannot produce is printed as
"not measured"; every row names the card and its power limit, read in this run.
Usage: python scripts/diag_group_device.py [--steps 200] [--warmup 20] [--rounds 2] [--out FILE]
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
from containerpilot_b200.group import GroupBus  # noqa: E402

BATCH, RING, DT_NS, TICK_NS = 512, 1024, 10_000, 1_000_000
SHAPES = {"config2": dict(subs=65_536, timers=0), "config3": dict(subs=1_048_576, timers=1)}


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown card"
    except Exception:
        return "unknown card"


def _batches(n_steps):
    """n_steps device batches of BATCH broadcast records, codes 1..16, one record every DT_NS, on GPU 0"""
    import torch
    ev = np.zeros(n_steps * BATCH, dtype=EVENT_DTYPE)
    ev["seq"] = np.arange(ev.size)
    ev["ts_ns"] = (np.arange(ev.size) + 1) * DT_NS
    ev["code"] = 1 + np.arange(ev.size) % 16
    ev["target"] = nat.TARGET_ALL
    t = torch.from_numpy(ev.view(np.uint8).reshape(-1, 32).copy()).cuda(0)
    torch.cuda.synchronize(0)
    return t


def _time(bus, shape, d, steps, warmup):
    n = shape["subs"]
    bus.subscribe_many(np.full(n, nat.MASK_ALL, dtype=np.uint32))
    if shape["timers"]:
        bus.timer_add_many(0, n, TICK_NS, source_id0=1)
    base = d.data_ptr()
    for i in range(warmup + steps):
        if i == warmup:
            bus.sync()
            d0 = bus.stats()["deliveries"]
            t0 = time.perf_counter()
        nat.check(bus.publish_device(base + i * BATCH * 32, BATCH, (i + 1) * BATCH * DT_NS), "publish_device")
    bus.sync()
    dt = time.perf_counter() - t0
    st = bus.stats()
    return (st["deliveries"] - d0) / dt, dt / steps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    n_gpus = torch.cuda.device_count() if torch.cuda.is_available() else 0
    card = _card()
    configs = [("one bus", None), ("group, 1 shard, 1 GPU", [0]), ("group, 2 shards, 1 GPU", [0, 0]),
               ("group, 4 shards, 1 GPU", [0, 0, 0, 0])]
    configs += [(f"group, {g} shards on {g} GPUs", list(range(g))) for g in (2, 4, 8)]
    d = _batches(a.warmup + a.steps) if n_gpus else None
    rows = []
    for shape_name, shape in SHAPES.items():
        runs = {name: [] for name, _ in configs}
        for _ in range(a.rounds):
            for name, devices in configs:
                if n_gpus == 0 or (devices and max(devices) >= n_gpus):
                    continue
                kw = dict(ring_cap=RING, batch_cap=BATCH, timers_per_sub=shape["timers"], digest=True)
                bus = Bus(shape["subs"], device=0, **kw) if devices is None else GroupBus(shape["subs"], devices, **kw)
                try:
                    runs[name].append(_time(bus, shape, d, a.steps, a.warmup))
                finally:
                    bus.close()
        for name, _ in configs:
            row = {"shape": shape_name, "config": name, "card": card, "batch": BATCH, "ring_cap": RING}
            if runs[name]:
                row["deliveries_per_s"] = [float(f"{r[0]:.4g}") for r in runs[name]]
                row["ms_per_batch"] = [round(r[1], 4) for r in runs[name]]
            else:
                row["deliveries_per_s"] = "not measured"
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
