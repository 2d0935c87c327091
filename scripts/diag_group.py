"""µs per publish + flush on a group of shards against one bus: 65,536 subscribers, 512-event batches.

Rows: one bus; a group of 1 and 2 shards on one GPU; groups over 2, 4 and 8 GPUs where the box has them; and each of these
in lossless mode with `consume_all` between flushes.  A row the run cannot produce is printed as "not measured".  Every
row names the card and its power limit.  Usage: python scripts/diag_group.py [--steps 200] [--warmup 20] [--out FILE]
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

N_SUBS, BATCH = 65536, 512


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown card"
    except Exception:
        return "unknown card"


def _time(bus, steps, warmup, lossless):
    bus.subscribe_many(np.full(N_SUBS, nat.MASK_ALL, dtype=np.uint32))
    ev = np.zeros(BATCH, dtype=EVENT_DTYPE)
    ev["code"] = 1 + np.arange(BATCH) % 16
    for i in range(warmup + steps):
        if i == warmup:
            bus.sync()
            t0 = time.perf_counter()
        nat.check(bus.publish_many(ev), "publish")
        nat.check(bus.flush(), "flush")
        if lossless:
            bus.consume_all()
    bus.sync()
    return (time.perf_counter() - t0) / steps * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    n_gpus = torch.cuda.device_count() if torch.cuda.is_available() else 0
    card = _card()
    kw = dict(ring_cap=1024, batch_cap=BATCH, digest=True)
    rows = []
    for lossless in (False, True):
        configs = [("one bus", None), ("group, 1 shard, 1 GPU", [0]), ("group, 2 shards, 1 GPU", [0, 0])]
        configs += [(f"group, {g} shards on {g} GPUs", list(range(g))) for g in (2, 4, 8)]
        for name, devices in configs:
            row = {"config": name, "mode": "lossless + consume_all" if lossless else "throughput", "card": card}
            if n_gpus == 0 or (devices and max(devices) >= n_gpus):
                row["us_per_publish_flush"] = "not measured"
            else:
                bus = Bus(N_SUBS, device=0, lossless=lossless, **kw) if devices is None else \
                    GroupBus(N_SUBS, devices, lossless=lossless, **kw)
                try:
                    row["us_per_publish_flush"] = round(_time(bus, a.steps, a.warmup, lossless), 1)
                finally:
                    bus.close()
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
