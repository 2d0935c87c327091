"""Lossless mode on the multi-GPU stream: µs per 512-event batch of LocalShardedBus over this box's GPUs, 65,536
subscribers per shard, consumers that keep up (consume_all every step), lossless against throughput mode in one run,
alternating.  With the mailboxes emptied every step the admission fast path proves every batch fits: no admission
kernel and no host sync, so lossless should cost about what throughput mode costs.  usage: diag_stream_lossless.py [out.json]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from containerpilot_b200 import _native as nat  # noqa: E402
from containerpilot_b200.bus import EVENT_DTYPE  # noqa: E402
from containerpilot_b200.sharding import LocalShardedBus  # noqa: E402

SUBS_PER_SHARD, B, WARM, STEPS, REPS = 65_536, 512, 50, 400, 3


def run(lossless, G, batches):
    sb = LocalShardedBus(SUBS_PER_SHARD * G, list(range(G)), ring_cap=1024, batch_cap=B, stream_slots=64, lossless=lossless)
    try:
        sb.subscribe_many(np.full(SUBS_PER_SHARD * G, nat.MASK_ALL, dtype=np.uint32))

        def go(lo, hi):
            for j in range(lo, hi):
                assert sb.publish(batches[j % len(batches)], (j + 1) * 10_000) == nat.OK
                sb.consume_all()
        go(0, WARM); sb.sync()
        t0 = time.perf_counter()
        go(WARM, WARM + STEPS); sb.sync()
        us = (time.perf_counter() - t0) / STEPS * 1e6
        st = [bus.stats() for _, _, bus in sb.shards]
        return us, sum(s["admit_passes"] for s in st), sum(s["admit_skipped"] for s in st)
    finally:
        sb.close()


def main():
    G = torch.cuda.device_count()
    rng = np.random.default_rng(5)
    batches = []
    for _ in range(16):
        ev = np.zeros(B, dtype=EVENT_DTYPE)
        ev["code"] = rng.integers(1, 17, B); ev["source_id"] = rng.integers(0, 4096, B)
        batches.append(ev)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"gpus": G, "gpu": gpu, "subs_per_shard": SUBS_PER_SHARD, "batch": B, "steps": STEPS, "runs": []}
    for rep in range(REPS):
        for lossless in (False, True):
            us, passes, skipped = run(lossless, G, batches)
            res["runs"].append({"lossless": lossless, "us_per_batch": round(us, 2), "admit_passes": passes, "admit_skipped": skipped})
            print(f"rep {rep} lossless={lossless}: {us:8.2f} us per batch (admit passes {passes}, skipped {skipped})", flush=True)
    for lossless in (False, True):
        v = [r["us_per_batch"] for r in res["runs"] if r["lossless"] == lossless]
        res["median_lossless" if lossless else "median_throughput"] = float(np.median(v))
    print(json.dumps(res))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
