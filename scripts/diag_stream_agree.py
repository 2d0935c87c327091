"""Cost of agreeing on the admitted prefix through the publisher's memory (cpbus_stream_offer / _agree, what
ShardedBus(lossless=True) runs per batch across processes): µs per 512-event batch of LocalShardedBus over this box's GPUs,
65,536 subscribers per shard, consumers that keep up (consume_all every step).  Three drivers in one run, alternating:
throughput mode, lossless with the host minimum, lossless with the device agreement.  The consumers keep up, so admission
stays on its fast path; what the device agreement adds is one offer kernel, one agree kernel and one host event wait per
shard and batch.  usage: diag_stream_agree.py [out.json]"""
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
MODES = {"throughput": dict(lossless=False), "lossless-host": dict(lossless=True),
         "lossless-device": dict(lossless=True, agree="device")}


def run(mode, G, batches):
    sb = LocalShardedBus(SUBS_PER_SHARD * G, list(range(G)), ring_cap=1024, batch_cap=B, stream_slots=64, **MODES[mode])
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
        dg = sb.digests()
        return us, sum(s["admit_passes"] for s in st), int(dg["count"].sum()), int(dg["digest"].sum(dtype=np.uint64))
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
    results = {}
    for rep in range(REPS):
        order = list(MODES) if rep % 2 == 0 else list(reversed(MODES))
        for mode in order:
            us, passes, count, digest = run(mode, G, batches)
            results.setdefault(mode, set()).add((count, digest))
            res["runs"].append({"mode": mode, "us_per_batch": round(us, 2), "admit_passes": passes})
            print(f"rep {rep} {mode:16s}: {us:8.2f} us per batch (admit passes {passes})", flush=True)
    assert len(set().union(*results.values())) == 1, "the three drivers delivered different records"
    for mode in MODES:
        res[f"median_{mode}"] = float(np.median([r["us_per_batch"] for r in res["runs"] if r["mode"] == mode]))
    res["agree_cost_us"] = round(res["median_lossless-device"] - res["median_lossless-host"], 2)
    print(json.dumps(res))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
