"""Cost of a lossless follower round (cpbus_stream_round_next: admit, offer, agree and the fan-out of the agreed prefix
enqueued on the device, never waited for on the host) against the host-driven lossless round and throughput followers:
µs per 512-event batch of LocalShardedBus over this box's GPUs, 65,536 subscribers per shard, consumers that keep up
(consume_all every step), 400 timed steps after 50 warm-up steps, three alternations with the order reversed every other
time.  Drivers:
  throughput-follow : throughput mode, cpbus_stream_fanout_next per batch
  lossless-device   : one host-driven round per batch (admit, offer, agree with its host wait, fanout_prefix)
  lossless-rounds   : cpbus_stream_round_next per batch, resolved every 4 batches (cpbus_stream_progress)
All three must deliver the same records.  usage: diag_stream_lossless_rounds.py [out.json]"""
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

SUBS_PER_SHARD, B, WARM, STEPS, REPS, DEPTH = 65_536, 512, 50, 400, 3, 4
MODES = {"throughput-follow": dict(lossless=False), "lossless-device": dict(lossless=True, agree="device"),
         "lossless-rounds": dict(lossless=True, agree="device")}


def run(mode, G, batches):
    sb = LocalShardedBus(SUBS_PER_SHARD * G, list(range(G)), ring_cap=1024, batch_cap=B, stream_slots=64, **MODES[mode])
    try:
        sb.subscribe_many(np.full(SUBS_PER_SHARD * G, nat.MASK_ALL, dtype=np.uint32))

        def go(lo, hi):
            for j0 in range(lo, hi, DEPTH):
                js = range(j0, min(hi, j0 + DEPTH))
                for j in js:                                   # the publisher runs ahead by DEPTH batches
                    nat.check(sb.put(batches[j % len(batches)], (j + 1) * 10_000), "put")
                for j in js:
                    if mode == "lossless-device":
                        assert sb.fanout(B, (j + 1) * 10_000) == nat.OK
                    elif mode == "throughput-follow":
                        for g in range(G):
                            sb.follow(g, 1)
                    else:
                        for g in range(G):
                            sb.follow_rounds(g, 1)
                    sb.consume_all()
                if mode == "lossless-rounds":
                    assert sb.progress() == (js[-1] + 1, 0, 0)
                else:
                    for g, (_, _, bus) in enumerate(sb.shards):
                        assert bus.stream_status(sb._st[g]) == nat.OK
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
    res = {"gpus": G, "gpu": gpu, "subs_per_shard": SUBS_PER_SHARD, "batch": B, "steps": STEPS, "depth": DEPTH, "runs": []}
    results = {}
    for rep in range(REPS):
        order = list(MODES) if rep % 2 == 0 else list(reversed(MODES))
        for mode in order:
            us, passes, count, digest = run(mode, G, batches)
            results.setdefault(mode, set()).add((count, digest))
            res["runs"].append({"mode": mode, "us_per_batch": round(us, 2), "admit_passes": passes})
            print(f"rep {rep} {mode:18s}: {us:8.2f} us per batch (admit passes {passes})", flush=True)
    assert len(set().union(*results.values())) == 1, "the three drivers delivered different records"
    for mode in MODES:
        res[f"median_{mode}"] = float(np.median([r["us_per_batch"] for r in res["runs"] if r["mode"] == mode]))
    print(json.dumps(res))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
