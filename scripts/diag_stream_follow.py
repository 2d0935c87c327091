"""What a consumer that does not know the batches' shapes pays per batch: µs per 512-event batch of LocalShardedBus over
this box's GPUs (shards on one GPU when there is only one), 65,536 subscribers per shard, throughput mode.  Modes, in one
run and alternating after a warm-up:
  spmd     every shard is told (n, now_ns) and calls cpbus_stream_fanout;
  poll     every shard asks cpbus_stream_poll for the next batch's shape (a synchronous read of the slot header), then
           cpbus_stream_fanout — today's path for a consumer that is not told;
  follow-r every shard calls cpbus_stream_fanout_next, r follower launches queued before the publisher puts their batches,
           resolved every 8 batches.
Every mode must deliver the same records (sum of counts and digests); the script exits non-zero otherwise.
usage: diag_stream_follow.py [out.json]"""
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

SUBS_PER_SHARD, B, WARM, STEPS, REPS, ROUND = 65_536, 512, 48, 400, 3, 8
MODES = ["spmd", "poll", "follow-0", "follow-2", "follow-4"]


def run(mode, G, batches):
    sb = LocalShardedBus(SUBS_PER_SHARD * G, list(range(G)), ring_cap=1024, batch_cap=B, stream_slots=64)
    shards = [(bus, sb._st[g]) for g, (_, _, bus) in enumerate(sb.shards)]
    ahead = int(mode.split("-")[1]) if mode.startswith("follow") else 0
    try:
        sb.subscribe_many(np.full(SUBS_PER_SHARD * G, nat.MASK_ALL, dtype=np.uint32))

        def put(j):   # EAGAIN: the ring is full of batches the queued launches have not pulled yet
            while (rc := sb.put(batches[j % len(batches)], (j + 1) * 10_000)) == nat.EAGAIN:
                pass
            nat.check(rc, "cpbus_stream_put")

        def follow():
            for bus, st in shards:
                nat.check(bus.stream_fanout_next(st), "cpbus_stream_fanout_next")

        def go(lo, hi):
            if mode.startswith("follow"):
                # Rounds of ROUND batches, resolved at the end (cpbus_stream_status), as a rank that reads its statistics
                # every ROUND batches would.  One thread puts AND follows here, so a resolve may only come once every
                # queued follower's batch has been put (at most 8 are outstanding: the 9th call would resolve first).
                for r0 in range(lo, hi, ROUND):
                    r1 = min(hi, r0 + ROUND)
                    for _ in range(r0, min(r1, r0 + ahead)):
                        follow()
                    for j in range(r0, r1):
                        put(j)
                        if j + ahead < r1:
                            follow()
                    for bus, st in shards:
                        nat.check(bus.stream_status(st), "cpbus_stream_status")
                return
            for j in range(lo, hi):
                put(j)
                for bus, st in shards:
                    if mode == "spmd":
                        shape = (len(batches[j % len(batches)]), (j + 1) * 10_000)
                    else:
                        while (shape := bus.stream_poll(st)) is None:
                            pass
                    nat.check(bus.stream_fanout(st, *shape), "cpbus_stream_fanout")
        go(0, WARM); sb.sync()
        t0 = time.perf_counter()
        go(WARM, WARM + STEPS); sb.sync()
        us = (time.perf_counter() - t0) / STEPS * 1e6
        dg = sb.digests()
        return us, int(dg["count"].sum()), int(dg["digest"].sum(dtype=np.uint64))
    finally:
        sb.close()


def main():
    G = torch.cuda.device_count()
    rng = np.random.default_rng(5)
    batches = []
    for i in range(16):
        n = B if i % 4 else int(rng.integers(1, B))       # some ragged batches: the followers must learn each shape
        ev = np.zeros(n, dtype=EVENT_DTYPE)
        ev["code"] = rng.integers(1, 17, n); ev["source_id"] = rng.integers(0, 4096, n)
        batches.append(ev)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"gpus": G, "gpu": gpu, "subs_per_shard": SUBS_PER_SHARD, "batch": B, "steps": STEPS, "runs": []}
    results = set()
    for rep in range(REPS):
        for mode in (MODES if rep % 2 == 0 else list(reversed(MODES))):
            us, count, digest = run(mode, G, batches)
            results.add((count, digest))
            res["runs"].append({"mode": mode, "us_per_batch": round(us, 2)})
            print(f"rep {rep} {mode:9s}: {us:8.2f} us per batch", flush=True)
    for mode in MODES:
        res[f"median_{mode}"] = float(np.median([r["us_per_batch"] for r in res["runs"] if r["mode"] == mode]))
    res["digests_identical"] = len(results) == 1
    print(json.dumps(res))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)
    if len(results) != 1:
        sys.exit("the modes delivered different records")


if __name__ == "__main__":
    main()
