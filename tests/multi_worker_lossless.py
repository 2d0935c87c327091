"""Worker of tests/test_gpu_multi_lossless.py, launched as
`python -m torch.distributed.run --nproc-per-node G tests/multi_worker_lossless.py ...`: one process per GPU, each owning a
contiguous shard of the subscribers, in lossless mode (ShardedBus(lossless=True): the ranks agree on every admission round
through the publisher's memory).  Small rings; after every round that stalls, each rank drains its own part of a drain
schedule that depends only on the round number, so every rank retries in lockstep.  Writes every subscriber's
(count, digest), the number of rounds and the global digest fold to <out>/rank<r>.npz."""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def make_case(n_subs: int, n_batches: int, batch: int, seed: int = 0x10551E55):
    rng = np.random.default_rng(seed)
    masks = np.where(rng.random(n_subs) < 0.5, 0x1FFFF, rng.integers(0, 1 << 17, n_subs)).astype(np.uint32)
    masks[::7] = 0
    codes = rng.integers(1, 17, n_batches * batch).astype(np.uint32)
    srcs = rng.integers(0, 64, n_batches * batch).astype(np.uint32)
    return {"masks": masks, "codes": codes, "sources": srcs, "now": [(j + 1) * 1000 for j in range(n_batches)]}


def drain_schedule(round_no: int, n_subs: int, ring_cap: int):
    """(subscriber, records to take) of the consumers that run after stalled round `round_no` — the same on every rank"""
    rng = np.random.default_rng(1_000_003 * (round_no + 1))
    subs = np.nonzero(rng.random(n_subs) < 0.5)[0]
    return [(int(s), int(t)) for s, t in zip(subs, rng.integers(1, ring_cap + 1, len(subs)))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--subs", type=int, default=256)
    ap.add_argument("--batches", type=int, default=24)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--ring", type=int, default=64)
    args = ap.parse_args()

    import torch
    import torch.distributed as dist
    from containerpilot_b200 import _native as nat
    from containerpilot_b200.bus import EVENT_DTYPE
    from containerpilot_b200.sharding import ShardedBus

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    case = make_case(args.subs, args.batches, args.batch)
    sb = ShardedBus(args.subs, dist=dist, rank=rank, world=world, device=local, ring_cap=args.ring, batch_cap=args.batch,
                    digest=True, stream_slots=4, lossless=True)
    try:
        assert sb.stream_ok, "stream handshake failed"
        sb.subscribe_many(case["masks"][sb.first:sb.first + sb.count])
        B, rounds, stalls = args.batch, 0, 0
        for j in range(args.batches):
            ev = np.zeros(B, dtype=EVENT_DTYPE)
            ev["code"], ev["source_id"] = case["codes"][j * B:(j + 1) * B], case["sources"][j * B:(j + 1) * B]
            nat.check(sb.put(ev, case["now"][j]), "cpbus_stream_put")
            while True:
                rc = sb.fanout(B, case["now"][j])
                rounds += 1
                if rc == nat.OK:
                    break
                assert rc == nat.EAGAIN, rc
                stalls += 1
                for s, take in drain_schedule(rounds - 1, args.subs, args.ring):
                    if sb.first <= s < sb.first + sb.count:
                        sb.bus.drain(s, cap=take)
        sb.bus.sync()
        assert sb.bus.stream_status(sb._st) == nat.OK
        dg = sb.digests()
        st = sb.bus.stats()
        assert st["overwritten"] == 0
        fold = sb.digest_fold_all()
        np.savez(os.path.join(args.out, f"rank{rank}.npz"), first=sb.first, count=dg["count"], digest=dg["digest"],
                 rounds=rounds, stalls=stalls, deliveries=st["deliveries"], fold=np.array(fold, dtype=np.uint64))
        sb.barrier()
    finally:
        sb.close()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
