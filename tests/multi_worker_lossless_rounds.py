"""Worker of tests/test_gpu_multi_lossless_rounds.py, launched as
`python -m torch.distributed.run --nproc-per-node G tests/multi_worker_lossless_rounds.py ...`: one process per GPU, each
owning a contiguous shard of the subscribers, every bus lossless.  Rank 0 holds the event source: it puts every batch into
the stream.  Ranks >= 1 learn only the number of batches, once.  Every rank then runs ShardedBus.run_rounds: admission
rounds queued on the device, the ranks agreeing through the offer words in the publisher's memory; the pump drains some
mailboxes (and, on rank 0, puts the batches the ring has room for).  Writes every subscriber's drained records and
(count, digest) to <out>/rank<r>.npz."""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def make_case(n_subs: int, n_batches: int, batch: int, seed: int = 0x1055_1E55):
    """random masks, ragged and empty batches"""
    rng = np.random.default_rng(seed)
    masks = np.where(rng.random(n_subs) < 0.5, 0x1FFFF, rng.integers(0, 1 << 17, n_subs)).astype(np.uint32)
    sizes = [0 if j % 9 == 4 else (int(rng.integers(1, batch + 1)) if j % 3 == 1 else batch) for j in range(n_batches)]
    codes = [rng.integers(1, 17, n).astype(np.uint32) for n in sizes]
    srcs = [rng.integers(0, 64, n).astype(np.uint32) for n in sizes]
    return {"masks": masks, "codes": codes, "sources": srcs, "now": [(j + 1) * 20_000 for j in range(n_batches)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--subs", type=int, default=256)
    ap.add_argument("--batches", type=int, default=30)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--ring", type=int, default=128)
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
    case = make_case(args.subs, args.batches, args.batch)    # the masks every rank configures; events: rank 0 only
    sb = ShardedBus(args.subs, dist=dist, rank=rank, world=world, device=local, ring_cap=args.ring, batch_cap=args.batch,
                    digest=True, stream_slots=8, lossless=True)
    drained = {s: [] for s in range(sb.first, sb.first + sb.count)}
    try:
        assert sb.stream_ok, "stream handshake failed"
        sb.subscribe_many(case["masks"][sb.first:sb.first + sb.count])
        box = [args.batches if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)                  # all the other ranks are ever told
        n_batches = int(box[0])
        sb.barrier()
        put = 0
        rng = np.random.default_rng(1000 + rank)

        def pump():
            nonlocal put
            while rank == 0 and put < n_batches:
                ev = np.zeros(len(case["codes"][put]), dtype=EVENT_DTYPE)
                ev["code"], ev["source_id"] = case["codes"][put], case["sources"][put]
                if sb.bus.stream_put(sb._st, ev, case["now"][put], nowait=True) != nat.OK:
                    break
                put += 1
            for s in rng.permutation(np.arange(sb.first, sb.first + sb.count))[:max(1, sb.count // 3)]:
                drained[int(s)].append(sb.bus.drain(int(s), cap=int(rng.integers(1, args.ring + 1))))

        pump()
        rounds = sb.run_rounds(n_batches, pump=pump, depth=4)
        for s in drained:
            drained[s].append(sb.bus.drain(s))
        st = sb.bus.stats()
        dg = sb.digests()
        recs = [np.concatenate(drained[s]) if drained[s] else np.zeros(0, dtype=EVENT_DTYPE) for s in drained]
        np.savez(os.path.join(args.out, f"rank{rank}.npz"), first=sb.first, count=dg["count"], digest=dg["digest"],
                 rounds=rounds, publishes=st["publishes"], partial=st["admit_partial"],
                 records=np.concatenate(recs).view(np.uint8), lens=np.array([len(x) for x in recs]))
        sb.barrier()
    finally:
        sb.close()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
