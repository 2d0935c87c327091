"""Worker of tests/test_gpu_multi_follow.py, launched as
`python -m torch.distributed.run --nproc-per-node G tests/multi_worker_follow.py ...`: one process per GPU, each owning a
contiguous shard of the subscribers.  Rank 0 holds the event source: it puts every batch into the stream and fans out its
own shard with the shapes it knows.  Ranks >= 1 learn only the number of batches, once, and then follow the stream
(ShardedBus.follow: the fan-out kernels take each batch's shape from its slot header); they never see an event.  Writes
every subscriber's (count, digest) and the global digest fold to <out>/rank<r>.npz."""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def make_case(n_subs: int, n_batches: int, batch: int, seed: int = 0xF0110E55):
    """random masks, ragged and empty batches, one periodic timer per subscriber"""
    rng = np.random.default_rng(seed)
    masks = np.where(rng.random(n_subs) < 0.5, 0x1FFFF, rng.integers(0, 1 << 17, n_subs)).astype(np.uint32)
    sizes = [0 if j % 9 == 4 else (int(rng.integers(1, batch + 1)) if j % 3 == 1 else batch) for j in range(n_batches)]
    codes = [rng.integers(1, 17, n).astype(np.uint32) for n in sizes]
    srcs = [rng.integers(0, 64, n).astype(np.uint32) for n in sizes]
    return {"masks": masks, "codes": codes, "sources": srcs, "now": [(j + 1) * 20_000 for j in range(n_batches)],
            "period": 70_000, "timer_src0": 5000}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--subs", type=int, default=512)
    ap.add_argument("--batches", type=int, default=40)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--ahead", type=int, default=4)
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
    case = make_case(args.subs, args.batches, args.batch)    # the masks and timers every rank configures; events: rank 0 only
    sb = ShardedBus(args.subs, dist=dist, rank=rank, world=world, device=local, batch_cap=args.batch, timers_per_sub=1,
                    digest=True, stream_slots=8)
    try:
        assert sb.stream_ok, "stream handshake failed"
        sb.subscribe_many(case["masks"][sb.first:sb.first + sb.count])
        sb.timer_add_many(case["period"], source_id0=case["timer_src0"])
        box = [args.batches if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)                  # all a follower is ever told
        n_batches = int(box[0])
        sb.barrier()
        if rank == 0:
            for j in range(n_batches):
                ev = np.zeros(len(case["codes"][j]), dtype=EVENT_DTYPE)
                ev["code"], ev["source_id"] = case["codes"][j], case["sources"][j]
                while (rc := sb.put(ev, case["now"][j])) == nat.EAGAIN:   # a follower is a whole ring behind: it catches up
                    pass
                nat.check(rc, "cpbus_stream_put")
                nat.check(sb.fanout(len(ev), case["now"][j]), "cpbus_stream_fanout")
        else:
            j = 0
            while j < n_batches:
                k = min(args.ahead, n_batches - j)
                sb.follow(k)
                j += k
                assert sb.bus.stream_status(sb._st) == nat.OK      # resolves the k launches
        sb.bus.sync()
        assert sb.bus.stream_status(sb._st) == nat.OK
        dg = sb.digests()
        st = sb.bus.stats()
        assert st["now_ns"] == case["now"][n_batches - 1], st["now_ns"]
        fold = sb.digest_fold_all()
        np.savez(os.path.join(args.out, f"rank{rank}.npz"), first=sb.first, count=dg["count"], digest=dg["digest"],
                 deliveries=st["deliveries"], publishes=st["publishes"], fold=np.array(fold, dtype=np.uint64))
        sb.barrier()
    finally:
        sb.close()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
