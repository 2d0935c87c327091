"""Worker of tests/test_gpu_multi_stream_blockers.py, launched as
`python -m torch.distributed.run --nproc-per-node G tests/multi_worker_stream_blockers.py ...`: one process per GPU, each
owning a contiguous shard of the subscribers, every bus lossless, nobody consuming.  Rank 0 puts every batch into the
stream; every rank then queues one device round at a time (ShardedBus.follow_rounds) until a round stalls, and asks the
fleet-wide blockers() and lagging(); then drains exactly the blockers it owns and goes on, STALLS times.  Writes every
answer to <out>/rank<r>.npz.  `replay_on_one_process` drives a LocalShardedBus through the same steps."""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

STALLS = 4
LAG_ARGS = [(0, None, 1, None), (None, 7, 0, 5), (3, 40, 2, 3)]   # (first_sub, start offset, min_backlog, cap)


def make_case(n_subs: int, n_batches: int, batch: int, seed: int = 0xB10C):
    """random masks, some taking everything; full and ragged batches"""
    rng = np.random.default_rng(seed)
    masks = np.where(rng.random(n_subs) < 0.3, 0x1FFFF, rng.integers(0, 1 << 17, n_subs)).astype(np.uint32)
    sizes = [int(rng.integers(1, batch + 1)) if j % 3 == 1 else batch for j in range(n_batches)]
    codes = [rng.integers(1, 17, n).astype(np.uint32) for n in sizes]
    srcs = [rng.integers(0, 64, n).astype(np.uint32) for n in sizes]
    return {"masks": masks, "codes": codes, "sources": srcs, "now": [(j + 1) * 20_000 for j in range(n_batches)]}


def events(case, j):
    from containerpilot_b200.bus import EVENT_DTYPE
    ev = np.zeros(len(case["codes"][j]), dtype=EVENT_DTYPE)
    ev["code"], ev["source_id"] = case["codes"][j], case["sources"][j]
    return ev


def ask(sb, n_subs):
    """the fleet's answers at a stall: blockers, and lagging for each LAG_ARGS entry (entries as bytes, next_sub, summary)"""
    out = {"blockers": sb.blockers().tolist(), "lagging": []}
    for first, start, mb, cap in LAG_ARGS:
        first = 0 if first is None else first
        n = n_subs - first
        ent, nxt, summ = sb.lagging(first, n, start_sub=first + (start or 0) % n, min_backlog=mb, cap=cap)
        out["lagging"].append((ent.tobytes(), nxt, [summ[k] for k in ("active", "lagging", "backlog_total", "backlog_max",
                                                                     "lost_total")] + list(summ["hist"])))
    return out


def run_to_stalls(sb, queue_round, drain_own, n_batches, n_subs):
    """queue one round at a time until it stalls; at each stall ask, then drain exactly the blockers"""
    answers, stalled = [], 0
    while len(answers) < STALLS:
        done, off, st = sb.progress()
        if done == n_batches:
            break
        queue_round()
        done, off, st = sb.progress()
        if st > stalled:
            stalled = st
            a = ask(sb, n_subs)
            a["position"] = [done, off]
            answers.append(a)
            assert a["blockers"], "a stalled round with no blockers"
            for s in a["blockers"]:
                drain_own(s)
    return answers


def replay_on_one_process(G, n_subs, n_batches, batch, ring):
    from containerpilot_b200.sharding import LocalShardedBus
    case = make_case(n_subs, n_batches, batch)
    sb = LocalShardedBus(n_subs, [0] * G, ring_cap=ring, batch_cap=batch, stream_slots=n_batches, lossless=True)
    try:
        sb.subscribe_many(case["masks"])
        for j in range(n_batches):
            assert sb.put(events(case, j), case["now"][j]) == 0
        return run_to_stalls(sb, lambda: [sb.follow_rounds(g, 1) for g in range(G)], lambda s: sb.drain(s), n_batches, n_subs)
    finally:
        sb.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--subs", type=int, default=64)
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--ring", type=int, default=64)
    args = ap.parse_args()

    import torch
    import torch.distributed as dist
    from containerpilot_b200 import _native as nat
    from containerpilot_b200.sharding import ShardedBus

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    case = make_case(args.subs, args.batches, args.batch)
    sb = ShardedBus(args.subs, dist=dist, rank=rank, world=world, device=local, ring_cap=args.ring, batch_cap=args.batch,
                    digest=True, stream_slots=args.batches, lossless=True)
    try:
        assert sb.stream_ok, "stream handshake failed"
        sb.subscribe_many(case["masks"][sb.first:sb.first + sb.count])
        if rank == 0:
            for j in range(args.batches):
                nat.check(sb.bus.stream_put(sb._st, events(case, j), case["now"][j], nowait=True), "cpbus_stream_put")
        sb.barrier()

        def drain_own(s):
            if sb.first <= s < sb.first + sb.count:
                sb.bus.drain(s)

        answers = run_to_stalls(sb, lambda: sb.follow_rounds(1), drain_own, args.batches, args.subs)
        np.save(os.path.join(args.out, f"rank{rank}.npy"), np.array(answers, dtype=object), allow_pickle=True)
        sb.barrier()
    finally:
        sb.close()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
