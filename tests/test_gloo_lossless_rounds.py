"""The lossless-round driver (ShardedBus.run_rounds / sharding.drive_rounds) at world_size 2 on CPU/gloo.  Each rank's GPU
bus is replaced by a stand-in: stream_round_next only queues, and stream_progress resolves the queued rounds by exchanging
each round's offer over gloo (the agree kernel's minimum), with the room each rank's mailboxes have in each round scripted
("stall": that rank's admission stalls).  Ranks >= 1 are told only the number of batches.  The driver must never queue
more rounds than batches remain, both ranks must queue the same sequence, and both must stop together at T after the
stalls.  The device rounds themselves run in tests/test_gpu_stream_rounds.py and tests/test_gpu_multi_lossless_rounds.py."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from containerpilot_b200 import _native as nat
from containerpilot_b200 import sharding

SIZES = [10, 5, 0, 7, 3]            # the batches' record counts (known to the stand-in stream, never to the driver)
ROOM = {                            # per rank, per round: records its mailboxes can take
    0: [10, "stall", 3, 10, 5, 0, 0, 2, 2, 9, 9, 9, 9, 9, 9],
    1: [4, 10, "stall", 10, 5, "stall", 0, 9, 0, 9, 9, 9, 9, 9, 9],
}


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


class _RoundBus:
    rank = 0

    def __init__(self, n, **kw):
        self.kw, self.calls = kw, []
        self.queued = self.round = 0
        self.batch, self.off, self.stalled = 0, 0, 0

    def stream_create(self, slots, n_consumers):
        return "st0", b"H" * 64

    def stream_open(self, handle, idx):
        return f"st{idx}"

    def stream_round_next(self, st):
        self.calls.append(("round", self.queued))
        self.queued += 1
        return nat.OK

    def stream_progress(self, st):
        mine = torch.tensor([self.queued - self.round], dtype=torch.int64)
        got = [torch.zeros(1, dtype=torch.int64) for _ in range(dist.get_world_size())]
        dist.all_gather(got, mine)
        assert len({int(g) for g in got}) == 1, "ranks queued different numbers of rounds"
        while self.round < self.queued:
            assert self.batch < len(SIZES), "a round was queued past the last batch"
            rem = SIZES[self.batch] - self.off
            room = ROOM[_RoundBus.rank][self.round]
            offer = (0, 1) if room == "stall" else (min(room, rem), 0)
            t = torch.tensor(offer, dtype=torch.int64)
            both = [torch.zeros(2, dtype=torch.int64) for _ in range(dist.get_world_size())]
            dist.all_gather(both, t)
            m = None if any(int(b[1]) for b in both) else min(int(b[0]) for b in both)
            self.calls.append(("resolved", self.round, self.batch, m))
            if m is None or (m == 0 and rem):
                self.stalled += 1
            elif m == rem:
                self.batch, self.off = self.batch + 1, 0
            else:
                self.off += m
            self.round += 1
        self.calls.append(("progress", self.batch, self.off))
        return nat.OK, self.batch, self.off, self.stalled

    def stream_close(self, st):
        pass

    def close(self):
        pass


def _worker(rank, world, port, out, depth):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        _RoundBus.rank = rank
        sb = sharding.ShardedBus(37, dist=dist, rank=rank, world=world, bus_factory=_RoundBus, batch_cap=16,
                                 stream_slots=8, lossless=True)
        box = [len(SIZES) if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)                      # all a follower is told
        pumps = []
        queued = sb.run_rounds(int(box[0]), pump=lambda: pumps.append(sb.bus.queued), depth=depth)
        refused = False
        try:
            sharding.ShardedBus(37, dist=dist, rank=rank, world=world, bus_factory=_RoundBus, batch_cap=16,
                                stream_slots=8).follow_rounds(1)
        except RuntimeError:
            refused = True
        torch.save({"calls": sb.bus.calls, "queued": queued, "pumps": pumps, "progress": sb.progress(),
                    "refused": refused}, f"{out}.{rank}")
        sb.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(180)
@pytest.mark.parametrize("depth", [1, 3, 8])
def test_round_driver_stops_together_at_T(tmp_path, depth):
    out = str(tmp_path / "rr")
    mp.spawn(_worker, args=(2, _free_port(), out, depth), nprocs=2, join=True)
    r0, r1 = (torch.load(f"{out}.{r}", weights_only=False) for r in (0, 1))
    assert r0["calls"] == r1["calls"] and r0["queued"] == r1["queued"] and r0["pumps"] == r1["pumps"]
    assert r0["progress"] == r1["progress"]
    assert r0["progress"][:2] == (len(SIZES), 0) and r0["progress"][2] > 0      # done at T, after stalls
    assert r0["refused"] and r1["refused"]                          # throughput mode queues no rounds
    # never more rounds outstanding than batches remain (nor than the depth), and nothing past batch T
    done, outstanding = 0, 0
    for c in r0["calls"]:
        if c[0] == "round":
            outstanding += 1
            assert outstanding <= min(depth, len(SIZES) - done)
        elif c[0] == "resolved":
            assert c[2] < len(SIZES)
        elif c[0] == "progress":
            done, outstanding = c[1], 0
    assert r0["calls"][-1] == ("progress", len(SIZES), 0)
    assert r0["queued"] == sum(1 for c in r0["calls"] if c[0] == "round")
