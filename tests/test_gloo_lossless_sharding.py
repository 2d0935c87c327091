"""ShardedBus(lossless=True) host logic at world_size 2 on CPU/gloo.  Each rank's GPU bus is replaced by a stand-in that
scripts the prefix its mailboxes admit (or a stall) round by round, and whose offer / agree exchange the offers over gloo
in place of the offer words and the agree kernel.  Every rank must offer before it waits, see the same agreed prefix,
return EAGAIN in the same rounds (when either rank stalls) and resume the batch at the same record.  The device protocol
itself runs in tests/test_gpu_stream_agree.py and tests/test_gpu_multi_lossless.py."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import oracle_binding as ob
from containerpilot_b200 import _native as nat
from containerpilot_b200 import sharding

# (n, now_ns) of each batch, and per rank the room its mailboxes have in each admission round ("stall": admit says EAGAIN)
BATCHES = [(10, 1000), (5, 2000), (0, 3000), (7, 4000)]
SCRIPT = {
    0: [10, "stall", 3, 10, 5, 0, 0, 2, 2, 9],
    1: [4, 10, "stall", 10, 5, "stall", 0, 9, 0, 9],
}
# what both ranks must see: fanout's return per round, and the agreed prefix (None: a stall) per round
WANT_RC = [nat.EAGAIN, nat.EAGAIN, nat.EAGAIN, nat.OK, nat.OK, nat.EAGAIN, nat.OK, nat.EAGAIN, nat.EAGAIN, nat.OK]
WANT_M = [4, None, None, 6, 5, None, 0, 2, 0, 5]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


class _ScriptedBus:
    rank = 0

    def __init__(self, n, **kw):
        self.kw, self.calls = kw, []
        self.round, self.get_off, self.offer = 0, 0, None

    def stream_create(self, slots, n_consumers):
        return "st0", b"H" * 64

    def stream_open(self, handle, idx):
        return f"st{idx}"

    def stream_put(self, st, ev, now, raw=False, nowait=False):
        self.calls.append(("put", len(ev), now)); return nat.OK

    def stream_admit(self, st, n, now):
        room = SCRIPT[_ScriptedBus.rank][self.round]
        self.calls.append(("admit", self.round, n, now))
        if room == "stall":
            raise nat.CpbusError(nat.EAGAIN, "cpbus_stream_admit")
        return min(room, n - self.get_off)

    def stream_offer(self, st, prefix, stalled=False):
        assert self.offer is None, "second offer in one round"
        self.calls.append(("offer", self.round, prefix, bool(stalled)))
        self.offer = (prefix, bool(stalled))

    def stream_agree(self, st):
        assert self.offer is not None, "agree without an offer"
        mine = torch.tensor([self.offer[0], int(self.offer[1]), self.round], dtype=torch.int64)
        got = [torch.zeros(3, dtype=torch.int64) for _ in range(dist.get_world_size())]
        dist.all_gather(got, mine)
        assert len({int(g[2]) for g in got}) == 1, "ranks in different rounds"
        stalled = any(int(g[1]) for g in got)
        m = None if stalled else min(int(g[0]) for g in got)
        self.calls.append(("agree", self.round, m))
        self.round, self.offer = self.round + 1, None
        if stalled:
            raise nat.CpbusError(nat.EAGAIN, "cpbus_stream_agree")
        return m

    def stream_fanout_prefix(self, st, n, now, m):
        self.calls.append(("fanout_prefix", n, now, m, self.get_off))
        if m == n - self.get_off:
            self.get_off = 0
            return nat.OK
        self.get_off += m
        return nat.EAGAIN

    def stream_fanout(self, st, n, now):
        raise AssertionError("a lossless ShardedBus must not use the throughput-mode fan-out")

    def stream_close(self, st):
        pass

    def close(self):
        pass


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        _ScriptedBus.rank = rank
        sb = sharding.ShardedBus(37, dist=dist, rank=rank, world=world, bus_factory=_ScriptedBus, batch_cap=16,
                                 stream_slots=8, lossless=True)
        assert sb.stream_ok and sb.bus.kw["lossless"] is True
        rcs = []
        for n, now in BATCHES:
            rc = sb.publish(np.zeros(n, dtype=ob.EVENT_DTYPE), now)   # one round: publish does not retry
            rcs.append(rc)
            while rc != nat.OK:
                assert rc == nat.EAGAIN
                rc = sb.fanout(n, now)                                 # (consumers drain here) then the next round
                rcs.append(rc)
        refused = []
        for call in (lambda: sb.fanout_trace(0, 1, 1), lambda: sb.fanout_broadcast(None, 1, 1)):
            try:
                call()
            except RuntimeError:
                refused.append(True)
        torch.save({"rcs": rcs, "calls": sb.bus.calls, "refused": refused}, f"{out}.{rank}")
        sb.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(180)
def test_lossless_sharded_bus_rounds_in_lockstep_at_world2(tmp_path):
    out = str(tmp_path / "ll")
    mp.spawn(_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    r0, r1 = (torch.load(f"{out}.{r}", weights_only=False) for r in (0, 1))
    assert r0["rcs"] == r1["rcs"] == WANT_RC
    assert r0["refused"] == r1["refused"] == [True, True]          # device batches stay throughput-only
    for r in (r0, r1):
        calls = [c for c in r["calls"] if c[0] != "put"]
        # every round: admit, offer, agree — the offer strictly before the wait — then a fan-out unless someone stalled
        agreed = [c[2] for c in calls if c[0] == "agree"]
        assert agreed == WANT_M
        i = 0
        for rnd, m in enumerate(WANT_M):
            assert [c[0] for c in calls[i:i + 3]] == ["admit", "offer", "agree"] and calls[i][1] == rnd
            i += 3
            if m is not None:
                assert calls[i][0] == "fanout_prefix" and calls[i][3] == m
                i += 1
        assert i == len(calls)
    rank_offers = [[c for c in r["calls"] if c[0] == "offer"] for r in (r0, r1)]
    assert [c[3] for c in rank_offers[0]] == [s == "stall" for s in SCRIPT[0]]   # a stalled admit offers (0, stalled)
    assert all(c[2] == 0 for c in rank_offers[1] if c[3])
    # both ranks fan out the same records: the same m at the same resume offset of the same batch
    fan = [[c for c in r["calls"] if c[0] == "fanout_prefix"] for r in (r0, r1)]
    assert fan[0] == fan[1]
    assert [(c[1], c[4]) for c in fan[0]] == [(10, 0), (10, 4), (5, 0), (0, 0), (7, 0), (7, 2), (7, 2)]
    puts0 = [c for c in r0["calls"] if c[0] == "put"]
    assert puts0 == [("put", n, now) for n, now in BATCHES] and not any(c[0] == "put" for c in r1["calls"])
