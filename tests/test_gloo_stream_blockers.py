"""ShardedBus.blockers / ShardedBus.lagging at world_size 2 on CPU/gloo: the aggregation only.  Each rank's GPU bus is
replaced by a stand-in whose per-shard answers (stream_blockers, lagging) are scripted from one fleet-wide table of
backlogs, losses and blocking mailboxes.  Every rank must return the identical global answer: the ids merged in ascending
order, the summaries added with backlog_max the maximum, and lagging's entries and next_sub those of one bus over the
whole fleet, paging across the ranks in cyclic order.  The per-shard queries run on hardware in
tests/test_gpu_stream_blockers.py and tests/test_gpu_multi_stream_blockers.py."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from containerpilot_b200 import _native as nat
from containerpilot_b200 import sharding

N = 41                                              # shards [0, 21) and [21, 41)
_rng = np.random.default_rng(77)
BACKLOG = _rng.integers(0, 9, N) * (_rng.random(N) < 0.6)
LOST = np.where(_rng.random(N) < 0.2, _rng.integers(1, 50, N), 0)
ACTIVE = _rng.random(N) < 0.9
BLOCKING = [[2, 5, 6, 19], [21, 30, 40]]            # per rank, ascending, inside its shard


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def one_bus_lagging(first, n, start, min_backlog, cap):
    """cpbus_lagging of one bus holding every mailbox of the table"""
    lag, summ = [], {"active": 0, "lagging": 0, "backlog_total": 0, "backlog_max": 0, "lost_total": 0, "hist": [0] * 33}
    for p in range(n):
        s = first + (start - first + p) % n
        if not ACTIVE[s]:
            continue
        b, l = int(BACKLOG[s]), int(LOST[s])
        summ["active"] += 1; summ["backlog_total"] += b; summ["lost_total"] += l
        summ["backlog_max"] = max(summ["backlog_max"], b); summ["hist"][b.bit_length()] += 1
        if b >= min_backlog:
            lag.append((s, b, l))
    summ["lagging"] = len(lag)
    ent = np.zeros(min(cap, len(lag)), dtype=nat.LAG_DTYPE)
    for i, (s, b, l) in enumerate(lag[:cap]):
        ent[i] = (s, b, l)
    return ent, (lag[cap][0] if len(lag) > cap else start), summ


class _ScriptedBus:
    rank = 0

    def __init__(self, n, sub_id_base=0, **kw):
        self.first, self.n = sub_id_base, n

    def stream_create(self, slots, n_consumers):
        return "st0", b"H" * 64

    def stream_open(self, handle, idx):
        return f"st{idx}"

    def stream_blockers(self, st, cap=None):
        ids = np.array(BLOCKING[_ScriptedBus.rank], dtype=np.uint32)
        return ids if cap is None else ids[:cap]

    def lagging(self, first_sub, n, start_sub=None, min_backlog=1, cap=None):
        assert self.first <= first_sub and first_sub + n <= self.first + self.n, "a piece outside this shard"
        return one_bus_lagging(first_sub, n, first_sub if start_sub is None else start_sub, min_backlog,
                               n if cap is None else cap)

    def stream_close(self, st):
        pass

    def close(self):
        pass


QUERIES = [(0, N, 0, 1, None), (0, N, 30, 1, None), (0, N, 10, 0, 5), (3, 30, 25, 2, 3), (20, 2, 21, 0, 1),
           (0, N, 40, 3, 0), (5, 36, 5, 1, 100), (10, 20, 29, 1, 4)]


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        _ScriptedBus.rank = rank
        sb = sharding.ShardedBus(N, dist=dist, rank=rank, world=world, bus_factory=_ScriptedBus, batch_cap=16,
                                 stream_slots=8, lossless=True)
        res = {"blockers": [sb.blockers().tolist(), sb.blockers(cap=2).tolist(), sb.blockers(cap=5).tolist()]}
        lag = []
        for first, n, start, mb, cap in QUERIES:
            ent, nxt, summ = sb.lagging(first, n, start_sub=start, min_backlog=mb, cap=cap)
            lag.append((ent.tobytes(), nxt, summ))
        res["lagging"] = lag
        pages = []                                  # page through the whole fleet, 3 entries at a time
        cur = 17
        for _ in range(8):
            ent, cur, _ = sb.lagging(0, N, start_sub=cur, min_backlog=1, cap=3)
            pages.append(([int(x) for x in ent["sub_id"]], cur))
        res["pages"] = pages
        torch.save(res, f"{out}.{rank}")
        sb.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(180)
def test_every_rank_returns_the_one_bus_answer(tmp_path):
    out = str(tmp_path / "sb")
    mp.spawn(_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    r0, r1 = (torch.load(f"{out}.{r}", weights_only=False) for r in (0, 1))
    assert r0 == r1
    every = sorted(BLOCKING[0] + BLOCKING[1])
    assert r0["blockers"] == [every, every[:2], every[:5]]
    for (first, n, start, mb, cap), (ent, nxt, summ) in zip(QUERIES, r0["lagging"]):
        e, x, s = one_bus_lagging(first, n, start, mb, n if cap is None else cap)
        assert ent == e.tobytes() and nxt == x and summ == s, (first, n, start, mb, cap)
    assert any(s["backlog_max"] > 0 and s["lagging"] > 0 for _, _, s in r0["lagging"])
    # paging resumes at next_sub across the shard boundary and around the end of the range
    lag_ids = [s for s in list(range(17, N)) + list(range(17)) if ACTIVE[s] and BACKLOG[s] >= 1]
    walked = [i for ids, _ in r0["pages"] for i in ids]
    L = len(lag_ids)
    assert L > 8 and walked[:L] == lag_ids
    assert [nx for _, nx in r0["pages"]][:L // 3] == [lag_ids[3 * (k + 1) % L] for k in range(L // 3)]
