"""The sparse drains' list scan across tile boundaries: a CPBUS_CFG_SPARSE_DRAINS bus whose ready calls scan a candidate
list of more than one tile (1,024 candidates) gives the results of a twin without the flag, which scans the whole range.
That takes a bus of more than 1,024 x 4,096 mailboxes, since the list is used for at most max(256, N / 4096) candidates.
Records reach the candidates through sparse record launches after consume_all, so the flagged bus's index knows them; each
cpbus_drain_ready, cpbus_take_ready and ticket is cut in the list's first tile, in its second, or not at all, with the walk
starting at and wrapping around several start ids, in throughput and lossless mode."""
import numpy as np
import pytest

from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus

pytestmark = pytest.mark.gpu
N = 5 << 20                       # list cap N / 4096 = 1,280 candidates
R, TILE, M = 64, 1024, 1200       # ring_cap, candidates per tile of the scan, candidates
GROUPS = 4                        # candidate j takes code 1 + group[j]; everyone else code 5 (never published)


def _result(r):
    return r[0].tobytes(), r[1].tobytes(), len(r[1]), len(r[0]), r[2]


def _launches(bus):
    return bus.stats()["kernel_launches"]


@pytest.mark.parametrize("lossless", [False, True])
def test_list_scan_across_tiles_equals_dense_scan(lossless):
    rng = np.random.default_rng(4242 + lossless)
    cand = np.sort(rng.choice(N - 1, M, replace=False)).astype(np.uint32)
    group = rng.integers(0, GROUPS, M)
    masks = np.full(N, 1 << 5, dtype=np.uint32)
    masks[cand] = (1 << (1 + group)).astype(np.uint32)
    kw = dict(ring_cap=R, batch_cap=32, timers_per_sub=0, lossless=lossless, device=0, sparse_records=True)
    with Bus(N, **kw) as plain, Bus(N, sparse_drains=True, **kw) as bus:
        both = (plain, bus)
        for x in both:
            x.subscribe_many(masks)
            x.consume_all()
        empty = (int(cand[-1]) + 1, N - int(cand[-1]) - 1)   # a range without candidates: the flagged bus launches nothing

        def deliver(counts):
            """counts[g] records of code 1 + g, at most 16 per flush: each flush is a sparse record launch"""
            for g, c in enumerate(counts):
                for i in range(0, c, 16):
                    for x in both:
                        for _ in range(min(16, c - i)):
                            assert x.publish(1 + g, 7) == nat.OK
                        assert x.flush() == nat.OK

        def call(kind, start, cap, ready_cap):
            got = []
            for x in both:
                b0 = _launches(x)
                if kind == "ticket":
                    t = (x.take_ready_begin if lossless else x.drain_ready_begin)(0, N, start, cap, ready_cap)
                    r = x.drain_ready_end(t, cap, ready_cap)
                else:
                    r = getattr(x, kind)(0, N, start, cap, ready_cap)
                got.append((_result(r), _launches(x) - b0))
                if lossless and kind != "drain_ready" and len(r[1]):   # a take: release what it took
                    assert (x.ack_many(r[1]["sub_id"], r[1]["count"]) == nat.OK).all()
            (want, n_plain), (res, n_bus) = got
            assert res == want, (kind, start, cap, ready_cap)
            assert n_plain == 2 and n_bus == 2     # a scan and a gather on both
            return res

        def known():
            """the flagged bus's index knows where records are: a drain of a range without candidates launches nothing"""
            b0 = _launches(bus)
            r = bus.drain_ready(empty[0], empty[1], empty[0], 4 * R, 16)
            assert len(r[1]) == 0 and _launches(bus) == b0

        kinds = ["drain_ready", "ticket"] + (["take_ready"] if lossless else [])
        # throughput mode: group 0 is overwritten (more than ring_cap records), so its cursor is tail - ring_cap
        counts = [R + 6 if not lossless else 5, 1, 3, 2]
        for start, start_at in ((0, 0), (int(cand[700]), 700), (int(cand[M - 50]), M - 50)):
            walk = np.roll(np.arange(M), -start_at)               # candidates in walk order
            cum = np.cumsum([min(counts[g], R) for g in group[walk]])
            for kind in kinds:
                # (entries taken, cap, ready_cap): cut by ready_cap or by cap in the first tile, in the second, or not at all
                for taken, cap, ready_cap in ((300, 1 << 20, 300), (TILE + 100, 1 << 20, TILE + 100),
                                              (400, int(cum[399]), M), (TILE + 50, int(cum[TILE + 49]), M), (M, 1 << 20, M)):
                    for x in both:   # empty mailboxes; in lossless mode also a full room bound, so each flush stays sparse
                        x.consume_all()
                    deliver(counts)
                    known()
                    res = call(kind, start, cap, ready_cap)
                    assert res[2] == taken and res[3] == cum[taken - 1], (kind, start, taken)
                    assert res[4] == (start if taken == M else int(cand[walk[taken]]))
                    if taken < M:                                       # the rest, so that every case starts empty
                        rest = call("drain_ready", res[4], 1 << 20, M)
                        assert res[2] + rest[2] == M and rest[4] == res[4]
                    known()
