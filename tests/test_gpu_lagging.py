"""Consumer backlog on the device: `cpbus_lagging` (which mailboxes fall behind, by how much, how much they lost) and
`cpbus_blockers` (which mailboxes a stalled lossless publish waits on), against the oracle, read-only, paged, on the group,
behind outstanding stream followers and rounds, and through the Python mirror."""
import os
import subprocess

import numpy as np
import pytest

import lag_oracle as lo
import oracle_binding as ob
from containerpilot_b200 import _native as nat
from containerpilot_b200 import events
from containerpilot_b200.bus import Bus, EVENT_DTYPE
from containerpilot_b200.events import Event
from containerpilot_b200.group import GroupBus
from test_gpu_group import _apply, _consume, _consumers, _eq, _trace

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _hist(backlogs):
    h = [0] * 33
    for b in backlogs:
        h[int(b).bit_length()] += 1
    return h


def _expected(orc, subs, R, lossless, min_backlog):
    """(entries, summary) the oracle implies for mailboxes `subs` (the active ones, in visiting order)"""
    ent, bl, lost = [], [], []
    for s in subs:
        held = int(lo.backlog(orc, s))
        b, l = (held, 0) if lossless else (min(held, R), max(0, held - R))
        bl.append(b); lost.append(l)
        if b >= min_backlog:
            ent.append((s, b, l))
    summary = {"active": len(subs), "lagging": len(ent), "backlog_total": sum(bl), "backlog_max": max(bl, default=0),
               "lost_total": sum(lost), "hist": _hist(bl)}
    return ent, summary


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("lossless", [False, True])
def test_backlog_matches_the_oracle(lossless, seed):
    """Random traces with partial drains, unsubscribes, pair tables, unicast sends and timers.  Lossless mode: the oracle's
    mailbox_cap is the ring, and consumers keep every mailbox from stalling.  Throughput mode: the oracle is unbounded, so
    backlog = min(held, R) and lost = held - R since the last drain.  Every entry and the whole summary match."""
    N, R, B, K = 24, 64, 32, 2
    rng = np.random.default_rng(seed * 31 + lossless)
    orc = ob.Oracle(N, timers_per_sub=K, keep_window=0, mailbox_cap=R if lossless else 0)
    active = []
    with Bus(N, ring_cap=R, batch_cap=B, timers_per_sub=K, lossless=lossless) as bus:
        for s in range(N):
            mask = nat.MASK_ALL if s % 4 == 0 else (0 if s % 7 == 6 else int(rng.integers(0, 1 << 8)))
            pairs = [(int(rng.integers(0, 8)), int(rng.integers(0, 5))) for _ in range(2)] if s % 3 == 1 else []
            assert (bus.subscribe_pairs(mask, pairs) if pairs else bus.subscribe(mask)) == s
            orc.subscribe(mask, pairs=pairs)
            active.append(s)
            if s % 5 == 0 or mask == 0:
                p = int(rng.integers(400, 1500))
                bus.timer_add(s, p, 900 + s, oneshot=s % 10 == 5)
                orc.timer_add(s, p, 900 + s, s % 10 == 5)
        now, lost_seen = 0, False
        for step in range(120):
            now += int(rng.integers(0, 700))
            assert bus.advance(now) == nat.OK and orc.advance(now) == 0
            for _ in range(int(rng.integers(0, 12))):
                if rng.random() < 0.85:
                    code, src = int(rng.integers(0, 8)), int(rng.integers(0, 5))
                    assert bus.publish(code, src) == nat.OK and orc.publish(code, src) == 0
                else:
                    s = active[int(rng.integers(0, len(active)))]
                    assert bus.send(s, 3, 7) == nat.OK and orc.receive(s, 3, 7) == 0
            assert bus.flush() == nat.OK
            for s in list(active):                            # consumers: partial drains, whole drains past the ring
                held = int(lo.backlog(orc, s))
                if rng.random() < 0.25 or (lossless and held > R - 20):
                    take = int(rng.integers(1, R + 1)) if (held <= R and not (lossless and held > R - 20)) else R
                    take = max(take, held - (R - 20)) if lossless else take
                    g = bus.drain(s, cap=take)
                    if held > R:                              # throughput: the oldest were overwritten; take the rest
                        orc.consume(s, held)
                    else:
                        assert g.tobytes() == orc.consume(s, take).tobytes()
            if step == 70:
                for s in (2, 9):
                    bus.unsubscribe(s); orc.unsubscribe(s); active.remove(s)
            mb = int(rng.integers(0, 40)) if step % 3 else 0
            ent, nxt, summ = bus.lagging(0, N, min_backlog=mb)
            exp, exp_sum = _expected(orc, active, R, lossless, mb)
            assert [tuple(int(x) for x in e) for e in ent] == exp, step
            assert summ == exp_sum, step
            assert nxt == 0
            start = int(rng.integers(0, N))
            order = [s for s in list(range(start, N)) + list(range(start)) if s in active]
            ent, nxt, summ = bus.lagging(0, N, start_sub=start, min_backlog=mb)
            assert [int(e["sub_id"]) for e in ent] == [e[0] for e in _expected(orc, order, R, lossless, mb)[0]]
            assert summ == exp_sum and nxt == start
            lost_seen = summ["lost_total"] > 0 or lost_seen
        assert lost_seen != lossless


def _fill(bus, rng, N, steps=40):
    for _ in range(steps):
        ev = np.zeros(int(rng.integers(1, 32)), dtype=EVENT_DTYPE)
        ev["code"] = rng.integers(0, 6, ev.size); ev["source_id"] = rng.integers(0, 9, ev.size)
        assert bus.publish_many(ev) == nat.OK
        if rng.random() < 0.3:
            assert bus.send(int(rng.integers(0, N)), 4, 1) == nat.OK
        rc = bus.flush()
        assert rc == nat.OK
        s = int(rng.integers(0, N))
        bus.drain(s, cap=int(rng.integers(1, 65)))


@pytest.mark.parametrize("lossless", [False, True])
def test_lagging_is_read_only_and_lists_what_drain_ready_takes(lossless):
    """lagging then drain_ready equals drain_ready alone (records, ready list, next_sub); with min_backlog=1 and large caps
    lagging lists exactly the ids, counts and losses drain_ready then takes; repeated calls are byte-identical."""
    N, R = 300, 128
    masks = np.random.default_rng(5).integers(0, 1 << 6, N).astype(np.uint32)
    masks[::4] = nat.MASK_ALL
    buses = [Bus(N, ring_cap=R, batch_cap=32, lossless=lossless) for _ in range(2)]
    try:
        for b in buses:
            b.subscribe_many(masks)
            _fill(b, np.random.default_rng(6), N, steps=3 if lossless else 40)
        a, b = buses
        first = [a.lagging(0, N, start_sub=37, min_backlog=1) for _ in range(3)]
        for x in first[1:]:
            assert x[0].tobytes() == first[0][0].tobytes() and x[1:] == first[0][1:]
        st0 = a.stats()["kernel_launches"]
        a.lagging(10, 200, start_sub=50, min_backlog=0, cap=0)
        assert a.stats()["kernel_launches"] == st0 + 1
        ra = a.drain_ready(0, N, 37, cap=N * R, ready_cap=N)
        rb = b.drain_ready(0, N, 37, cap=N * R, ready_cap=N)
        assert ra[0].tobytes() == rb[0].tobytes() and ra[1].tobytes() == rb[1].tobytes() and ra[2] == rb[2]
        ent = first[0][0]
        assert len(ent) == len(ra[1]) > 0
        assert (ent["sub_id"] == ra[1]["sub_id"]).all() and (ent["backlog"] == ra[1]["count"]).all()
        assert (ent["lost"] == ra[1]["lost"]).all()
        assert (ent["lost"] > 0).any() != lossless
        ent2, _, summ2 = a.lagging(0, N, min_backlog=0)
        assert summ2["backlog_total"] == 0 and summ2["active"] == N and len(ent2) == N
    finally:
        for x in buses:
            x.close()


def test_paging_visits_every_lagging_mailbox_once_in_cyclic_order():
    N, R = 500, 64
    rng = np.random.default_rng(11)
    with Bus(N, ring_cap=R, batch_cap=32) as bus:
        masks = rng.integers(0, 1 << 5, N).astype(np.uint32)
        bus.subscribe_many(masks)
        _fill(bus, rng, N, steps=20)
        for cap in (1, 2, 7):
            for _ in range(3):
                first, n = int(rng.integers(0, 100)), int(rng.integers(50, 400))
                start = first + int(rng.integers(0, n))
                mb = int(rng.integers(1, 6))
                full, _, summ = bus.lagging(first, n, start_sub=start, min_backlog=mb)
                assert len(full) == summ["lagging"]
                L = summ["lagging"]
                assert L > cap
                got, cur = [], start
                while len(got) < L:
                    page, nxt, s2 = bus.lagging(first, n, start_sub=cur, min_backlog=mb, cap=cap)
                    assert s2 == summ and len(page) == cap
                    got += [int(x) for x in page["sub_id"]]
                    assert nxt == int(full["sub_id"][len(got) % L])     # the first lagging mailbox not returned
                    cur = nxt
                assert got[:L] == [int(x) for x in full["sub_id"]]


def _stall_run(seed, via, policy):
    """The loop of test_flush_blocks_per_event_like_the_go_bus with timers, pair cases and unicast sends.  Tick phase: the
    clock moves and the ticks due fire with nothing staged.  Record phase: B events (broadcast or unicast) are staged and
    pushed by cpbus_flush, by the auto-flush of one more publish, or by a membership call.  The oracle sends one at a time.
    At every CPBUS_EAGAIN, blockers() equals the oracle's blockers for the refused unit.  policy 'blockers' drains exactly
    the blockers and checks that the next attempt delivers more."""
    N, R, B, K = 8, 64, 32, 1
    rng = np.random.default_rng(200 + seed)
    masks = [nat.MASK_ALL, 1 << 2, (1 << 3) | (1 << 2), nat.MASK_ALL, 1 << 5, 1 << 1, 1 << 4, 0]
    pairs = {1: [(3, 1), (5, 2)], 4: [(2, 0)]}
    orc = ob.Oracle(N, timers_per_sub=K, keep_window=0, mailbox_cap=R)
    stalls = {"tick": 0, "record": 0, "partial": 0}
    with Bus(N, ring_cap=R, batch_cap=B, timers_per_sub=K, lossless=True) as bus:
        for s, m in enumerate(masks):
            assert (bus.subscribe_pairs(m, pairs[s]) if s in pairs else bus.subscribe(m)) == s
            orc.subscribe(m, pairs=pairs.get(s))
        for s in (0, 5, 7):
            bus.timer_add(s, 700 + 100 * s, 50 + s)
            orc.timer_add(s, 700 + 100 * s, 50 + s)

        def counts():
            return [int(c) for c in bus.digests(0, N)["count"]]

        def on_stall(expected):
            got = bus.blockers()
            assert got.tolist() == expected.tolist()
            assert len(got) >= 1
            before = sum(counts())
            if policy == "blockers":
                for s in got:
                    assert bus.drain(int(s), cap=R).tobytes() == orc.consume(int(s), R).tobytes()
            else:
                for s in rng.permutation(N)[:3]:
                    take = int(rng.integers(1, R + 1))
                    assert bus.drain(int(s), cap=take).tobytes() == orc.consume(int(s), take).tobytes()
            return before

        now = 0
        for step in range(45):
            now += int(rng.integers(0, 6000))
            assert bus.advance(now) == nat.OK
            progress_from = None
            while True:                                               # tick phase
                exp = lo.blockers(orc, now)
                rc = bus.flush()
                if progress_from is not None and policy == "blockers":
                    assert sum(counts()) > progress_from
                if len(exp) == 0:
                    assert rc == nat.OK and orc.advance(now) == 0
                    break
                assert rc == nat.EAGAIN
                stalls["tick"] += 1
                progress_from = on_stall(exp)
            assert counts() == [int(orc.count(s)) for s in range(N)]
            evs = []
            for _ in range(B + (via == "auto")):
                if rng.random() < 0.2:
                    evs.append((int(rng.integers(1, 7)), 0, int(rng.integers(0, N))))
                else:
                    evs.append((int(rng.integers(1, 7)), int(rng.integers(0, 3)), nat.TARGET_ALL))
            for code, src, tgt in evs[:B]:
                assert (bus.publish(code, src) if tgt == nat.TARGET_ALL else bus.send(tgt, code, src)) == nat.OK
            i, extra_pending, progress_from = 0, via == "auto", None
            while True:                                               # record phase
                if extra_pending:
                    code, src, tgt = evs[B]
                    rc = bus.publish(code, src) if tgt == nat.TARGET_ALL else bus.send(tgt, code, src)
                    extra_pending = rc != nat.OK
                    if rc == nat.OK:
                        rc = bus.flush()
                elif via == "member":
                    s = int(rng.integers(0, N))
                    rc = bus._lib.cpbus_set_mask(bus._h, s, masks[s])
                else:
                    rc = bus.flush()
                if progress_from is not None and policy == "blockers":
                    assert sum(counts()) > progress_from
                while i < len(evs) and not (extra_pending and i == B):
                    code, src, tgt = evs[i]
                    r = orc.publish(code, src) if tgt == nat.TARGET_ALL else orc.receive(tgt, code, src)
                    if r == ob.EAGAIN:
                        break
                    assert r == 0
                    i += 1
                assert counts() == [int(orc.count(s)) for s in range(N)], (step, i, rc)
                if rc == nat.OK:
                    assert i == len(evs)
                    break
                assert rc == nat.EAGAIN and i < len(evs)
                stalls["record"] += 1
                stalls["partial"] += i > 0
                code, src, tgt = evs[i]
                progress_from = on_stall(lo.blockers(orc, now, code, src, tgt))
        for s in range(N):
            assert bus.drain(s, cap=R).tobytes() == orc.consume(s, R).tobytes()
        assert bus.stats()["overwritten"] == 0
    return stalls


@pytest.mark.parametrize("via", ["flush", "auto", "member"])
@pytest.mark.parametrize("policy", ["random", "blockers"])
def test_blockers_match_the_oracle_at_every_stall(via, policy):
    stalls = _stall_run({"flush": 1, "auto": 2, "member": 3}[via] + (10 if policy == "blockers" else 0), via, policy)
    assert stalls["tick"] > 0 and stalls["record"] > 0, stalls
    if policy == "random":
        assert stalls["partial"] > 0, stalls


def test_blockers_in_throughput_mode_launch_nothing():
    with Bus(64, ring_cap=64, batch_cap=32, timers_per_sub=1) as bus:
        bus.subscribe_many(np.full(64, nat.MASK_ALL, dtype=np.uint32))
        bus.timer_add(3, 100, 1)
        for i in range(200):
            assert bus.publish(1, i) == nat.OK
        bus.advance(10_000)
        k0 = bus.stats()["kernel_launches"]
        assert len(bus.blockers()) == 0 and len(bus.blockers(cap=0)) == 0
        assert bus.stats()["kernel_launches"] == k0
        ent, _, summ = bus.lagging(0, 64)
        assert summ["backlog_max"] == 64 and summ["lost_total"] > 0


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("G", [1, 2, 3, 4])
def test_group_queries_equal_one_bus(G, lossless, monkeypatch):
    """The group's seeded twin trace (pairs, unicast, timers, clock jumps, consumers): after every op, lagging (random
    range, start, min_backlog and cap) and blockers give the same outputs on G shards of one GPU as on one bus."""
    monkeypatch.setenv("CPBUS_PDL", "0")
    monkeypatch.setenv("CPBUS_HINTS", "2")
    seed = 300 + 10 * G + lossless
    ops, n_total = _trace(seed, 24, 900, 4, jump_every=150)
    rng = np.random.default_rng(seed + 1)
    R = 64
    kw = dict(ring_cap=R, batch_cap=32, timers_per_sub=4, lossless=lossless)
    one, grp = Bus(n_total + 4, device=0, **kw), GroupBus(n_total + 4, [0] * G, **kw)
    ha, hb = [], []
    n_ids = n_block = 0
    try:
        for i, op in enumerate(ops):
            a, b = _apply(one, op, ha), _apply(grp, op, hb)
            _eq(a, b, f"op {i} {op}")
            n_ids += op[0] == "sub" and a[0] == nat.OK
            if not n_ids:
                continue
            if a[0] == nat.EAGAIN or rng.random() < 0.15:
                x, y = one.blockers(), grp.blockers()
                assert x.tolist() == y.tolist(), (i, op)
                n_block += len(x) > 0
                if a[0] == nat.EAGAIN and lossless:
                    assert len(x) > 0, (i, op)
                first = int(rng.integers(0, n_ids))
                n = int(rng.integers(1, n_ids - first + 1))
                args = (first, n, first + int(rng.integers(0, n)), int(rng.integers(0, 4)), int(rng.integers(0, 6)))
                la, lb = one.lagging(*args[:2], start_sub=args[2], min_backlog=args[3], cap=args[4]), \
                    grp.lagging(*args[:2], start_sub=args[2], min_backlog=args[3], cap=args[4])
                assert la[0].tobytes() == lb[0].tobytes() and la[1:] == lb[1:], (i, args)
            if a[0] == nat.EAGAIN or rng.random() < 0.08:
                for _ in range(int(rng.integers(1, 4))):
                    c = _consumers(rng, n_ids, R)
                    _eq(_consume(one, c), _consume(grp, c), f"op {i} consumer {c}")
        if lossless:
            assert n_block > 0
    finally:
        one.close(); grp.close()


@pytest.mark.parametrize("lossless", [False, True])
def test_queries_resolve_outstanding_followers_and_rounds_first(lossless):
    """lagging / blockers called with stream followers (throughput) or lossless rounds outstanding equal the same calls
    made after cpbus_stream_progress has resolved them."""
    N, R, B = 64, 64, 32
    rng = np.random.default_rng(41 + lossless)
    batches = []
    for _ in range(5):
        ev = np.zeros(int(rng.integers(8, B + 1)), dtype=EVENT_DTYPE)
        ev["code"] = rng.integers(0, 5, ev.size); ev["source_id"] = rng.integers(0, 4, ev.size)
        batches.append(ev)
    masks = rng.integers(0, 1 << 5, N).astype(np.uint32)
    out = []
    for resolve_first in (False, True):
        with Bus(N, ring_cap=R, batch_cap=B, timers_per_sub=1, lossless=lossless) as bus:
            bus.subscribe_many(masks)
            bus.timer_add_many(0, N, 3000, source_id0=10)
            st, _ = bus.stream_create(8, 1)
            for k, ev in enumerate(batches):
                assert bus.stream_put(st, ev, (k + 1) * 1000) == nat.OK
            for _ in batches:
                assert (bus.stream_round_next(st) if lossless else bus.stream_fanout_next(st)) == nat.OK
            if resolve_first:
                assert bus.stream_progress(st)[0] == nat.OK
            ent, nxt, summ = bus.lagging(0, N, start_sub=5, min_backlog=1)
            blk = bus.blockers()
            out.append((ent.tobytes(), nxt, summ, blk.tolist()))
            assert bus.stream_progress(st)[0] == nat.OK
            bus.stream_close(st)
    assert out[0] == out[1]
    assert out[0][2]["backlog_total"] > 0


def test_event_bus_mirror_names_the_full_subscriber():
    """events.EventBus in lossless mode: when a publish stalls, Blocking() names the subscriber whose channel is full,
    and Lagging() reports its backlog."""
    bus = events.EventBus(lossless=True, ring_cap=64, batch_cap=32)
    try:
        slow, fast = events.Subscriber(events.Chan()), events.Subscriber(events.Chan())
        slow.Subscribe(bus)
        fast.Subscribe(bus)
        assert bus.Blocking() == [] and bus.Lagging() == []
        for i in range(64):
            bus.Publish(Event(events.StatusHealthy, f"e{i}"))
        assert len(fast.Received()) == 64                  # (flushes: slow now holds 64 of 64)
        bus.Publish(Event(events.StatusHealthy, "one more"))
        with pytest.raises(BlockingIOError):
            bus.Flush()
        assert bus.Blocking() == [slow]
        assert bus.Lagging() == [(slow, 64, 0)]
        assert [(s, b) for s, b, _ in bus.Lagging(min_backlog=0)] == [(slow, 64), (fast, 0)]
        assert len(bus._bus.drain(slow._id)) == 64         # the consumer of the full channel runs
        bus.Flush()
        assert bus.Blocking() == [] and bus.Lagging() == [(slow, 1, 0), (fast, 1, 0)]
    finally:
        bus.close()


def test_cpp_mirror_blocking_and_lagging():
    """csrc/host/events_lag_test: Blocking() / Lagging() of events.hpp on one bus and on a group of three shards"""
    exe = os.path.join(ROOT, "containerpilot_b200", "csrc", "host", "events_lag_test")
    assert os.path.exists(exe), "built by the host Makefile"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
