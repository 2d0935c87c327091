"""Every consumer call against the plain reference of `tests/drain_check.py`, at fleet scale: N = 2^20 + 333 mailboxes
(the last scan tile is partial), R = 64, B = 32, one shard at sub_id_base = 3 * 2^20.  Each call is compared byte for
byte with the answer the reference computes from a snapshot of the bus's memory taken just before it, and is followed
by a check that it changed nothing but the cursors it owns.

The fleet is built through the API only.  Code masks from a palette give runs of 0, 1, 2, 15, 16, 17, 31, 32, 33, 63, 64
and (throughput mode) 100 records, an overwritten mailbox; blocks of 40 one-record mailboxes give the ticket gather a
chunk made of 16 runs.  Cursors land on every ring offset, and the ready cells assert it: partial drains of a sample and
overwrites (throughput), consume_all between fills, partial drains, takes of a quarter of the fleet and acks of arbitrary
counts (lossless).  Some mailboxes are unsubscribed or released while they still hold records.  Every cell asserts from
the reference's layout the geometry it claims: the tile the cut fell in, a walk that wrapped, and for tickets where the
16-record chunks fall on the runs."""
import ctypes as C

import numpy as np
import pytest
import torch

import drain_check as dc
import ring_check as rc
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE

pytestmark = pytest.mark.gpu
N, R, B, BASE = (1 << 20) + 333, 64, 32, 3 << 20
HIST = {1: 1, 2: 1, 3: 15, 4: 31, 5: 63, 6: 100}          # records of each code in one fill
SPARE = 8                                                 # a code no fill publishes: the publishes between tickets
# (mask, weight): runs of 0, 1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 100 records per fill
PALETTE = [(1 << SPARE, .46), (0b10, .25), (0b110, .06), (0b1000, .02), (0b1010, .02), (0b1110, .02), (0b10000, .02),
           (0b10010, .02), (0b10110, .02), (0b100000, .02), (0b100010, .02), (0b1000000, .07)]


def _masks(rng, lossless):
    m = np.array([p[0] for p in PALETTE], dtype=np.uint32)
    w = np.array([p[1] for p in PALETTE])
    if lossless:                          # no run beyond R: the 100-record mask takes the 64-record one's place
        m[-1] = 0b100010
    masks = m[rng.choice(len(m), N, p=w / w.sum())]
    for b0 in range(4096, N - 64, 1 << 15):
        masks[b0:b0 + 40] = 0b10         # 40 consecutive one-record mailboxes
    return masks


def _fill(bus, rng, hist=HIST, lossless=False):
    """one round of broadcast records, as device batches of B with the watermark of their last record"""
    codes = rng.permutation(np.repeat(list(hist), list(hist.values())))
    if lossless:
        codes = codes[codes != 6]
    now = bus.stats()["now_ns"]
    rec = np.zeros(len(codes), dtype=EVENT_DTYPE)
    rec["seq"], rec["ts_ns"] = np.arange(len(codes)), now + 1000 * (1 + np.arange(len(codes)))
    rec["code"], rec["source_id"], rec["target"] = codes, rng.integers(0, 4096, len(codes)), nat.TARGET_ALL
    dev = torch.from_numpy(rec.view(np.uint8).reshape(-1, 32).copy()).cuda()
    for i in range(0, len(rec), B):
        j = min(len(rec), i + B)
        nat.check(bus.publish_device(dev.data_ptr() + i * 32, j - i, int(rec["ts_ns"][j - 1])), "publish_device")
    bus.sync()


class Cell:
    """One bus, its zero-copy views and the reference over them"""

    def __init__(self, bus, views, lossless, masks):
        self.bus, self.lossless = bus, lossless
        self.f = dc.Fleet(views[0], views[1], BASE, lossless, sync=bus.sync)
        self.subscribed = torch.ones(N, dtype=torch.bool, device="cuda")
        self.known = torch.ones(N, dtype=torch.bool, device="cuda")
        self.masks = masks

    def snap(self):
        return dc.Snapshot(self.f)

    def ready(self, mode, first, n, start, cap, ready_cap, ticket=None, what=""):
        """one ready call (ticket: 'begin' returns (ticket, want) for a later end) against the reference"""
        before = self.snap()
        want = self.f.expected_ready(before.ctl, first, n, start, cap, ready_cap, mode)
        fn = {"drain": self.bus.drain_ready, "take": self.bus.take_ready}[mode]
        if ticket == "begin":
            t = (self.bus.take_ready_begin if mode == "take" else self.bus.drain_ready_begin)(first, n, start, cap, ready_cap)
            self.f.took(want, mode)
            return t, want
        got = fn(first, n, start, cap, ready_cap)
        dc.assert_ready_equal(got, want, f"{mode} {what}")
        self.f.took(want, mode)
        self.unchanged(before, want, mode)
        return want

    def unchanged(self, before, want, mode):
        heads = (want["loc"], want["tail"]) if mode == "drain" else None
        dc.assert_unchanged(before, self.snap(), BASE, heads)

    def probe(self, mode, first, n, start):
        """ready positions and cumulative records of a walk, nothing taken"""
        w = self.f.expected_ready(self.snap().ctl, first, n, start, 1 << 40, 1 << 40, mode)
        return w["rp"].cpu().numpy(), w["csum"].cpu().numpy()

    def start_with_ready_at(self, mode, first, n, P, rng):
        """a start_sub whose walk has ready mailboxes at positions P - 1 and P: (start, ready before P)"""
        ready = self.f.cursor(self.snap().ctl, torch.arange(first - BASE, first - BASE + n, device="cuda"), mode)
        cnt = (ready[0] - ready[2]).cpu().numpy()
        ok = np.flatnonzero((cnt > 0) & (np.roll(cnt, P) > 0) & (np.roll(cnt, 1) > 0))
        assert len(ok), f"{mode}: no ready mailboxes at walk positions 0 and {P} of [{first}, {first + n})"
        t = int(ok[rng.integers(len(ok))])
        start = first + (t - P) % n
        rp, _ = self.probe(mode, first, n, start)
        assert P in rp
        return start, int((rp < P).sum())


def _ready_cells(c, mode, rng):
    """the synchronous calls: cuts by ready_cap at walk positions 1, 1023, 1024, 1025, in a middle tile and in the partial
    last tile, over the whole range and a sub-range (cap at exactly the records taken, so both limits cut there); a cut by
    ready_cap alone in a later tile; cuts by cap at the cumulative total and one below; no cut, wrapping"""
    _vary_cursors(c, rng)
    _assert_every_offset(c, mode)
    whole, sub = (BASE, N), (BASE + 1000 + 7, 700_001)
    # ready_cap alone: cap holds every record of the range
    P = 3 * dc.TILE + 7
    start, k = c.start_with_ready_at(mode, BASE, N, P, rng)
    everything = max(R, int(c.probe(mode, BASE, N, start)[1][-1]))
    want = c.ready(mode, BASE, N, start, everything, k, what=f"ready_cap cut at {P}")
    assert want["cut"] == P and len(want["ready"]) == k and want["total"] < everything
    for first, n in (whole, sub):
        last_tile = (n - 1) // dc.TILE
        for P in (1, 1023, 1024, 1025, (n // 2 // dc.TILE) * dc.TILE + 517, last_tile * dc.TILE + 100):
            if P > n // 2:                   # the cuts before took up to half the walk: fill again
                _vary_cursors(c, rng)
            start, k = c.start_with_ready_at(mode, first, n, P, rng)
            _, csum = c.probe(mode, first, n, start)
            want = c.ready(mode, first, n, start, max(R, int(csum[k - 1])), k, what=f"cut at {P}")
            assert want["cut"] == P and len(want["ready"]) == k and want["cut"] // dc.TILE == P // dc.TILE
            if P > n - dc.TILE:
                assert P // dc.TILE == last_tile and n % dc.TILE
            loc = want["loc"].cpu().numpy()
            if start - first + P >= n:                                      # the walk went through the end of the range
                assert (loc < start - BASE).any() and (loc >= start - BASE).any()
        # cap at exactly the cumulative total (fits) and one below it, in the second tile
        _vary_cursors(c, rng)
        for below in (0, 1):
            start, k = c.start_with_ready_at(mode, first, n, 1500, rng)
            rp, csum = c.probe(mode, first, n, start)
            cap, cut = int(csum[k]) - below, rp[k + 1 - below]
            want = c.ready(mode, first, n, start, max(cap, R), 1 << 30, what=f"cap {cap}")
            assert cap < R or want["cut"] == cut
            assert not below or want["cut"] == 1500
    # no cut at all, from the middle of a sub-range: the walk wraps
    _vary_cursors(c, rng)
    first, n = sub
    start = first + n - 5000
    want = c.ready(mode, first, n, start, max(R, int(c.probe(mode, first, n, start)[1][-1])), n, what="no cut")
    loc = want["loc"].cpu().numpy()
    assert want["cut"] is None and want["next_sub"] == start
    assert (loc < start - BASE).any() and (loc >= start - BASE).any()


def _ticket_cells(c, mode, rng):
    """up to 8 tickets outstanding, publishes and flushes queued between begins: each ends equal to the reference at its
    begin's place in stream order.  The cells reach every chunk geometry of the ticket gather."""
    tickets = []
    spare = np.flatnonzero(c.masks == 1 << SPARE)

    def between():
        for _ in range(2):
            assert c.bus.publish(SPARE, 7) == nat.OK
        assert c.bus.flush() == nat.OK

    first, n = BASE, N
    # a cut by cap whose total is 1 or 15 mod 16, in the second tile
    start = first + int(rng.integers(n))
    rp, csum = c.probe(mode, first, n, start)
    k = next(i for i in range(int(np.searchsorted(rp, 1100)), len(csum)) if csum[i] % 16 in (1, 15) and csum[i] >= R)
    tickets.append((c.ready(mode, first, n, start, int(csum[k]), 1 << 30, ticket="begin"), int(csum[k]), "total mod 16",
                    rp[k + 1]))
    between()
    for P in (1, 1024, 1025, (n // 2 // dc.TILE) * dc.TILE + 3, ((n - 1) // dc.TILE) * dc.TILE + 5):
        start, kk = c.start_with_ready_at(mode, first, n, P, rng)
        csum = c.probe(mode, first, n, start)[1]
        cap = max(R, int(csum[kk - 1]))
        tickets.append((c.ready(mode, first, n, start, cap, kk, ticket="begin"), cap, f"cut at {P}", P))
        between()
    # a sub-range whose first id is no multiple of 1,024, cut nowhere and wrapping; then the whole range, cut nowhere
    sub = (BASE + 77_777, 500_003)
    for first, n, start in ((sub[0], sub[1], sub[0] + 400_000), (BASE, N, BASE + N - 3)):
        _vary_cursors(c, rng)                # drains, fills, takes and acks between begin and end
        csum = c.probe(mode, first, n, start)[1]
        cap = max(R, int(csum[-1]))
        tickets.append((c.ready(mode, first, n, start, cap, n, ticket="begin"), cap, f"no cut {n}", None))
        between()
    assert len(tickets) == 8
    for i in rng.permutation(len(tickets)):                                 # ended in any order
        (t, want), cap, what, cut = tickets[i]
        before = c.snap()
        got = c.bus.drain_ready_end(t, cap, int(1 << 30))
        dc.assert_unchanged(before, c.snap(), BASE)                         # an end only copies out what its begin took
        dc.assert_ready_equal(got, want, f"ticket {what}")
        assert want["cut"] == cut, what
        if what == "total mod 16":
            assert want["total"] % 16 in (1, 15)
        if what == f"no cut {N}":                                         # the rest of the fleet
            g = dc.chunk_geometry(want["ready"])
            assert g["inside"] and g["at_start"] and g["at_end"] and g["long_run"] and g["ones_chunk"], (what, g)
    assert len(spare)


def _vary_cursors(c, rng):
    """throughput: another fill (overwrites, runs that wrap) and partial drains of a sample; lossless: consume_all (checked),
    a fill, partial drains of a sample, a take of a quarter of the fleet and acks of arbitrary counts over about 10^5 mailboxes (checked)"""
    bus = c.bus

    def drain_sample():
        """part of the run of 2,000 subscribed mailboxes holding two records or more: their cursors move by 1 .. run - 1"""
        tail, _, cur = c.f.cursor(c.snap().ctl, torch.arange(N, device="cuda"), "drain")
        backlog = (tail - cur).cpu().numpy()
        for g in rng.choice(np.flatnonzero(c.subscribed.cpu().numpy() & (backlog >= 2)), 2000, replace=False):
            bus.drain(BASE + int(g), int(rng.integers(1, backlog[g])))

    if not c.lossless:
        _fill(bus, rng)
        drain_sample()
        return
    before = c.snap()
    bus.consume_all()
    dc.assert_unchanged(before, c.snap(), BASE, (torch.arange(N, device="cuda"), before.ctl[:, 0]))
    _fill(bus, rng, lossless=True)
    drain_sample()                           # heads at every offset, also for the mailboxes the quarter does not take
    rp, csum = c.probe("take", BASE, N, BASE)
    k = int(np.searchsorted(rp, N // 4))   # a quarter: cuts at every position still find untaken mailboxes
    want = c.ready("take", BASE, N, BASE, max(R, int(csum[k])), 1 << 30, what="a quarter")
    _acks(c, rng, want)


def _assert_every_offset(c, mode):
    """the ready mailboxes' cursors fall on every ring offset, and some of their runs wrap the ring"""
    tail, _, cur = c.f.cursor(c.snap().ctl, torch.arange(N, device="cuda"), mode)
    ready = tail > cur
    off = cur[ready] % R
    assert len(torch.unique(off)) == R, f"{mode}: cursors on {len(torch.unique(off))} of {R} ring offsets"
    assert bool((off + (tail - cur)[ready] > R).any()), f"{mode}: no run wraps the ring"


def _acks(c, rng, taken):
    """ack_many with about 10^5 elements: duplicates, over-acks, unknown and released ids, zeros, unsubscribed mailboxes"""
    rdy = taken["ready"]
    pick = rng.choice(len(rdy), min(len(rdy), 80_000), replace=False)
    ids = rdy["sub_id"][pick].astype(np.int64)
    counts = rng.integers(0, rdy["count"][pick].astype(np.int64) + 3)       # some beyond what is held
    dup = rng.choice(len(ids), 15_000)
    unknown = np.array([BASE - 1, BASE + N, BASE + N + 5, 0], dtype=np.int64)
    released = np.flatnonzero(~c.known.cpu().numpy())[:50] + BASE
    unsub = np.flatnonzero(~c.subscribed.cpu().numpy())[:2000] + BASE
    ids = np.concatenate([ids, ids[dup], unknown, released, unsub])
    counts = np.concatenate([counts, rng.integers(0, 4, len(dup)), [1, 1, 0, 1], np.ones(len(released), np.int64),
                             rng.integers(0, 3, len(unsub))])
    order = rng.permutation(len(ids))
    ids, counts = ids[order].astype(np.uint32), counts[order].astype(np.uint32)
    before = c.snap()
    want = c.f.expected_acks(before.ctl, ids, counts, c.known)
    st = c.bus.ack_many(ids, counts)
    bad = np.flatnonzero(st != want["status"])
    assert not len(bad), f"ack element {bad[0]} (mailbox {ids[bad[0]]}, count {counts[bad[0]]}): status {st[bad[0]]}, " \
                         f"expected {want['status'][bad[0]]}"
    assert (st == nat.OK).sum() > 50_000 and (st == nat.EINVAL).any() and (st == nat.ENOENT).sum() >= 4
    dc.assert_unchanged(before, c.snap(), BASE, want["heads"])


def _membership(c, rng):
    """unsubscribe some mailboxes that hold records, and release a part of them"""
    gone = np.sort(rng.choice(N, 3000, replace=False))
    assert (c.bus.unsubscribe_many(gone + BASE) == nat.OK).all()
    c.subscribed[torch.from_numpy(gone).cuda()] = False
    rel = gone[::3]
    assert (c.bus.release_many(rel + BASE) == nat.OK).all()
    c.known[torch.from_numpy(rel).cuda()] = False


def _lagging_cells(c, rng):
    """min_backlog in {0, 1, 17, R}, caps that cut at walk positions 1, 1023, 1024 and 1025 and paging to completion from a
    start in the middle: every lagging mailbox once, and the summary exact on every page"""
    first, n = BASE, N
    for min_backlog in (0, 1, 17, R):
        start = first + int(rng.integers(n))
        before = c.snap()
        seen, s, left = [], start, None
        for cap in (1, 1023, 1024, 1025, 300_000, 300_000, 300_000, 300_000, 300_000):
            want = c.f.expected_lagging(before.ctl, c.subscribed, first, n, s, min_backlog, cap)
            out, nxt, summary = c.bus.lagging(first, n, s, min_backlog, cap)
            if out.tobytes() != want["out"].tobytes():
                k = min(len(out), len(want["out"]))
                bad = np.flatnonzero(out[:k] != want["out"][:k])
                i = int(bad[0]) if len(bad) else k
                raise AssertionError(f"lagging (min_backlog {min_backlog}, cap {cap}) entry {i}: got "
                                     f"{out[i] if i < len(out) else None}, expected {want['out'][i] if i < len(want['out']) else None}")
            assert nxt == want["next_sub"] and summary == want["summary"], (min_backlog, cap)
            left = summary["lagging"] if left is None else left
            seen.append(out["sub_id"][:left].astype(np.int64))         # a page past the last lagging mailbox wraps
            left -= len(seen[-1])
            s = nxt
            if left == 0:
                break
        seen = np.concatenate(seen)
        assert len(seen) == len(np.unique(seen)) == want["summary"]["lagging"]
        assert want["summary"]["lagging"] > 2000
        dc.assert_unchanged(before, c.snap(), BASE)


def _fold_cells(c):
    before = c.snap()
    for first, n in ((BASE, N), (BASE + 1, 1023), (BASE + 1000, 654_321), (BASE + N - 333, 333)):
        want = c.f.expected_fold(before.ctl, first, n)
        assert c.bus.digest_fold(first, n) == want, (first, n)
        assert c.bus.digest_fold_end(c.bus.digest_fold_begin(first, n)) == want, (first, n)
    dc.assert_unchanged(before, c.snap(), BASE)


def _drain_many_cells(c):
    """offsets depend on atomic order: each nonzero count is exactly the mailbox's run at its offset and empties it, runs are
    disjoint and inside cap, and a mailbox left out is untouched; with cap = every record, nothing is left out"""
    first, n = BASE + 3, N - 3
    for frac in (2, 1):
        before = c.snap()
        want = c.f.expected_ready(before.ctl, first, n, first, 1 << 40, 1 << 40, "drain")
        cap = max(R, want["total"] // frac)
        out, offs, cnts = np.zeros(cap, dtype=EVENT_DTYPE), np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint32)
        total = C.c_size_t()
        nat.check(c.bus._lib.cpbus_drain_many(c.bus._h, first, n, out.ctypes.data, cap, offs.ctypes.data, cnts.ctypes.data,
                                              C.byref(total)), "cpbus_drain_many")
        assert total.value == int(cnts.sum()) <= cap
        wc = np.zeros(n, dtype=np.int64)
        wc[want["ready"]["sub_id"].astype(np.int64) - first] = want["ready"]["count"]
        got = np.flatnonzero(cnts)
        assert (cnts[got] == wc[got]).all(), "drain_many count differs from the run"
        o = offs[got].astype(np.int64)
        order = np.argsort(o)
        ends = o[order] + cnts[got][order]
        assert (ends <= cap).all() and (o[order][1:] >= ends[:-1]).all()
        recs = out.view(np.int64).reshape(-1, 4)
        wo, wo_off = want["out"].cpu().numpy(), want["ready"]["offset"].astype(np.int64)
        pos = np.zeros(n, dtype=np.int64)
        pos[want["ready"]["sub_id"].astype(np.int64) - first] = wo_off
        # every record of every returned run: record j of mailbox i's run at offs[i] + j against the reference's
        e = np.repeat(got, cnts[got].astype(np.int64))
        j = np.arange(len(e)) - np.repeat(np.cumsum(cnts[got].astype(np.int64)) - cnts[got], cnts[got].astype(np.int64))
        bad = np.flatnonzero((recs[offs[e].astype(np.int64) + j] != wo[pos[e] + j]).any(1))
        assert not len(bad), f"drain_many record {int(j[bad[0]])} of the run of mailbox {first + int(e[bad[0]])} differs"
        if frac == 1:
            assert (cnts == wc).all()
        loc = torch.from_numpy(got + first - BASE).cuda()
        dc.assert_unchanged(before, c.snap(), BASE, (loc, before.ctl[loc, 0]))


@pytest.fixture(params=[False, True], ids=["throughput", "lossless"])
def fleet(request):
    lossless = request.param
    rng = np.random.default_rng(0xC0A5 + lossless)
    masks = _masks(rng, lossless)
    with Bus(N, ring_cap=R, batch_cap=B, lossless=lossless, sub_id_base=BASE,
             stream=torch.cuda.current_stream().cuda_stream) as bus:
        assert bus.subscribe_many(masks) == BASE
        _fill(bus, rng, lossless=lossless)
        with rc.fleet_views(bus.device_ptrs(), N, R) as views:
            c = Cell(bus, views, lossless, masks)
            _membership(c, rng)
            yield c, rng


def test_consumer_calls_equal_the_reference(fleet):
    c, rng = fleet
    mode = "take" if c.lossless else "drain"
    _ready_cells(c, mode, rng)
    if c.lossless:                      # a lossless drain reads from head: held records included
        _ready_cells(c, "drain", rng)
    _vary_cursors(c, rng)
    _ticket_cells(c, mode, rng)
    _vary_cursors(c, rng)
    _lagging_cells(c, rng)
    _fold_cells(c)
    _drain_many_cells(c)
    before = c.snap()
    c.bus.consume_all()
    dc.assert_unchanged(before, c.snap(), BASE, (torch.arange(N, device="cuda"), before.ctl[:, 0]))


@pytest.mark.parametrize("K", [0, 1])
def test_blockers_equal_the_reference(K):
    """lossless, one staged record, and with K = 1 periodic timers armed after the fill on a third of the fleet, due by
    the clock: the mailboxes whose share exceeds their room, ascending"""
    rng = np.random.default_rng(0xB10C + K)
    masks = _masks(rng, True)
    with Bus(N, ring_cap=R, batch_cap=B, lossless=True, sub_id_base=BASE, timers_per_sub=K,
             stream=torch.cuda.current_stream().cuda_stream) as bus:
        bus.subscribe_many(masks)
        _fill(bus, rng, lossless=True)
        with rc.fleet_views(bus.device_ptrs(), N, R) as views:
            c = Cell(bus, views, True, masks)
            _membership(c, rng)
            for g in rng.choice(np.flatnonzero(c.subscribed.cpu().numpy()), 5000, replace=False):
                bus.drain(BASE + int(g), int(rng.integers(1, R + 1)))
            timers = ()
            now = bus.stats()["now_ns"]
            if K:
                loc = np.flatnonzero((np.arange(N) % 3 == 0) & c.subscribed.cpu().numpy())
                period = 1_000 + (loc % 5) * 100
                _, st = bus.timer_add_list(loc + BASE, period, np.full(len(loc), 9, np.uint32))
                assert (st == nat.OK).all()
                due = torch.full((N,), 1 << 62, dtype=torch.int64, device="cuda")
                per = torch.ones(N, dtype=torch.int64, device="cuda")
                armed = torch.zeros(N, dtype=torch.bool, device="cuda")
                li = torch.from_numpy(loc).cuda()
                due[li], per[li], armed[li] = now + torch.from_numpy(period).cuda(), torch.from_numpy(period).cuda(), True
                timers = ((due, per, armed),)
                now += 10_000
                assert bus.advance(now) == nat.OK
            assert bus.publish(1, 3) == nat.OK                                # staged: the next unit's record
            takes = torch.from_numpy((masks & 0b10) != 0).cuda()
            before = c.snap()
            want = c.f.expected_blockers(before.ctl, c.subscribed, takes, now, timers)
            got = bus.blockers()
            assert got.tobytes() == want.tobytes(), (len(got), len(want), got[:5], want[:5])
            assert len(want) > 1000
            dc.assert_unchanged(before, c.snap(), BASE)


def test_sparse_list_scan_cut_in_its_second_tile():
    """CPBUS_CFG_SPARSE_DRAINS at 5 * 2^20 mailboxes: the list scan of 1,200 candidates (the list is used up to N / 4,096 =
    1,280) cut in its second tile by ready_cap and by cap, and not cut, from a start inside the list, against the
    reference; records reach the candidates through sparse record launches after consume_all, so the index knows them"""
    n_big, M = 5 << 20, 1200
    rng = np.random.default_rng(0x5CA1)
    cand = np.sort(rng.choice(n_big - 1, M, replace=False))
    masks = np.full(n_big, 1 << 5, dtype=np.uint32)
    masks[cand] = (1 << (1 + rng.integers(0, 3, M))).astype(np.uint32)
    with Bus(n_big, ring_cap=R, batch_cap=32, sparse_drains=True, sparse_records=True,
             stream=torch.cuda.current_stream().cuda_stream) as bus:
        bus.subscribe_many(masks)
        with rc.fleet_views(bus.device_ptrs(), n_big, R) as views:
            f = dc.Fleet(views[0], views[1], 0, False, sync=bus.sync)
            start = int(cand[300])
            empty = (int(cand[-1]) + 1, n_big - int(cand[-1]) - 1)
            for ready_cap, cap_at, taken in ((1100, None, 1100), (1 << 30, 1030, 1030), (1 << 30, None, M)):
                bus.consume_all()
                for code, k in ((1, R + 6), (2, 1), (3, 17)):        # code 1: overwritten, its cursor is tail - R
                    for i in range(0, k, 16):
                        for _ in range(min(16, k - i)):
                            assert bus.publish(code, 7) == nat.OK
                        assert bus.flush() == nat.OK
                # the index knows where records are, so the drain scans the candidate list: a range without candidates
                # launches nothing
                l0 = bus.stats()["kernel_launches"]
                assert len(bus.drain_ready(empty[0], empty[1], empty[0], 4 * R, 16)[1]) == 0
                assert bus.stats()["kernel_launches"] == l0
                before = dc.Snapshot(f)
                probe = f.expected_ready(before.ctl, 0, n_big, start, 1 << 40, 1 << 40)
                csum = probe["csum"].cpu().numpy()
                assert probe["n_ready_all"] == M
                cap = int(csum[cap_at] - 1) if cap_at else int(csum[-1])
                want = f.expected_ready(before.ctl, 0, n_big, start, cap, ready_cap)
                l0 = bus.stats()["kernel_launches"]
                got = bus.drain_ready(0, n_big, start, cap, ready_cap)
                assert bus.stats()["kernel_launches"] - l0 == 2
                dc.assert_ready_equal(got, want, f"list scan ready_cap {ready_cap} cap {cap}")
                assert len(want["ready"]) == taken and (want["cut"] is None) == (taken == M)
                dc.assert_unchanged(before, dc.Snapshot(f), 0, (want["loc"], want["tail"]))
