"""The consumer-side reference (`tests/drain_check.py`) against the C oracle, on the CPU.  The fleet is the one of
`tests/test_ring_reference.py` (code masks, exact {code, source} cases, unicast, two timer slots, rings that wrap); its
(ring, ctl) image is built from `ring_check.FleetModel.expected` with heads and take cursors the test chooses, and every
mailbox's run, lost count, backlog, ack outcome and fold term is compared with a per-mailbox oracle that consumed the
same records.  Throughput mode also has overwritten mailboxes whose head lies behind tail - R."""
import numpy as np
import pytest
import torch

import drain_check as dc
import lag_oracle as lo
import oracle_binding as ob
from containerpilot_b200 import _native as nat
from test_oracle_semantics import py_record_hash
from test_ring_reference import _fleet

BIG = 1 << 20


def _oracle(model, i):
    """mailbox i alone in an oracle with unbounded mailboxes (keep_window 0: every record stays readable)"""
    gid = model.base + i
    orc = ob.Oracle(1, timers_per_sub=len(model.timers), keep_window=0, sub_id_base=gid)
    rows = model.pair_shapes[model.shape_of[i]]
    orc.subscribe(int(model.masks[i]), [(int(c), int(s)) for c, s in rows if c != 0xFFFFFFFF] or None)
    for tm in model.timers:
        orc.timer_add(gid, int(tm["period"][i]), int(tm["source"][i]), bool(tm["oneshot"]))
    for a, b, w in model.batches:
        assert orc.publish_records(model.records[a:b], int(w)) == 0
    return orc


class Image:
    """(ring, ctl) of the model with chosen heads; per mailbox, the oracle's run from its cursor and its lost count"""

    def __init__(self, seed, lossless, base=0):
        self.model = m = _fleet(seed, base=base)
        count, image, _ = m.expected(0, m.n, "cpu")
        rng = np.random.default_rng(seed + 100 * lossless)
        cnt = count.numpy()
        lo_head = np.maximum(0, cnt - m.R) if lossless else np.zeros_like(cnt)   # lossless: at most R undrained
        head = rng.integers(lo_head, cnt + 1)
        head[::5] = cnt[::5]                                                     # drained to the end
        head[1::9] = lo_head[1::9]                                               # nothing drained (overwritten if > R)
        self.subscribed = torch.from_numpy(rng.random(m.n) < 0.9)
        ctl = torch.zeros(m.n, 4, dtype=torch.int64)
        ctl[:, 0], ctl[:, 1] = count, torch.from_numpy(head)
        self.orcs = [_oracle(m, i) for i in range(m.n)]
        ctl[:, 2] = torch.tensor([self.orcs[i].digest(m.base + i) for i in range(m.n)], dtype=torch.uint64).view(torch.int64)
        ctl[:, 3] = torch.from_numpy(m.masks.astype(np.int64)) | torch.where(self.subscribed, dc.ACTIVE_BIT, 0)
        self.fleet = dc.Fleet(image.view(m.n, m.R, 4), ctl, m.base, lossless)
        self.head = head
        for i, orc in enumerate(self.orcs):
            assert orc.count(m.base + i) == cnt[i]
            if head[i]:
                assert len(orc.consume(m.base + i, int(head[i]))) == head[i]

    def run(self, i, extra=0):
        """the oracle's records of mailbox i from its cursor (throughput mode: the last R of them), lost; consumes them.
        extra: records skipped first (a take cursor ahead of head)"""
        gid = self.model.base + i
        if extra:
            self.orcs[i].consume(gid, extra)
        r = self.orcs[i].consume(gid, BIG)
        lost = 0
        if not self.fleet.lossless and len(r) > self.model.R:
            lost, r = len(r) - self.model.R, r[-self.model.R:]
        return r, lost


@pytest.mark.parametrize("lossless", [False, True])
@pytest.mark.parametrize("seed", [1, 2])
def test_whole_range_drain_equals_the_oracle_on_every_mailbox(seed, lossless):
    im = Image(seed, lossless)
    f, m = im.fleet, im.model
    want = f.expected_ready(f.ctl, 0, m.n, 37, BIG, BIG)
    assert want["cut"] is None and want["next_sub"] == 37
    rdy, out = want["ready"], want["out"].numpy()
    entry = {int(e["sub_id"]): k for k, e in enumerate(rdy)}
    assert [int(g) for g in rdy["sub_id"]] == sorted(entry, key=lambda g: (g - 37) % m.n)   # walk order from 37
    overwritten = 0
    for i in range(m.n):
        r, lost = im.run(i)
        k = entry.get(i)
        if k is None:
            assert len(r) == 0, f"mailbox {i}: the oracle holds {len(r)} records, the reference none"
            continue
        e = rdy[k]
        assert int(e["count"]) == len(r) and int(e["lost"]) == lost and int(e["pad"]) == 0, f"mailbox {i}"
        run = out[int(e["offset"]):int(e["offset"]) + int(e["count"])]
        assert run.tobytes() == r.tobytes(), f"mailbox {i}: run differs from the oracle"
        overwritten += lost > 0
    assert (overwritten > 0) == (not lossless)
    assert (rdy["count"] == m.R).any() and (rdy["count"] < 16).any()


@pytest.mark.parametrize("lossless", [False, True])
def test_cuts_and_next_sub_follow_the_oracle_runs(lossless):
    """cuts by ready_cap, by cap at exactly the cumulative total and one below it, from several starts of a sub-range of a
    shard at a non-zero base: the taken prefix is the oracle's runs in walk order while they fit"""
    base = 70_000
    im = Image(3, lossless, base=base)
    f, m = im.fleet, im.model
    runs = [len(im.run(i)[0]) for i in range(m.n)]
    first, n = base + 7, m.n - 20
    for start in (first, first + 1, first + n - 1, first + 61):
        order = [(start - base + p - 7) % n + 7 for p in range(n)]
        ready = [i for i in order if runs[i]]
        csum = np.cumsum([runs[i] for i in ready])
        for k in (1, 2, len(ready) // 2, len(ready) - 1):
            for cap, rcap, taken in ((BIG, k, k), (max(m.R, int(csum[k - 1])), BIG, None), (int(csum[k - 1]) - 1, BIG, None)):
                if cap < m.R:
                    continue
                want = f.expected_ready(f.ctl, first, n, start, cap, rcap)
                t = taken if taken is not None else int((csum <= cap).sum())
                assert len(want["ready"]) == t and want["total"] == (int(csum[t - 1]) if t else 0)
                assert [int(g) - base for g in want["ready"]["sub_id"]] == ready[:t]
                assert want["next_sub"] == base + ready[t] and want["cut"] == order.index(ready[t])


def test_take_cursors_and_acks_follow_the_oracle():
    """take from T = max(T, head) with T ahead of head on some mailboxes; then acks of arbitrary counts, duplicates,
    over-acks, zeros and unknown ids, checked against the oracle consuming what each ack releases"""
    im = Image(4, True)
    f, m = im.fleet, im.model
    rng = np.random.default_rng(9)
    tail, head = f.ctl[:, 0].numpy(), f.ctl[:, 1].numpy()
    T = np.where(rng.random(m.n) < 0.4, rng.integers(head, tail + 1), rng.integers(0, head + 1))
    f.taken = torch.from_numpy(T)
    want = f.expected_ready(f.ctl, 0, m.n, 0, BIG, BIG, mode="take")
    rdy, out = want["ready"], want["out"].numpy()
    entry = {int(e["sub_id"]): k for k, e in enumerate(rdy)}
    for i in range(m.n):
        skip = max(0, int(T[i]) - int(head[i]))
        o = _oracle(m, i)
        o.consume(i, int(head[i]) + skip)
        r = o.consume(i, BIG)
        k = entry.get(i)
        assert (k is None) == (len(r) == 0), f"mailbox {i}"
        if k is not None:
            e = rdy[k]
            assert int(e["lost"]) == 0 and int(e["count"]) == len(r)
            assert out[int(e["offset"]):int(e["offset"]) + len(r)].tobytes() == r.tobytes(), f"mailbox {i}"
    f.took(want, "take")
    took = np.isin(np.arange(m.n), rdy["sub_id"].astype(np.int64))
    assert (f.taken.numpy() == np.where(took, tail, T)).all()
    # acks: held = T - head after the take
    known = torch.ones(m.n, dtype=torch.bool)
    known[5] = False                                                          # released
    ids = np.concatenate([rng.integers(0, m.n, 400), [m.n, m.n + 3, 5, 5], rng.integers(0, m.n, 100)])
    counts = np.concatenate([rng.integers(0, 8, 400), [1, 0, 1, 0], rng.integers(30, 80, 100)])
    acks = f.expected_acks(f.ctl, ids, counts, known)
    st = acks["status"]
    assert (st == nat.OK).any() and (st == nat.EINVAL).any() and (st[400:404] == [nat.ENOENT, nat.ENOENT, nat.ENOENT, nat.ENOENT]).all()
    hold = {i: max(int(f.taken[i]), int(head[i])) - int(head[i]) for i in range(m.n)}
    for j, (g, c) in enumerate(zip(ids, counts)):
        g, c = int(g), int(c)
        if g >= m.n or g == 5:
            assert st[j] == nat.ENOENT
            continue
        ok = c <= hold[g]
        assert st[j] == (nat.OK if ok else nat.EINVAL), f"element {j} (mailbox {g}, count {c})"
        if ok:
            hold[g] -= c
            assert len(im.orcs[g].consume(g, c)) == c
    for l, h in acks["heads"].items():   # the oracle's cursor after consuming head + what the acks released
        assert h == im.orcs[l].count(l) - lo.backlog(im.orcs[l], l), f"mailbox {l}"
    assert acks["applied"] == int((st == nat.OK).sum())


@pytest.mark.parametrize("lossless", [False, True])
def test_lagging_equals_the_oracle_backlog(lossless):
    im = Image(5, lossless)
    f, m = im.fleet, im.model
    backlog, lost = [], []
    for i in range(m.n):
        if lossless:   # lossless: the oracle's own backlog query
            backlog.append(lo.backlog(im.orcs[i], m.base + i)); lost.append(0)
        else:
            r, l = im.run(i)
            backlog.append(len(r)); lost.append(l)
    backlog, lost = np.array(backlog), np.array(lost)
    act = im.subscribed.numpy()
    for min_backlog, cap, start in ((0, BIG, 0), (1, BIG, 50), (17, 5, 100), (m.R, 2, 0), (1, 0, 3)):
        want = f.expected_lagging(f.ctl, im.subscribed, 0, m.n, start, min_backlog, cap)
        order = [(start + p) % m.n for p in range(m.n)]
        lag = [i for i in order if act[i] and backlog[i] >= min_backlog]
        assert [int(g) for g in want["out"]["sub_id"]] == lag[:cap]
        assert [int(b) for b in want["out"]["backlog"]] == [int(backlog[i]) for i in lag[:cap]]
        assert [int(x) for x in want["out"]["lost"]] == [int(lost[i]) for i in lag[:cap]]
        assert want["next_sub"] == (start if len(lag) <= cap else lag[cap])
        s = want["summary"]
        b = backlog[act]
        hist = [int((b == 0).sum())] + [int(((b >= 1 << (k - 1)) & (b < 1 << k)).sum()) for k in range(1, 33)]
        assert s == {"active": int(act.sum()), "lagging": int((act & (backlog >= min_backlog)).sum()),
                     "backlog_total": int(b.sum()), "backlog_max": int(b.max()), "lost_total": int(lost[act].sum()),
                     "hist": hist}
    assert (backlog > m.R // 2).any() and (backlog == 0).any() and (lost > 0).any() != lossless


def test_fold_equals_the_oracle_digests():
    im = Image(6, False, base=4242)
    f, m = im.fleet, im.model
    for first, n in ((m.base, m.n), (m.base + 3, 100), (m.base + m.n - 1, 1)):
        c = d = x = 0
        for g in range(first, first + n):
            orc = im.orcs[g - m.base]
            cnt, dig = int(orc.count(g)), int(orc.digest(g))
            c, d = (c + cnt) % (1 << 64), (d + dig) % (1 << 64)
            x ^= py_record_hash(dig, cnt, g, 0, 0, 0)
        assert f.expected_fold(f.ctl, first, n) == (c, d, x, n)


def test_blockers_share_and_room():
    """a full mailbox blocks on a record it takes, a mailbox with room r blocks on more than r ticks; unsubscribed never"""
    im = Image(7, True)
    f, m = im.fleet, im.model
    full = torch.arange(m.n) % 4 == 0                                       # a quarter with nothing drained
    f.ctl[:, 1] = torch.where(full, (f.ctl[:, 0] - m.R).clamp(min=0), f.ctl[:, 1])
    room = (m.R - (f.ctl[:, 0] - f.ctl[:, 1])).numpy()
    takes = torch.from_numpy(np.arange(m.n) % 3 == 0)
    due = torch.full((m.n,), 1_000, dtype=torch.int64)
    period = torch.from_numpy(100 + np.arange(m.n) % 7 * 50).long()
    armed = torch.from_numpy(np.arange(m.n) % 2 == 0)
    for clock, timers in ((0, ()), (5_000, ((due, period, armed),))):
        got = f.expected_blockers(f.ctl, im.subscribed, takes, clock, timers)
        ticks = np.where(armed.numpy() & (clock >= 1_000) & bool(timers), (clock - 1_000) // period.numpy() + 1, 0)
        share = ticks + takes.numpy()
        want = [i for i in range(m.n) if im.subscribed[i] and share[i] > room[i]]
        assert [int(g) for g in got] == want
        assert len(want) > 0


def test_a_flipped_record_word_is_named_by_mailbox():
    """the comparison names the entry, mailbox and record where a drained run differs from the reference"""
    im = Image(8, False)
    f, m = im.fleet, im.model
    want = f.expected_ready(f.ctl, 0, m.n, 0, BIG, BIG)
    rec = want["out"].numpy().copy().view(ob.EVENT_DTYPE).reshape(-1)
    got = (rec, want["ready"].copy(), want["next_sub"])
    dc.assert_ready_equal(got, want)
    e = want["ready"][len(want["ready"]) // 2]
    f.ring[int(e["sub_id"]) - m.base, (int(f.ctl[int(e["sub_id"]) - m.base, 0]) - 1) & (m.R - 1), 2] ^= 1 << 40
    again = f.expected_ready(f.ctl, 0, m.n, 0, BIG, BIG)
    r = int(e["offset"]) + int(e["count"]) - 1
    with pytest.raises(AssertionError, match=f"record {r} \\(entry {len(want['ready']) // 2}, mailbox {int(e['sub_id'])},"):
        dc.assert_ready_equal(got, again)
    before = dc.Snapshot(f)
    f.ring[3, 0, 1] += 1
    with pytest.raises(AssertionError, match="ring memory of mailboxes 0 .."):
        dc.assert_unchanged(before, dc.Snapshot(f), m.base)
    f.ctl[9, 2] ^= 1
    with pytest.raises(AssertionError, match="mailbox 9 control word 2 changed"):
        dc.assert_unchanged(before, dc.Snapshot(f), m.base)
