"""Periodic timers that drop missed ticks (CPBUS_CFG_DROP_MISSED_TICKS) without a GPU: the flag and the due-index op, a
plain-C99 caller, the host due index's catch-up (cpbus_due_trace with CPBUS_DUE_CATCHUP) and the oracle with missed ticks
dropped, both against an independent Python model of Go 1.9 tickers on seeded traces: periods near 2^64, one-shots,
re-arms, cancels, unsubscribes, ties at exactly clock + k * period.
The bus itself needs a GPU: tests/test_gpu_drop_missed_ticks.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from containerpilot_b200 import _native as nat
from drop_oracle import DropOracle
from test_sparse_ticks_abi import trace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDLE = (1 << 64) - 1   # "never"
TIMER_EXPIRED, F_TICK = 8, 0x1


class GoTickers:
    """Go 1.9 tickers (runtime/time.go) read by NewEventTimer (events/timer.go:40-71) on a virtual clock.  A ticker armed
    at t with period p is first due at when = t + p.  At each wake-up at `now` with when <= now, it sends one tick without
    blocking into a channel of capacity 1 and moves on: late = now - when, when += p * (1 + late // p).  The tick reports
    the firing it stands for, the last one due by now, by its ordinal on the grid.  A one-shot (NewEventTimeout) sends once.
    A firing at or past 2^64 - 1 never comes."""

    def __init__(self):
        self.clock, self.t = 0, {}   # slot -> [when, period, oneshot, ordinal of `when`, source]

    def arm(self, slot, period, oneshot, source=0):
        when = self.clock + period
        self.t[slot] = [when if when < IDLE else IDLE, period, oneshot, 0, source]

    def disarm(self, slot):
        self.t.pop(slot, None)

    def wake(self, now):
        """{slot: (ordinal, due)} of the ticks sent at a wake-up at now; the clock becomes now"""
        sent, w = {}, min(now, IDLE - 1)
        for slot in sorted(self.t):
            when, p, oneshot, n, src = self.t[slot]
            if when == IDLE or when > w:
                continue
            if oneshot:
                sent[slot] = (n, when)
                del self.t[slot]
                continue
            skip = (w - when) // p
            sent[slot] = (n + skip, when + skip * p)
            nxt = when + p * (1 + skip)
            self.t[slot] = [nxt if nxt < IDLE else IDLE, p, False, n + skip + 1, src]
        self.clock = now
        return sent


def test_flag_and_op():
    assert nat.CFG_DROP_MISSED_TICKS == 0x10 and nat.DUE_CATCHUP == 6
    assert not nat.CFG_DROP_MISSED_TICKS & (nat.CFG_LOSSLESS | nat.CFG_DIGEST | nat.CFG_SPARSE_TICKS | nat.CFG_SPARSE_RECORDS)
    hdr = open(os.path.join(ROOT, "include", "cpbus.h")).read()
    assert "#define CPBUS_CFG_DROP_MISSED_TICKS 0x10u" in hdr and "CPBUS_DUE_CATCHUP = 6" in hdr
    assert nat.load().cpbus_abi_version() == 2


def test_drop_missed_declarations_from_plain_c99(tmp_path):
    exe = str(tmp_path / "drop_missed_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "drop_missed_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr


def _period(rng, clock):
    q = rng.random()
    if q < 0.7:
        return int(rng.integers(1, 5000))
    if q < 0.8:
        return IDLE - int(rng.integers(0, 1 << 20))                  # first due saturates to "never"
    if q < 0.95:
        return max(1, IDLE - clock - int(rng.integers(0, 20_000)))   # first due just short of (or at) the top
    return 1 << 63


def _tie(rng, clock, model):
    """a clock exactly on a later firing of a live periodic timer of `model`: its next due + k * period, k >= 1 (the step
    has exactly k + 1 of its firings; k = 1, the smallest step that coalesces, half of the time); None: no such timer"""
    live = [(t[0], t[1]) for _, t in sorted(model.t.items()) if not t[2] and clock < t[0] < IDLE]
    if not live:
        return None
    when, p = live[int(rng.integers(0, len(live)))]
    k = 1 if rng.random() < 0.5 else int(rng.integers(2, 6))
    return when + k * p if k * p < IDLE - when else None


def _steps(rng, clock, periods, model):
    """the next clock: mostly short steps, some across hundreds of periods, a quarter exactly on a later firing of a live
    timer (ties: a step with exactly two firings of it, or a few)"""
    if rng.random() < 0.25:
        t = _tie(rng, clock, model)
        if t is not None:
            return t
    q = rng.random()
    if q < 0.5:
        step = int(rng.integers(0, 3000))
    elif q < 0.8:
        step = int(rng.integers(0, 500)) * max(1, min(periods or [1000]))
    elif q < 0.9 and periods:
        step = int(rng.integers(1, 500)) * int(rng.choice(periods))
    else:
        step = int(rng.integers(0, 1 << 36))
    return min(IDLE, clock + step)


def due_trace_steps(seed, n_subs, K, n_steps):
    """(ops, n_slots, per step: (ordinal of its first launch, of the launch after its last, clock)) for a bus driven like cpbus_advance on a flagged bus:
    each step catches up to the new clock and then launches to it, in one to three window launches"""
    rng = np.random.default_rng(seed)
    n_slots = n_subs * K
    ops, steps, clock, launches = [], [], 0, 0
    m = GoTickers()   # the generator's view of the live timers, for steps that tie with their grids
    if seed % 3 == 0:
        clock = IDLE - int(rng.integers(1 << 40, 1 << 44))   # the top of the clock within reach
        ops.append((nat.DUE_CLOCK, 0, clock))
        m.clock = clock
    periods = []
    for _ in range(n_steps):
        for _ in range(int(rng.integers(0, 4))):
            r = rng.random()
            if r < 0.6:
                slot = int(rng.integers(0, n_slots))
                p = _period(rng, clock)
                periods.append(p)
                one = rng.random() < 0.2
                ops.append((nat.DUE_ONESHOT if one else nat.DUE_ARM, slot, p))
                m.arm(slot, p, one)
            elif r < 0.8:
                ops.append((nat.DUE_DISARM, int(rng.integers(0, n_slots)), 0))
                m.disarm(ops[-1][1])
            else:
                ops.append((nat.DUE_UNSUB, int(rng.integers(0, n_subs)), 0))
                for k in range(K):
                    m.disarm(ops[-1][1] * K + k)
        now = _steps(rng, clock, [p for p in periods if p < 1 << 20], m)
        m.wake(now)
        ops.append((nat.DUE_CATCHUP, 0, now))
        cuts = sorted(min(now, clock + int(rng.random() * (now - clock + 1))) for _ in range(int(rng.integers(0, 3))))
        first = launches
        for w in cuts + [now]:   # the window split: every launch after the catch-up fires each slot at most once
            ops.append((nat.DUE_LAUNCH, 0, w))
            launches += 1
        steps.append((first, launches, now))
        clock = now
    return ops, n_slots, steps


def run_go(ops, K):
    """the model over the same ops, one wake-up per CPBUS_DUE_CATCHUP: {launch range: {slot: (ticks, next due)}}"""
    m, out = GoTickers(), []
    for kind, slot, value in ops:
        if kind == nat.DUE_CLOCK:
            m.clock = value
        elif kind in (nat.DUE_ARM, nat.DUE_ONESHOT):
            m.arm(slot, value, kind == nat.DUE_ONESHOT)
        elif kind == nat.DUE_DISARM:
            m.disarm(slot)
        elif kind == nat.DUE_UNSUB:
            for k in range(K):
                m.disarm(slot * K + k)
        elif kind == nat.DUE_CATCHUP:
            sent = m.wake(value)
            out.append({s: (1, m.t[s][0] if s in m.t else IDLE) for s in sent})
    return out


@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("seed", range(8))
def test_due_index_catchup_matches_go_tickers(K, seed):
    ops, n_slots, steps = due_trace_steps(7000 * K + seed, 12, K, 300)
    rc, got = trace(ops, n_slots, K)
    assert rc == 0
    want = run_go(ops, K)
    assert len(want) == len(steps)
    by_step = []
    for first, end, _ in steps:
        fired = {}
        for launch, slot, ticks, nd in got:
            if first <= launch < end:
                assert slot not in fired, ("a slot fired twice in one step", slot)
                fired[slot] = (ticks, nd)
        by_step.append(fired)
    for i, (g, w) in enumerate(zip(by_step, want)):
        assert g == w, f"step {i} to {steps[i][2]}: {g} vs {w}"
    assert sum(len(w) for w in want) > 20
    assert _boundary_steps(ops, K) > 0   # steps with exactly two firings of some timer


def _boundary_steps(ops, K):
    """how many catch-ups of the trace give some periodic timer exactly two firings: now - next due == period"""
    m, n = GoTickers(), 0
    for kind, slot, value in ops:
        if kind == nat.DUE_CLOCK:
            m.clock = value
        elif kind in (nat.DUE_ARM, nat.DUE_ONESHOT):
            m.arm(slot, value, kind == nat.DUE_ONESHOT)
        elif kind == nat.DUE_DISARM:
            m.disarm(slot)
        elif kind == nat.DUE_UNSUB:
            for k in range(K):
                m.disarm(slot * K + k)
        elif kind == nat.DUE_CATCHUP:
            w = min(value, IDLE - 1)
            n += any(not t[2] and t[0] < IDLE and t[0] <= w and w - t[0] == t[1] for t in m.t.values())
            m.wake(value)
    return n


def test_two_firings_coalesce_into_one():
    """armed with period p at clock c, a step to exactly c + 2p (two firings due, the smallest step that coalesces) fires
    once, the firing at c + 2p, and next at c + 3p; a step to c + 2p - 1 (one firing due) is left alone"""
    for c, p in ((0, 10), (1000, 7), (IDLE - 40, 10), (5, (IDLE - 10) // 3)):
        ops = [(nat.DUE_CLOCK, 0, c), (nat.DUE_ARM, 0, p), (nat.DUE_CATCHUP, 0, c + 2 * p), (nat.DUE_LAUNCH, 0, c + 2 * p)]
        rc, got = trace(ops, 1, 1)
        assert rc == 0
        nxt = c + 3 * p if c + 3 * p < IDLE else IDLE
        assert got == [(0, 0, 1, nxt)], (c, p, got)
        ops = [(nat.DUE_CLOCK, 0, c), (nat.DUE_ARM, 0, p), (nat.DUE_CATCHUP, 0, c + 2 * p - 1),
               (nat.DUE_LAUNCH, 0, c + 2 * p - 1)]
        assert trace(ops, 1, 1) == (0, [(0, 0, 1, c + 2 * p)])


def test_catchup_keeps_the_phase_and_ties():
    """armed at 0 with period 10: a catch-up to 95 leaves the firing due at 90; to exactly 100, the one due at 100"""
    ops = [(nat.DUE_ARM, 0, 10), (nat.DUE_ARM, 1, 10), (nat.DUE_CATCHUP, 0, 95), (nat.DUE_LAUNCH, 0, 95),
           (nat.DUE_CATCHUP, 0, 200), (nat.DUE_LAUNCH, 0, 200), (nat.DUE_CATCHUP, 0, 205), (nat.DUE_LAUNCH, 0, 215)]
    rc, got = trace(ops, 2, 1)
    assert rc == 0
    assert got == [(0, 0, 1, 100), (0, 1, 1, 100), (1, 0, 1, 210), (1, 1, 1, 210), (2, 0, 1, 220), (2, 1, 1, 220)]
    # without the catch-up every firing comes
    rc, got = trace([op for op in ops if op[0] != nat.DUE_CATCHUP], 2, 1)
    assert got[:2] == [(0, 0, 9, 100), (0, 1, 9, 100)]


def test_catchup_near_the_top_of_the_clock():
    """a grid that reaches 2^64 - 1: the last firing below it is kept, the one at it never comes"""
    p = 1 << 62
    ops = [(nat.DUE_ARM, 0, p - 1), (nat.DUE_CATCHUP, 0, IDLE), (nat.DUE_LAUNCH, 0, IDLE)]
    rc, got = trace(ops, 1, 1)
    assert rc == 0
    assert got == [(0, 0, 1, IDLE)]   # fired at 4 (2^62 - 1) = 2^64 - 4; the next firing is past the top
    ops = [(nat.DUE_ARM, 0, 3), (nat.DUE_CATCHUP, 0, IDLE - 1), (nat.DUE_LAUNCH, 0, IDLE)]
    rc, got = trace(ops, 1, 1)
    assert got == [(0, 0, 1, IDLE)]   # 2^64 - 1 is a multiple of 3: the firing there never comes


def test_catchup_rejects_a_step_behind_the_last_launch():
    assert trace([(nat.DUE_LAUNCH, 0, 9), (nat.DUE_CATCHUP, 0, 8)], 8, 1)[0] == nat.EINVAL


def oracle_trace(seed, K, n_subs=10, n_steps=250):
    """The flagged oracle against the model: subscribers with timers (armed, cancelled, re-armed, unsubscribed) and clock
    steps; after every step each mailbox's new tick records must be the model's, one per timer that fired."""
    rng = np.random.default_rng(seed)
    orc = DropOracle(n_subs, timers_per_sub=K)
    m = GoTickers()
    for _ in range(n_subs):
        orc.subscribe(0)
    live, owner, tid = set(range(n_subs)), {}, {}   # slot -> subscriber, slot -> oracle timer id
    clock, checked = 0, 0
    if seed % 3 == 0:
        clock = IDLE - int(rng.integers(1 << 40, 1 << 44))   # the top of the clock within reach
        assert orc.advance(clock) == 0
        m.clock = clock
    periods = []
    for _ in range(n_steps):
        for _ in range(int(rng.integers(0, 3))):
            r = rng.random()
            if r < 0.6 and live:
                s = int(rng.choice(sorted(live)))
                free = [k for k in range(K) if s * K + k not in owner]
                if not free:
                    continue
                p = _period(rng, clock)
                one = bool(rng.random() < 0.2)
                src = int(rng.integers(0, 1000))
                tid[s * K + free[0]] = orc.timer_add(s, p, src, one)
                assert tid[s * K + free[0]] == s * K + free[0]
                owner[s * K + free[0]] = s
                m.arm(s * K + free[0], p, one, src)
                periods.append(p)
            elif r < 0.85 and owner:
                slot = int(rng.choice(sorted(owner)))
                orc.timer_cancel(tid.pop(slot))
                del owner[slot]
                m.disarm(slot)
            elif len(live) > 1:
                s = int(rng.choice(sorted(live)))
                assert orc.unsubscribe(s) == 0
                live.discard(s)
                for k in range(K):
                    owner.pop(s * K + k, None); tid.pop(s * K + k, None)
                    m.disarm(s * K + k)
        now = _steps(rng, clock, [p for p in periods if p < 1 << 20], m)
        srcs = {s: m.t[s][4] for s in m.t}
        sent = m.wake(now)
        assert orc.advance(now) == 0
        for slot, (n, due) in sent.items():   # one-shots that fired and periodic timers are no longer armed in the model
            if slot in owner and slot not in m.t:
                del owner[slot]; tid.pop(slot, None)
        want = {s: [] for s in range(n_subs)}
        for slot in sorted(sent, key=lambda x: (sent[x][1], x)):   # (due, slot) order inside a mailbox
            n, due = sent[slot]
            want[slot // K].append((n & 0xFFFFFFFF, due, TIMER_EXPIRED, srcs[slot], slot // K, F_TICK))
        for s in range(n_subs):
            got = [tuple(int(r[f]) for f in ("seq", "ts_ns", "code", "source_id", "target", "flags"))
                   for r in orc.consume(s, 64)]
            assert got == want[s], f"seed {seed}, step to {now}, subscriber {s}: {got} vs {want[s]}"
            checked += len(got)
        clock = now
    return checked


@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("seed", range(4))
def test_flagged_oracle_matches_go_tickers(K, seed):
    assert oracle_trace(9000 * K + seed, K) > 50


def test_flagged_oracle_two_firings_coalesce_into_one():
    """the oracle: armed with period p at clock c, a step to exactly c + 2p delivers one tick, seq 1 and ts c + 2p, and the
    next at c + 3p with seq 2"""
    for c, p in ((0, 10), (1000, 7), (IDLE - 40, 10)):
        orc = DropOracle(1, timers_per_sub=1)
        orc.subscribe(0)
        assert orc.advance(c) == 0
        orc.timer_add(0, p, 5, False)
        assert orc.advance(c + 2 * p) == 0
        box = orc.consume(0, 8)
        assert [(int(r["seq"]), int(r["ts_ns"])) for r in box] == [(1, c + 2 * p)]
        if c + 3 * p < IDLE:
            assert orc.advance(c + 3 * p) == 0
            assert [(int(r["seq"]), int(r["ts_ns"])) for r in orc.consume(0, 8)] == [(2, c + 3 * p)]


def test_flagged_oracle_concrete_heartbeat():
    """1,000 timers of 1 s, one step of 1,000 s: one tick each, seq 999, due at 1,000 s; the plain oracle delivers 1,000"""
    import oracle_binding as ob
    s = 10 ** 9
    counts = []
    for orc in (DropOracle(1000, timers_per_sub=1), ob.Oracle(1000, timers_per_sub=1)):
        for i in range(1000):
            orc.subscribe(0x1FFFF)
            orc.timer_add(i, s, 7, False)
        assert orc.advance(1000 * s) == 0
        counts.append([orc.count(i) for i in range(1000)])
        if isinstance(orc, DropOracle):
            box = orc.mailbox(3)
            assert len(box) == 1 and int(box["seq"][0]) == 999 and int(box["ts_ns"][0]) == 1000 * s
            assert orc.advance(1001 * s) == 0 and int(orc.mailbox(3)["seq"][-1]) == 1000
    assert counts[0] == [1] * 1000 and counts[1] == [1000] * 1000
