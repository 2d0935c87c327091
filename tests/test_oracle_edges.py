"""The checker's side of the edge rules for complete records and clocks (CPU only): broadcast codes outside the enum,
due times that saturate instead of wrapping past 2^64, and the publish ordinal after a batch of complete records.  The
GPU suite holds the bus to the same rules (test_gpu_record_edges.py)."""
import numpy as np
import pytest

import oracle_binding as ob
import trace as tr

U64 = (1 << 64) - 1
TARGET_ALL = 0xFFFFFFFF
OUT_OF_RANGE = [17, 20, 23, 24, 25, 27, 28, 29, 31, 32, 1000, 0xFFFFFFFF]


def _records(rows):
    """rows of (seq, ts, code, source, target, flags)"""
    ev = np.zeros(len(rows), dtype=ob.EVENT_DTYPE)
    for i, r in enumerate(rows):
        ev[i] = r
    return ev


@pytest.mark.parametrize("code", OUT_OF_RANGE)
def test_broadcast_code_outside_the_enum_reaches_no_mailbox(code):
    """A complete broadcast record with a code >= 17 is matched by no mask (not even every bit set) and no pair, is not
    counted per code, and still enters the debug ring.  The same code in a unicast record is delivered."""
    orc = ob.Oracle(4)
    everyone = orc.subscribe(0xFFFFFFFF)
    dense = orc.subscribe(tr.MASK_ALL)
    paired = orc.subscribe(0, pairs=[(16, 5), (1, 5)])
    target = orc.subscribe(0)
    ev = _records([(10, 100, 3, 5, TARGET_ALL, 0), (11, 101, code, 5, TARGET_ALL, 0), (12, 102, 16, 5, TARGET_ALL, 0),
                   (13, 103, code, 7, target, 2)])
    assert orc.publish_records(ev, 200) == 0
    assert [int(r["seq"]) for r in orc.mailbox(everyone)] == [10, 12]
    assert [int(r["seq"]) for r in orc.mailbox(dense)] == [10, 12]
    assert [int(r["seq"]) for r in orc.mailbox(paired)] == [12]
    assert orc.mailbox(target).tobytes() == ev[3:].tobytes()
    assert [orc.published_by_code(c) for c in (3, 16)] == [1, 1]
    assert sum(orc.published_by_code(c) for c in range(17)) == 2
    assert orc.debug_events().tobytes() == ev[:3].tobytes()


def test_host_publish_of_an_out_of_range_code_reaches_no_mailbox():
    orc = ob.Oracle(1)
    s = orc.subscribe(0xFFFFFFFF)
    assert orc.publish(31, 1) == 0 and orc.publish(1, 1) == 0
    assert [int(r["code"]) for r in orc.mailbox(s)] == [1]


@pytest.mark.parametrize("t0,period", [(3, U64 - 2), (1 << 63, 1 << 63), ((1 << 64) - (1 << 40), U64),
                                       (U64 - 5, 5), (U64 - 1, 1)])
@pytest.mark.parametrize("oneshot", [False, True])
def test_first_due_time_past_the_top_saturates_to_never(t0, period, oneshot):
    """now + period > 2^64 - 2 (a wrap, or exactly UINT64_MAX) is "never": nothing fires even at the largest clock, and the
    timer stays armed (a cancel finds it)."""
    orc = ob.Oracle(1, timers_per_sub=1)
    s = orc.subscribe()
    assert orc.advance(t0) == 0
    tid = orc.timer_add(s, period, 9, oneshot)
    assert orc.advance(U64) == 0
    assert orc.count(s) == 0 and orc.total_ticks() == 0
    assert orc.timer_cancel(tid) == 0


def test_periodic_rearm_past_the_top_saturates():
    """A periodic timer fires each due time up to 2^64 - 2 and then never again; the clock may still reach UINT64_MAX."""
    orc = ob.Oracle(2, timers_per_sub=1)
    a, b = orc.subscribe(), orc.subscribe()
    assert orc.advance(U64 - 7) == 0
    orc.timer_add(a, 3, 1)                               # due -4, -1 (= 2^64 - 2), then 2^64 + 2: never
    tb = orc.timer_add(b, 1, 2)                          # due -6 ... -1: six ticks, then 2^64 - 1: never
    assert orc.advance(U64) == 0
    ma, mb = orc.mailbox(a), orc.mailbox(b)
    assert [int(r["ts_ns"]) for r in ma] == [U64 - 4, U64 - 1]
    assert [int(r["seq"]) for r in ma] == [0, 1]
    assert [int(r["ts_ns"]) for r in mb] == list(range(U64 - 6, U64))
    assert orc.total_ticks() == 8
    assert orc.timer_cancel(tb) == 0


def test_period_of_go_max_duration_fires_once_then_never():
    orc = ob.Oracle(1, timers_per_sub=1)
    s = orc.subscribe()
    assert orc.advance(2) == 0
    orc.timer_add(s, (1 << 63) - 1, 4)                   # due 2^63 + 1, then 2^64: never
    assert orc.advance((1 << 63)) == 0 and orc.count(s) == 0
    assert orc.advance(U64) == 0
    assert [int(r["ts_ns"]) for r in orc.mailbox(s)] == [(1 << 63) + 1]


def test_due_time_of_top_minus_one_fires_and_a_tick_precedes_a_record_at_its_due_time():
    orc = ob.Oracle(1, timers_per_sub=2)
    s = orc.subscribe()
    assert orc.advance(U64 - 11) == 0
    orc.timer_add(s, 10, 7, oneshot=True)                # due 2^64 - 2
    ev = _records([(1 << 40, U64 - 1, 2, 1, TARGET_ALL, 0xABCD)])
    assert orc.publish_records(ev, U64) == 0
    m = orc.mailbox(s)
    assert [int(r["code"]) for r in m] == [8, 2] and int(m[0]["ts_ns"]) == U64 - 1 and int(m[1]["flags"]) == 0xABCD


def test_publish_records_advances_the_ordinal_by_the_record_count():
    """The next host publish after n complete records carries the previous ordinal + n, whatever seqs the records had."""
    orc = ob.Oracle(2)
    s = orc.subscribe()
    t = orc.subscribe()
    assert orc.publish(1, 1) == 0 and orc.publish(2, 1) == 0                     # seqs 0, 1
    ev = _records([(1 << 33, 5, 3, 1, TARGET_ALL, 0), (7, 6, 4, 1, t, 2), ((1 << 64) - 1, 7, 5, 1, TARGET_ALL, 0)])
    assert orc.publish_records(ev, 10) == 0
    assert orc.publish(6, 1) == 0 and orc.receive(t, 7, 1) == 0
    assert [int(r["seq"]) for r in orc.mailbox(s)] == [0, 1, 1 << 33, (1 << 64) - 1, 5]
    assert [int(r["seq"]) for r in orc.mailbox(t)][-2:] == [5, 6]
