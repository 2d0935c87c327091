"""cpbus_drain_ready: the sparse mailbox -> host drain.  Equivalence with the oracle (lossless) and with cpbus_drain on a twin
bus (throughput), the exact selection rules against a host model, shards and subranges, interplay with the other consumers,
a 1,048,576-subscriber bus with few ready mailboxes, the error codes, and the C++ mirror's pump on large fleets."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_binding as ob
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE, READY_DTYPE

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


class Stepper:
    """Applies trace ops one at a time to a bus (and the oracle), keeping the timer handles of the whole trace."""

    def __init__(self, bus, orc=None, base=0):
        self.bus, self.orc, self.base, self.hb, self.ho = bus, orc, base, [], []
        self.n_subs = 0                      # subscribers so far: the ids a drain may name mid-trace

    def apply(self, op):
        bus, orc, base, k = self.bus, self.orc, self.base, op[0]
        if k == "sub":
            bus.subscribe_pairs(op[1], op[2]) if len(op) > 2 else bus.subscribe(op[1])
            self.n_subs += 1
            if orc:
                orc.subscribe(op[1], op[2] if len(op) > 2 else None)
        elif k == "unsub":
            bus.unsubscribe(base + op[1])
            if orc:
                assert orc.unsubscribe(base + op[1]) == 0
        elif k == "pub":
            nat.check(bus.publish(op[1], op[2]), "publish")
            if orc:
                assert orc.publish(op[1], op[2]) == 0
        elif k == "send":
            nat.check(bus.send(base + op[1], op[2], op[3]), "send")
            if orc:
                assert orc.receive(base + op[1], op[2], op[3]) == 0
        elif k == "adv":
            nat.check(bus.advance(op[1]), "advance")
            if orc:
                assert orc.advance(op[1]) == 0
        elif k == "tadd":
            self.hb.append(bus.timer_add(base + op[1], op[2], op[3], op[4]))
            if orc:
                self.ho.append(orc.timer_add(base + op[1], op[2], op[3], op[4]))
        elif k == "tcancel":
            try:
                bus.timer_cancel(self.hb[op[1]])
            except nat.CpbusError as e:
                assert e.status == nat.ENOENT
            if orc:
                assert orc.timer_cancel(self.ho[op[1]]) in (0, ob.ENOENT)
        elif k == "flush":
            nat.check(bus.flush(), "flush")


def check_call(rec, rdy, first, n, start):
    """Shape rules of one call: runs packed back to back in entry order, entries in cyclic order from start, no empty run."""
    assert (rdy["pad"] == 0).all() and (rdy["count"] > 0).all()
    off = np.concatenate([[0], np.cumsum(rdy["count"].astype(np.int64))])
    assert (rdy["offset"] == off[:-1]).all() and off[-1] == len(rec)
    pos = (rdy["sub_id"].astype(np.int64) - start) % n
    assert (np.diff(pos) > 0).all()
    assert ((rdy["sub_id"] >= first) & (rdy["sub_id"] < first + n)).all()


def drain_until_empty(bus, first, n, cap, ready_cap, start=None, runs=None, lost=None, log=None):
    """drain_ready until nothing is ready, always resuming at next_sub; runs[gid] += records, lost[gid] += lost."""
    start = first if start is None else start
    runs = {} if runs is None else runs
    lost = {} if lost is None else lost
    while True:
        rec, rdy, nxt = bus.drain_ready(first, n, start, cap, ready_cap)
        check_call(rec, rdy, first, n, start)
        if log is not None:
            log.append((rec.tobytes(), rdy.tobytes(), nxt))
        if len(rdy) == 0:
            assert nxt == start and len(rec) == 0
            return runs, lost
        for e in rdy:
            g = int(e["sub_id"])
            runs.setdefault(g, []).append(rec[int(e["offset"]):int(e["offset"]) + int(e["count"])].copy())
            lost[g] = lost.get(g, 0) + int(e["lost"])
        start = nxt


def drain_with_lost(bus, sub_id, cap):
    out = np.zeros(cap, dtype=EVENT_DTYPE)
    n, lost = C.c_size_t(), C.c_uint64()
    nat.check(bus._lib.cpbus_drain(bus._h, sub_id, out.ctypes.data, cap, C.byref(n), C.byref(lost)), "cpbus_drain")
    return out[:n.value], lost.value


def cat(parts):
    return np.concatenate(parts) if parts else np.zeros(0, dtype=EVENT_DTYPE)


# ------------------------------------------------------------------------------------------------ 1. equivalence ---
@pytest.mark.parametrize("K", [0, 1, 8])
@pytest.mark.parametrize("seed", [1, 2])
def test_lossless_runs_equal_the_oracle(K, seed):
    """Random traces (filters, pair tables, unicast, membership changes, timers) in lossless mode, drained every 100 ops
    with cap = ring_cap and ready_cap = 7: each subscriber's concatenated runs are exactly its oracle mailbox."""
    R, B = 1024, 64
    ops, n_total = tr.random_ops(seed * 31 + K, 40, 3000, timers_per_sub=K, p_pairs=0.3, p_member=0.01)
    orc = ob.Oracle(n_total + 1, timers_per_sub=K, keep_window=0)
    runs = {}
    with Bus(n_total + 1, ring_cap=R, batch_cap=B, timers_per_sub=K, lossless=True) as bus:
        st = Stepper(bus, orc)
        for i, op in enumerate(ops):
            st.apply(op)
            if i % 100 == 99:
                nat.check(bus.flush(), "flush")
                drain_until_empty(bus, 0, st.n_subs, R, 7, start=(i * 13) % st.n_subs, runs=runs)
        nat.check(bus.flush(), "flush")
        drain_until_empty(bus, 0, n_total, R, 7, runs=runs)
        for s in range(n_total):
            assert cat(runs.get(s, [])).tobytes() == orc.mailbox(s).tobytes(), f"subscriber {s}"
        assert bus.stats()["overwritten"] == 0


@pytest.mark.parametrize("K", [0, 1, 8])
@pytest.mark.parametrize("seed", [1, 2])
def test_throughput_runs_and_lost_equal_cpbus_drain_on_a_twin(K, seed):
    """Throughput mode with 64-record rings, so mailboxes overflow between drains: the runs and the lost counts equal what
    cpbus_drain returns on a twin bus given the same trace and drained at the same points."""
    R, B = 64, 32
    ops, n_total = tr.random_ops(seed * 17 + K, 30, 2500, timers_per_sub=K, p_pairs=0.3)
    runs, lost = {}, {}
    twin_runs, twin_lost = {}, {}
    with Bus(n_total + 1, ring_cap=R, batch_cap=B, timers_per_sub=K) as bus, \
            Bus(n_total + 1, ring_cap=R, batch_cap=B, timers_per_sub=K) as twin:
        sa, sb = Stepper(bus), Stepper(twin)

        def drain_both(start):
            n = sa.n_subs
            nat.check(bus.flush(), "flush"); nat.check(twin.flush(), "flush")
            drain_until_empty(bus, 0, n, R, 7, start=start % n, runs=runs, lost=lost)
            for s in range(n):
                g, l_ = drain_with_lost(twin, s, R)
                if len(g):
                    twin_runs.setdefault(s, []).append(g)
                    twin_lost[s] = twin_lost.get(s, 0) + l_
                else:
                    assert l_ == 0

        for i, op in enumerate(ops):
            sa.apply(op); sb.apply(op)
            if i % 150 == 149:
                drain_both(i * 7)
        drain_both(0)
        assert sum(lost.values()) > 0                                  # the trace did overflow some mailboxes
        for s in range(n_total):
            assert cat(runs.get(s, [])).tobytes() == cat(twin_runs.get(s, [])).tobytes(), f"subscriber {s}"
            assert lost.get(s, 0) == twin_lost.get(s, 0), f"subscriber {s}"


# --------------------------------------------------------------------------------------------- 2. selection rules ---
def model_call(counts, first, n, start, cap, ready_cap):
    """The documented selection: ready mailboxes in cyclic order from start while the whole run fits."""
    taken, tot = [], 0
    for i in range(n):
        s = first + (start - first + i) % n
        c = counts.get(s, 0)
        if not c:
            continue
        if len(taken) + 1 > ready_cap or tot + c > cap:
            return taken, s
        taken.append((s, c, tot))
        tot += c
    return taken, start


@pytest.mark.parametrize("base,first_off,n_range", [(0, 0, 48), (1000, 0, 48), (1000, 13, 29)])
def test_selection_rules_match_the_model(base, first_off, n_range):
    """Unicast records of known counts (0 to a full ring) in a 48-mailbox shard; random start, cap in [R, 3R] and ready_cap
    in [1, 9]: the entries (global ids, counts, offsets), the records (FIFO) and next_sub equal the model's, including the
    stop at the first run that does not fit and wrap-around.  Also a shard with sub_id_base != 0 and a range that starts
    mid-shard."""
    R, B, N = 64, 32, 48
    rng = np.random.default_rng(base + first_off)
    first = base + first_off
    with Bus(N, ring_cap=R, batch_cap=B, sub_id_base=base) as bus:
        bus.subscribe_many(np.zeros(N, dtype=np.uint32))
        queues = {g: [] for g in range(base, base + N)}
        nxt_src = [0]

        def refill():
            for _ in range(int(rng.integers(1, 4))):
                g = base + int(rng.integers(0, N))
                k = int(rng.integers(1, R - len(queues[g]) + 1)) if len(queues[g]) < R else 0
                for _ in range(k):
                    nat.check(bus.send(g, 1 + g % 16, nxt_src[0]), "send")
                    queues[g].append(nxt_src[0]); nxt_src[0] += 1
            nat.check(bus.flush(), "flush")

        n_cut = 0
        for it in range(120):
            refill()
            start = first + int(rng.integers(0, n_range))
            cap = int(rng.integers(R, 3 * R + 1))
            rcap = int(rng.integers(1, 10))
            counts = {g: len(q) for g, q in queues.items() if first <= g < first + n_range}
            want, want_next = model_call(counts, first, n_range, start, cap, rcap)
            rec, rdy, nxt = bus.drain_ready(first, n_range, start, cap, rcap)
            check_call(rec, rdy, first, n_range, start)
            assert [(int(e["sub_id"]), int(e["count"]), int(e["offset"])) for e in rdy] == want
            assert nxt == want_next
            n_cut += want_next != start
            for g, c, o in want:
                run = rec[o:o + c]
                assert (run["target"] == g).all() and (run["flags"] == nat.F_UNICAST).all()
                assert list(run["source_id"]) == queues[g][:c] and c == len(queues[g])
                queues[g] = []
        assert n_cut >= 5                                           # the stop rule was exercised
        for g in range(base, base + N):                                # untouched mailboxes kept their records
            assert len(bus.drain(g)) == len(queues[g])


def test_full_range_drains_in_exactly_n_calls_and_is_deterministic():
    """Every mailbox full: calls at cap = ring_cap take one mailbox each, in ascending cyclic order from start_sub, and
    the whole range is empty after exactly n calls.  Two identical buses give byte-identical outputs call by call."""
    R, B, N = 64, 32, 24
    logs = []
    for _ in range(2):
        with Bus(N, ring_cap=R, batch_cap=B) as bus:
            bus.subscribe_many(np.full(N, nat.MASK_ALL, dtype=np.uint32))
            ev = np.zeros(R, dtype=EVENT_DTYPE)
            ev["code"] = np.arange(R) % 16 + 1; ev["source_id"] = np.arange(R)
            nat.check(bus.publish_many(ev), "publish"); nat.check(bus.flush(), "flush")
            start, log = 17, []
            for i in range(N):
                rec, rdy, nxt = bus.drain_ready(0, N, start, R, 100)
                assert len(rdy) == 1 and int(rdy[0]["sub_id"]) == (17 + i) % N and len(rec) == R
                assert (rec["source_id"] == np.arange(R)).all()
                assert nxt == (18 + i) % N if i < N - 1 else nxt == start
                log.append((rec.tobytes(), rdy.tobytes(), nxt))
                start = nxt
            rec, rdy, nxt = bus.drain_ready(0, N, start, R, 100)
            assert len(rdy) == 0 and nxt == start
            logs.append(log)
    assert logs[0] == logs[1]


def test_identical_buses_give_byte_identical_drains():
    """A random trace (throughput mode, so some runs report lost records) on two buses: every drain_ready call returns
    byte-identical records, ready lists and next_sub."""
    R, B = 64, 32
    ops, n_total = tr.random_ops(77, 60, 2000, timers_per_sub=1, p_pairs=0.3)
    logs = []
    for _ in range(2):
        log = []
        with Bus(n_total + 1, ring_cap=R, batch_cap=B, timers_per_sub=1) as bus:
            st = Stepper(bus)
            for i, op in enumerate(ops):
                st.apply(op)
                if i % 200 == 199:
                    nat.check(bus.flush(), "flush")
                    drain_until_empty(bus, 0, st.n_subs, 2 * R, 5, start=i % st.n_subs, log=log)
        logs.append(log)
    assert logs[0] == logs[1] and len(logs[0]) > 20


# ---------------------------------------------------------------------------------------------------- 4. interplay ---
def test_mixed_consumers_on_one_bus():
    """drain, drain_many, consume_all and drain_ready on one lossless bus: every record a host consumer receives is the
    next one of that subscriber's oracle mailbox; consume_all discards up to the delivered count.  (Rings of 4096 records:
    a consumer that only drains a few mailboxes never lets one fill up, so no flush is refused.)"""
    R, B = 4096, 64
    ops, n_total = tr.random_ops(5, 50, 3000, timers_per_sub=1, p_pairs=0.3)
    orc = ob.Oracle(n_total + 1, timers_per_sub=1, keep_window=0)
    pos = [0] * n_total
    rng = np.random.default_rng(5)

    def took(s, recs):
        want = orc.mailbox(s)[pos[s]:pos[s] + len(recs)]
        assert recs.tobytes() == want.tobytes(), f"subscriber {s}"
        pos[s] += len(recs)

    kinds = []
    with Bus(n_total + 1, ring_cap=R, batch_cap=B, timers_per_sub=1, lossless=True) as bus:
        st = Stepper(bus, orc)
        for i, op in enumerate(ops):
            st.apply(op)
            if i % 100 != 99:
                continue
            nat.check(bus.flush(), "flush")
            n = st.n_subs
            kind = ["drain", "drain_many", "consume_all", "drain_ready"][int(rng.integers(0, 4))]
            kinds.append(kind)
            if kind == "drain":
                for s in rng.permutation(n)[:10]:
                    took(int(s), bus.drain(int(s), cap=int(rng.integers(1, 50))))
            elif kind == "drain_many":
                rec, offs, cnts = bus.drain_many(0, n, n * R)
                for s in range(n):
                    took(s, rec[offs[s]:offs[s] + cnts[s]])
            elif kind == "consume_all":
                bus.consume_all(); bus.sync()
                pos[:n] = [orc.count(s) for s in range(n)]
            else:
                runs, _ = drain_until_empty(bus, 0, n, R, 7, start=int(rng.integers(0, n)))
                for s, parts in runs.items():
                    took(s, cat(parts))
        nat.check(bus.flush(), "flush")
        runs, _ = drain_until_empty(bus, 0, n_total, R, 7)
        for s, parts in runs.items():
            took(s, cat(parts))
        assert pos == [orc.count(s) for s in range(n_total)]
    assert set(kinds) == {"drain", "drain_many", "consume_all", "drain_ready"}


@pytest.mark.parametrize("seed", [1, 2])
def test_lossless_back_pressure_is_released_by_drain_ready(seed):
    """A full mailbox makes cpbus_flush return EAGAIN at the oracle's stall point (mailbox_cap = ring_cap); drain_ready
    frees the room, the flush continues with the first undelivered event, and the drained sequences equal the oracle's."""
    R, B, N = 128, 64, 6
    rng = np.random.default_rng(300 + seed)
    masks = [nat.MASK_ALL, 1 << 2, (1 << 3) | (1 << 2), nat.MASK_ALL, 1 << 5, 0]
    orc = ob.Oracle(N, keep_window=0, mailbox_cap=R)
    for m_ in masks:
        orc.subscribe(m_)
    n_again = 0
    with Bus(N, ring_cap=R, batch_cap=B, lossless=True) as bus:
        bus.subscribe_many(np.array(masks, dtype=np.uint32))
        for step in range(40):
            ev = np.zeros(B, dtype=EVENT_DTYPE)
            ev["code"] = rng.integers(1, 7, B); ev["source_id"] = step * B + np.arange(B)
            nat.check(bus.publish_many(ev), "publish")
            i = 0
            while True:
                rc = bus.flush()
                while i < B:
                    r = orc.publish(int(ev["code"][i]), int(ev["source_id"][i]))
                    if r == ob.EAGAIN:
                        break
                    assert r == 0
                    i += 1
                if rc == nat.OK:
                    assert i == B
                    break
                assert rc == nat.EAGAIN and i < B
                n_again += 1
                if rng.random() < 0.5:                                # the consumers take everything
                    runs, _ = drain_until_empty(bus, 0, N, R, 3, start=int(rng.integers(0, N)))
                    for s in range(N):
                        got = cat(runs.get(s, []))
                        assert got.tobytes() == orc.consume(s, R).tobytes()
                else:                                                 # or only one call's worth
                    rec, rdy, _ = bus.drain_ready(0, N, int(rng.integers(0, N)), R, 2)
                    assert len(rdy) >= 1
                    for e in rdy:
                        s = int(e["sub_id"])
                        got = rec[int(e["offset"]):int(e["offset"]) + int(e["count"])]
                        assert got.tobytes() == orc.consume(s, int(e["count"])).tobytes()
        runs, _ = drain_until_empty(bus, 0, N, R, 3)
        for s in range(N):
            assert cat(runs.get(s, [])).tobytes() == orc.consume(s, R).tobytes()
        assert bus.stats()["overwritten"] == 0
    assert n_again > 5


# ------------------------------------------------------------------------------------------------- 5. sparse scale ---
def test_sparse_million_subscriber_bus():
    """1,048,576 subscribers, about 50 of which receive direct sends: one drain returns exactly those mailboxes, in id
    order from start_sub, with the oracle's records; an empty drain returns nothing, hands start_sub back and changes
    nothing."""
    N, R, B = 1 << 20, 64, 32
    rng = np.random.default_rng(11)
    hot = sorted(set(int(x) for x in rng.integers(0, N, 50)))
    orc = ob.Oracle(N, keep_window=0)
    for _ in range(N):
        orc.subscribe(0)
    with Bus(N, ring_cap=R, batch_cap=B) as bus:
        bus.subscribe_many(np.zeros(N, dtype=np.uint32))
        rec, rdy, nxt = bus.drain_ready(0, N, 12345, R, 64)
        assert len(rdy) == 0 and len(rec) == 0 and nxt == 12345
        for j in range(200):
            s = hot[j % len(hot)] if j < 150 else hot[int(rng.integers(0, len(hot)))]
            code, src = 1 + j % 16, j
            nat.check(bus.send(s, code, src), "send"); assert orc.receive(s, code, src) == 0
        nat.check(bus.flush(), "flush")
        start = hot[len(hot) // 2]
        rec, rdy, nxt = bus.drain_ready(0, N, start, 1 << 16, 1 << 16)
        order = sorted(hot, key=lambda g: (g - start) % N)
        assert [int(g) for g in rdy["sub_id"]] == order and nxt == start
        for e in rdy:
            g = int(e["sub_id"])
            assert rec[int(e["offset"]):int(e["offset"]) + int(e["count"])].tobytes() == orc.mailbox(g).tobytes()
        before = bus.digest_fold(0, N)
        rec, rdy, nxt = bus.drain_ready(0, N, 777, R, 64)
        assert len(rdy) == 0 and nxt == 777
        assert bus.digest_fold(0, N) == before
        assert all(len(bus.drain(g)) == 0 for g in hot[:5])


# ------------------------------------------------------------------------------------------------------- 6. errors ---
def test_error_codes():
    R = 64
    with Bus(32, ring_cap=R, batch_cap=32, sub_id_base=100) as bus:
        bus.subscribe_many(np.zeros(20, dtype=np.uint32))
        lib, h = bus._lib, bus._h
        out = np.zeros(4 * R, dtype=EVENT_DTYPE)
        rdy = np.zeros(16, dtype=READY_DTYPE)
        nr, tot, nxt = C.c_size_t(), C.c_size_t(), C.c_uint32()

        def call(first=100, n=20, start=100, o=out.ctypes.data, cap=R, r=rdy.ctypes.data, rcap=16, a=True, b=True, c=True, hh=h):
            return lib.cpbus_drain_ready(hh, first, n, start, o, cap, r, rcap, C.byref(nr) if a else None,
                                         C.byref(tot) if b else None, C.byref(nxt) if c else None)
        assert call() == nat.OK and nr.value == 0 and nxt.value == 100
        assert call(start=119) == nat.OK and nxt.value == 119
        assert call(hh=None) == nat.EINVAL
        assert call(o=None) == nat.EINVAL
        assert call(r=None) == nat.EINVAL
        assert call(a=False) == nat.EINVAL and call(b=False) == nat.EINVAL and call(c=False) == nat.EINVAL
        assert call(n=0) == nat.EINVAL
        assert call(cap=R - 1) == nat.EINVAL
        assert call(cap=0x1_0000_0000) == nat.EINVAL
        assert call(rcap=0) == nat.EINVAL
        assert call(start=99) == nat.EINVAL and call(start=120) == nat.EINVAL
        assert call(first=110, n=5, start=109) == nat.EINVAL and call(first=110, n=5, start=115) == nat.EINVAL
        assert call(first=99, n=20, start=99) == nat.ENOENT          # below this shard
        assert call(first=100, n=21, start=100) == nat.ENOENT         # beyond the subscribers this shard has
        assert call(first=0, n=5, start=0) == nat.ENOENT


# ------------------------------------------------------------------------------------------------ 7. C++ mirror ---
def test_cpp_mirror_pump_on_large_fleets():
    """events_sparse_test.cc: EventBus::DrainAll over cpbus_drain_ready with 6,000 subscribers of which 40 receive records
    (FIFO per subscriber, pending records of full channels), and with 5,000 ready mailboxes (more than one call takes)."""
    exe = os.path.join(os.path.dirname(HERE), "containerpilot_b200", "csrc", "host", "events_sparse_test")
    assert os.path.exists(exe), "build with __graft_entry__.build()"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("PASS"), r.stdout + r.stderr
