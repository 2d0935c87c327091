"""Sparse drains (CPBUS_CFG_SPARSE_DRAINS) without a GPU: the flag and the trace export, a plain-C99 caller, cpbus_create's
and the group's refusal of the flag, and the candidate index (cpbus_ready_trace, the bus's own code) against a model of
every mailbox's cursors on seeded op lists: each drain's candidates hold every mailbox with records for its predicate,
or the drain takes the dense scan.  Hand-built cases pin the exact lists.  The bus itself needs a GPU:
tests/test_gpu_sparse_drains.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from containerpilot_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DENSE = -1


def test_flag_and_export():
    lib = C.CDLL(nat.LIB_PATH)
    assert hasattr(lib, "cpbus_ready_trace") and "cpbus_ready_trace" in nat.SYMBOLS
    others = (nat.CFG_LOSSLESS | nat.CFG_DIGEST | nat.CFG_SPARSE_TICKS | nat.CFG_SPARSE_RECORDS
              | nat.CFG_DROP_MISSED_TICKS)
    assert nat.CFG_SPARSE_DRAINS == 0x20 and not nat.CFG_SPARSE_DRAINS & others
    hdr = open(os.path.join(ROOT, "include", "cpbus.h")).read()
    assert "#define CPBUS_CFG_SPARSE_DRAINS 0x20u" in hdr
    assert nat.load().cpbus_abi_version() == 2


def _cfg(flags):
    cfg = nat.Config()
    cfg.n_max_subs, cfg.ring_cap, cfg.batch_cap, cfg.timers_per_sub, cfg.device = 64, 1024, 256, 1, -1
    cfg.flags = flags
    return cfg


@pytest.mark.parametrize("lossless", [0, nat.CFG_LOSSLESS])
def test_create_refuses_the_flag_without_sparse_ticks(lossless):
    """CPBUS_EINVAL before any device is looked at (so also on a machine without one)"""
    lib = nat.load()
    for flags in (nat.CFG_SPARSE_DRAINS, nat.CFG_SPARSE_DRAINS | nat.CFG_SPARSE_RECORDS):
        h = C.c_void_p()
        assert lib.cpbus_create(C.byref(_cfg(flags | lossless)), C.byref(h)) == nat.EINVAL
        assert not h.value


def test_group_refuses_the_flag():
    lib = nat.load()
    devs = (C.c_int32 * 2)(0, 0)
    for flags in (nat.CFG_SPARSE_DRAINS, nat.CFG_SPARSE_DRAINS | nat.CFG_SPARSE_TICKS):
        h = C.c_void_p()
        assert lib.cpbus_group_create(C.byref(_cfg(flags | nat.CFG_LOSSLESS)), devs, 2, C.byref(h)) == nat.EINVAL
        assert not h.value


def test_sparse_drains_declarations_from_plain_c99(tmp_path):
    exe = str(tmp_path / "sparse_drains_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "sparse_drains_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr


class Trace:
    """An op list for cpbus_ready_trace, built call by call."""

    def __init__(self):
        self.ops, self.ids = [], []

    def _op(self, kind, ticket=0, first=0, n=0, ids=(), cut=0):
        self.ops.append((kind, ticket, first, n, len(self.ids), len(ids), cut))
        self.ids.extend(int(i) for i in ids)
        return len(self.ops) - 1

    def sparse(self, ids): return self._op(nat.READY_SPARSE, ids=ids)
    def full(self): return self._op(nat.READY_FULL)
    def begin(self, ticket, first, n, take=False): return self._op(nat.READY_TAKE if take else nat.READY_DRAIN, ticket, first, n)
    def end(self, ticket, ids, cut): return self._op(nat.READY_END, ticket, ids=ids, cut=cut)
    def consume_all(self): return self._op(nat.READY_CONSUME_ALL)
    def release(self, ids): return self._op(nat.READY_RELEASE, ids=ids)

    def drain(self, ticket, first, n, took, cut, take=False):
        i = self.begin(ticket, first, n, take)
        self.end(ticket, took, cut)
        return i

    def run(self, n_subs, list_cap=1024):
        """(status, per-op candidate list or DENSE, for the DRAIN / TAKE ops)"""
        lib = nat.load()
        ops = np.zeros(max(1, len(self.ops)), dtype=nat.READY_OP_DTYPE)
        for i, o in enumerate(self.ops):
            ops[i] = o
        ids = np.ascontiguousarray(self.ids or [0], dtype=np.uint32)
        counts = np.zeros(max(1, len(self.ops)), dtype=np.int64)
        n = C.c_size_t()
        args = (ops.ctypes.data, len(self.ops), ids.ctypes.data, len(self.ids), n_subs, list_cap)
        rc = lib.cpbus_ready_trace(*args, None, 0, counts.ctypes.data, C.byref(n))
        if rc:
            return rc, None
        out = np.zeros(max(1, n.value), dtype=np.uint32)
        nat.check(lib.cpbus_ready_trace(*args, out.ctypes.data, n.value, counts.ctypes.data, C.byref(n)), "cpbus_ready_trace")
        res, k = {}, 0
        for i, o in enumerate(self.ops):
            if o[0] in (nat.READY_DRAIN, nat.READY_TAKE):
                c = int(counts[i])
                res[i] = DENSE if c < 0 else [int(x) for x in out[k:k + c]]
                k += max(c, 0)
        return 0, res


class Model:
    """Every mailbox's tail, head and take cursor: which mailboxes hold records for each predicate."""

    def __init__(self, n):
        self.tail, self.head, self.taken = [0] * n, [0] * n, [0] * n

    def unread(self, l): return self.tail[l] > self.head[l]
    def untaken(self, l): return self.tail[l] > max(self.taken[l], self.head[l])


def _random_trace(seed, n_subs, list_cap, steps):
    rng = random.Random(seed)
    m, t = Model(n_subs), Trace()
    expect = {}                     # begin op -> (take, mailboxes with records for its predicate in its range)
    open_tk = {}                    # ticket -> (took, cut)
    next_ticket = 0
    for _ in range(steps):
        r = rng.random()
        if r < 0.25:                # sparse launch
            ids = rng.sample(range(n_subs), rng.randint(1, min(n_subs, 3 * list_cap if rng.random() < 0.1 else 6)))
            for l in ids:
                m.tail[l] += rng.randint(1, 3)
            t.sparse(ids)
        elif r < 0.30:              # full launch: any mailbox may take records, or none
            for l in range(n_subs):
                if rng.random() < 0.3:
                    m.tail[l] += rng.randint(1, 2)
            t.full()
        elif r < 0.62 and len(open_tk) < 8:   # a drain or take begins; its effect is at its place in stream order
            take = rng.random() < 0.4
            if rng.random() < 0.6:
                first, n = 0, n_subs
            else:
                first = rng.randrange(n_subs)
                n = rng.randint(1, n_subs - first)
            rot = rng.randrange(n)
            walk = [first + (rot + p) % n for p in range(n)]
            pred = m.untaken if take else m.unread
            ready = [l for l in walk if pred(l)]
            k = len(ready) if rng.random() < 0.7 else rng.randint(0, len(ready))
            took = ready[:k]
            cut = n if k == len(ready) else walk.index(ready[k]) if k < len(ready) else n
            for l in took:
                if take:
                    m.taken[l] = m.tail[l]
                else:
                    m.head[l] = m.tail[l]
            ticket = next_ticket
            next_ticket += 1
            i = t.begin(ticket, first, n, take)
            expect[i] = (take, {l for l in range(first, first + n) if (l in took) or pred(l)})
            open_tk[ticket] = (took, cut)
        elif r < 0.85 and open_tk:  # a ticket ends, in any order
            ticket = rng.choice(sorted(open_tk))
            took, cut = open_tk.pop(ticket)
            t.end(ticket, took, cut)
        elif r < 0.90:              # acks move head up to the take cursor: fewer records, nothing for the index
            for l in range(n_subs):
                if rng.random() < 0.5:
                    m.head[l] = max(m.head[l], min(m.taken[l], m.tail[l]))
        elif r < 0.94:
            m.head = list(m.tail)
            t.consume_all()
        else:
            ids = rng.sample(range(n_subs), rng.randint(1, 3))
            for l in ids:
                m.tail[l] = m.head[l] = m.taken[l] = 0
            t.release(ids)
    for ticket, (took, cut) in open_tk.items():
        t.end(ticket, took, cut)
    return t, expect


@pytest.mark.parametrize("seed", range(24))
def test_candidates_cover_every_mailbox_with_records(seed):
    """The invariant on seeded op lists: a drain's candidates hold every mailbox of its range that has records for its
    predicate at its place (the ones it takes included), or it takes the dense scan.  And the index is not merely
    conservative: known lists occur, and some of them skip mailboxes."""
    n_subs = [16, 64, 300][seed % 3]
    list_cap = [2, 8, 1024][seed % 3 if seed % 2 else 2]
    t, expect = _random_trace(seed, n_subs, list_cap, 400)
    rc, res = t.run(n_subs, list_cap)
    assert rc == 0
    known = 0
    for i, (take, need) in expect.items():
        got = res[i]
        if got == DENSE:
            continue
        known += 1
        assert got == sorted(set(got)) and len(got) <= list_cap, (i, got)
        assert need <= set(got), (i, take, sorted(need - set(got)))
    assert known > 0


def test_exact_lists():
    n = 10
    t = Trace()
    a = t.drain(0, 0, n, [], n)                      # a new bus: known and empty
    t.sparse([3, 7])
    b = t.drain(1, 0, n, [3, 7], n)                  # the sparse launch's mailboxes
    c = t.drain(2, 0, n, [], n)                      # ... emptied by that drain
    # a ticket's removal is skipped for a mailbox a later launch refilled
    t.sparse([3])
    t.begin(3, 0, n)
    t.sparse([3, 4])
    t.end(3, [3], n)
    d = t.drain(4, 0, n, [3, 4], n)
    # a cut leaves the remainder
    t.sparse([1, 2, 5])
    e = t.drain(5, 0, n, [1], 1)
    f = t.drain(6, 0, n, [2, 5], n)
    # a take empties only the take set
    t.sparse([6])
    g = t.drain(7, 0, n, [6], n, take=True)
    h = t.begin(8, 0, n, take=True)
    t.end(8, [], n)
    i = t.drain(9, 0, n, [6], n)
    # a full launch makes both unknown; a drain of part of the range does not make them known
    t.full()
    j = t.drain(10, 0, n - 1, [0, 8], n - 1)
    k = t.drain(11, 0, n, [9], n)                    # the whole range: known again
    l_ = t.drain(12, 0, n, [], n)
    # a drain begun before a full launch and ended after it does not make the sets known
    t.begin(13, 0, n)
    t.full()
    t.end(13, [], n)
    m = t.drain(14, 0, n, [4], n)
    # release drops the released mailboxes; consume_all empties everything
    t.sparse([4, 5, 8])
    t.release([4])
    o = t.drain(15, 2, 6, [5], 6)                    # only the range's candidates, from an inner range
    t.full()
    t.consume_all()
    p = t.drain(16, 0, n, [], n)
    t.sparse([7])
    q = t.drain(17, 0, n, [7], n)
    rc, res = t.run(n)
    assert rc == 0
    assert res[a] == [] and res[b] == [3, 7] and res[c] == []
    assert res[d] == [3, 4]
    assert res[e] == [1, 2, 5] and res[f] == [2, 5]
    assert res[g] == [6] and res[h] == [] and res[i] == [6]
    assert res[j] == DENSE and res[k] == DENSE and res[l_] == []
    assert res[m] == DENSE
    assert res[o] == [5]
    assert res[p] == [] and res[q] == [7]


def test_caps():
    n = 64
    t = Trace()
    t.sparse([1, 2, 3])
    a = t.drain(0, 0, n, [1, 2, 3], n)              # 3 candidates > list_cap 2: dense, and known again after it
    t.sparse([4, 5])
    b = t.drain(1, 0, n, [4, 5], n)
    t.sparse(list(range(10, 19)))                    # 9 > 4 * list_cap: the set is dropped
    c = t.drain(2, 0, n, list(range(10, 19)), n)
    d = t.drain(3, 0, n, [], n)
    rc, res = t.run(n, list_cap=2)
    assert rc == 0
    assert res[a] == DENSE and res[b] == [4, 5] and res[c] == DENSE and res[d] == []


def test_refusals():
    t = Trace()
    t.end(0, [], 1)
    assert t.run(4)[0] == nat.ENOENT
    t = Trace()
    t.begin(0, 0, 4)
    t.begin(0, 0, 4)
    assert t.run(4)[0] == nat.EINVAL
    t = Trace()
    t.begin(0, 2, 3)
    assert t.run(4)[0] == nat.EINVAL
    t = Trace()
    t.sparse([4])
    assert t.run(4)[0] == nat.EINVAL
    assert Trace().run(4, list_cap=0)[0] == nat.EINVAL
