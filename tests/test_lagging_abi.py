"""C-ABI of the consumer backlog queries (cpbus_lagging, cpbus_blockers and their group twins) without a GPU: exports,
layouts, bindings and a plain-C99 caller; and the oracle's side of both questions (orc_backlog, orc_blockers in
tests/c/lag_oracle.c, built on the oracle's own rules) against an independent Python model on seeded traces with pairs,
unicast sends, periodic and one-shot timers and a mailbox capacity.
The queries themselves need a bus, hence a GPU: tests/test_gpu_lagging.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lag_oracle as lo
import oracle_binding as ob
from containerpilot_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("cpbus_lagging", "cpbus_blockers", "cpbus_group_lagging", "cpbus_group_blockers")


def test_library_exports_the_four_entry_points_with_their_layouts():
    lib = C.CDLL(nat.LIB_PATH)
    for name in NEW:
        assert hasattr(lib, name), name
        assert name in nat.SYMBOLS, name

    class Lag(C.Structure):   # cpbus_lag, as the header declares it
        _fields_ = [("sub_id", C.c_uint32), ("backlog", C.c_uint32), ("lost", C.c_uint64)]

    assert C.sizeof(Lag) == 16 == nat.LAG_DTYPE.itemsize
    assert [f[0] for f in Lag._fields_] == list(nat.LAG_DTYPE.names)
    assert C.sizeof(nat.LagSummary) == 38 * 8
    assert nat.SYMBOLS["cpbus_group_lagging"] == nat.SYMBOLS["cpbus_lagging"]
    assert nat.SYMBOLS["cpbus_group_blockers"] == nat.SYMBOLS["cpbus_blockers"]
    lib = nat.load()
    n, nxt = C.c_size_t(), C.c_uint32()
    assert lib.cpbus_lagging(None, 0, 1, 0, 1, None, 0, C.byref(n), C.byref(nxt), None) == nat.EINVAL
    assert lib.cpbus_blockers(None, None, 0, C.byref(n)) == nat.EINVAL
    assert lib.cpbus_abi_version() == 2


def test_lag_declarations_from_plain_c99(tmp_path):
    exe = str(tmp_path / "lag_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "lag_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr


class CapModel:
    """Mailboxes of capacity `cap` that block the sender when full (events/subscriber.go:30-32), written from the Go
    semantics: Publish is refused as a whole when one wanting mailbox is full, a timer's send blocks on its own mailbox.
    Blocking is answered by arithmetic (ticks due + the record against the free room), not by a walk."""

    def __init__(self, cap, K):
        self.cap, self.K, self.now, self.subs = cap, K, 0, []

    def subscribe(self, mask, pairs=()):
        self.subs.append({"on": True, "mask": mask, "pairs": set(pairs), "held": 0, "timers": [None] * self.K})

    def unsubscribe(self, s):
        self.subs[s]["on"] = False
        self.subs[s]["timers"] = [None] * self.K

    def _wants(self, sub, code, src, target, s):
        if target != nat.TARGET_ALL:
            return target == s
        return bool((sub["mask"] >> code) & 1) or (code, src) in sub["pairs"]

    def publish(self, code, src):
        live = [u for u in self.subs if u["on"] and self._wants(u, code, src, nat.TARGET_ALL, -1)]
        if any(u["held"] >= self.cap for u in live):
            return ob.EAGAIN
        for u in live:
            u["held"] += 1
        return 0

    def receive(self, s, code, src):
        u = self.subs[s]
        if u["held"] >= self.cap:
            return ob.EAGAIN
        u["held"] += 1
        return 0

    def timer_add(self, s, period, oneshot):
        slots = self.subs[s]["timers"]
        k = slots.index(None)
        slots[k] = {"due": self.now + period, "period": period, "oneshot": oneshot}

    def advance(self, t):
        for u in self.subs:   # subscriber by subscriber, each one's firings oldest first (the oracle's order)
            while True:
                due = [(tm["due"], k) for k, tm in enumerate(u["timers"]) if tm is not None and tm["due"] <= t]
                if not due:
                    break
                if u["held"] >= self.cap:
                    return ob.EAGAIN
                k = min(due)[1]
                u["held"] += 1
                if u["timers"][k]["oneshot"]:
                    u["timers"][k] = None
                else:
                    u["timers"][k]["due"] += u["timers"][k]["period"]
        self.now = t
        return 0

    def consume(self, s, n):
        u = self.subs[s]
        u["held"] -= min(n, u["held"])

    def ticks_due(self, u, t):
        n = 0
        for tm in u["timers"]:
            if tm is not None and tm["due"] <= t:
                n += 1 if tm["oneshot"] else (t - tm["due"]) // tm["period"] + 1
        return n

    def blockers(self, t, code=None, src=0, target=nat.TARGET_ALL):
        out = []
        for s, u in enumerate(self.subs):
            if not u["on"]:
                continue
            want = code is not None and self._wants(u, code, src, target, s)
            if self.ticks_due(u, t) + int(want) > self.cap - u["held"]:
                out.append(s)
        return out


@pytest.mark.parametrize("seed", [1, 2, 3, 4, 5])
def test_oracle_blockers_and_backlog_agree_with_an_independent_model(seed):
    rng = np.random.default_rng(1000 + seed)
    N, K, CAP = 10, 2, 6
    orc, mod = ob.Oracle(N, timers_per_sub=K, keep_window=0, mailbox_cap=CAP), CapModel(CAP, K)
    for s in range(N):
        mask = int(rng.integers(0, 1 << 6)) if s % 3 else nat.MASK_ALL
        pairs = [(int(rng.integers(0, 6)), int(rng.integers(0, 4))) for _ in range(int(rng.integers(0, 3)))] if s % 2 else []
        if s == N - 1:
            mask = 0   # an implicit timer-only mailbox
        orc.subscribe(mask, pairs=pairs)
        mod.subscribe(mask, pairs)
    checked = blocked_seen = 0
    for step in range(400):
        op = rng.random()
        if op < 0.35:
            code, src = int(rng.integers(0, 7)), int(rng.integers(0, 4))
            assert orc.publish(code, src) == mod.publish(code, src)
        elif op < 0.5:
            s, code = int(rng.integers(0, N)), int(rng.integers(0, 7))
            if mod.subs[s]["on"]:
                assert orc.receive(s, code, 0) == mod.receive(s, code, 0)
        elif op < 0.6:
            s = int(rng.integers(0, N))
            if mod.subs[s]["on"] and None in mod.subs[s]["timers"]:
                period, oneshot = int(rng.integers(50, 400)), bool(rng.random() < 0.3)
                orc.timer_add(s, period, 7, oneshot)
                mod.timer_add(s, period, oneshot)
        elif op < 0.75:
            t = mod.now + int(rng.integers(0, 300))
            assert orc.advance(t) == mod.advance(t)
        elif op < 0.95:
            s, take = int(rng.integers(0, N)), int(rng.integers(1, CAP + 1))
            orc.consume(s, take)
            mod.consume(s, take)
        elif step > 200:
            s = int(rng.integers(0, N - 1))
            if mod.subs[s]["on"]:
                assert orc.unsubscribe(s) == 0
                mod.unsubscribe(s)
        for s in range(N):
            assert lo.backlog(orc, s) == min(mod.subs[s]["held"], CAP), (step, s)
        t = mod.now + int(rng.integers(0, 200))
        probes = [(None, 0, nat.TARGET_ALL), (int(rng.integers(0, 7)), int(rng.integers(0, 4)), nat.TARGET_ALL),
                  (int(rng.integers(0, 7)), 0, int(rng.integers(0, N)))]
        for code, src, target in probes:
            want = mod.blockers(t, code, src, target)
            got = lo.blockers(orc, t, code, src, target)
            assert got.tolist() == want, (step, code, target, got, want)
            checked += 1
            blocked_seen += len(want) > 0
    assert checked == 1200 and blocked_seen > 100


def test_oracle_backlog_is_capped_by_the_ring_and_unbounded_mailboxes_never_block():
    orc = ob.Oracle(2, timers_per_sub=1, keep_window=0)
    orc.subscribe(nat.MASK_ALL)
    orc.subscribe(0)
    orc.timer_add(1, 10, 0)
    for i in range(50):
        orc.publish(1, i)
    assert lo.backlog(orc, 0) == 50 and lo.backlog(orc, 1) == 0
    assert lo.blockers(orc, 10_000, 1).tolist() == []
    capped = ob.Oracle(1, keep_window=0, mailbox_cap=4)
    capped.subscribe(nat.MASK_ALL)
    for i in range(4):
        assert capped.publish(1, i) == 0
    assert capped.publish(1, 9) == ob.EAGAIN and lo.backlog(capped, 0) == 4
    assert lo.blockers(capped, 0, 1).tolist() == [0] and lo.blockers(capped, 0).tolist() == []
    capped.consume(0, 1)
    assert lo.backlog(capped, 0) == 3 and lo.blockers(capped, 0, 1).tolist() == []
