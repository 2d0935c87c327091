"""Sparse timer delivery (CPBUS_CFG_SPARSE_TICKS) without a GPU: the flag and the due-index export, a plain-C99 caller, the
group's refusal of the flag, and the host due index (cpbus_due_trace) against an independent Python model of Go timers on
seeded arm / cancel / unsubscribe / launch traces: periods near 2^64, one-shots, slots re-armed over and over (stale heap
entries) and launches that find most of the table due (the index's one-pass path).
The bus itself needs a GPU: tests/test_gpu_sparse_ticks.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from containerpilot_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDLE = (1 << 64) - 1   # "never"


def test_flag_and_export():
    lib = C.CDLL(nat.LIB_PATH)
    assert hasattr(lib, "cpbus_due_trace") and "cpbus_due_trace" in nat.SYMBOLS
    assert nat.CFG_SPARSE_TICKS == 0x4 and not nat.CFG_SPARSE_TICKS & (nat.CFG_LOSSLESS | nat.CFG_DIGEST)
    hdr = open(os.path.join(ROOT, "include", "cpbus.h")).read()
    assert "#define CPBUS_CFG_SPARSE_TICKS 0x4u" in hdr
    assert nat.load().cpbus_abi_version() == 2


def test_group_refuses_the_flag():
    lib = nat.load()
    cfg = nat.Config()
    cfg.n_max_subs, cfg.ring_cap, cfg.batch_cap, cfg.timers_per_sub, cfg.device = 64, 1024, 256, 1, -1
    cfg.flags = nat.CFG_SPARSE_TICKS | nat.CFG_LOSSLESS
    devs = (C.c_int32 * 2)(0, 0)
    h = C.c_void_p()
    assert lib.cpbus_group_create(C.byref(cfg), devs, 2, C.byref(h)) == nat.EINVAL
    assert not h.value


def test_sparse_declarations_from_plain_c99(tmp_path):
    exe = str(tmp_path / "sparse_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "sparse_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr


def trace(ops, n_slots, K):
    lib = nat.load()
    a = np.zeros(len(ops), dtype=nat.DUE_OP_DTYPE)
    for i, (kind, slot, value) in enumerate(ops):
        a[i] = (kind, slot, value)
    n = C.c_size_t()
    rc = lib.cpbus_due_trace(a.ctypes.data if len(a) else None, len(a), n_slots, K, None, 0, C.byref(n))
    if rc:
        return rc, None
    out = np.zeros(max(1, n.value), dtype=nat.DUE_FIRE_DTYPE)
    nat.check(lib.cpbus_due_trace(a.ctypes.data if len(a) else None, len(a), n_slots, K, out.ctypes.data, n.value, C.byref(n)),
              "cpbus_due_trace")
    return 0, [(int(f["launch"]), int(f["slot"]), int(f["ticks"]), int(f["next_due"])) for f in out[: n.value]]


class TimerModel:
    """Go timers (events/timer.go:12-71) on a virtual clock: a periodic timer armed at t fires at t + p, t + 2p, ...; a
    one-shot once at t + p.  A firing at or past 2^64 - 1 never comes.  A launch to w delivers every firing <= w."""

    def __init__(self, n_slots, K):
        self.K, self.clock, self.timers = K, 0, {}
        self.n_slots = n_slots

    def arm(self, slot, period, oneshot):
        self.timers[slot] = [self.clock + period, period, oneshot]

    def disarm(self, slot):
        self.timers.pop(slot, None)

    def launch(self, w, ordinal):
        out = []
        for slot in sorted(self.timers):
            due, period, oneshot = self.timers[slot]
            if due >= IDLE or due > w:
                continue
            if oneshot:
                out.append((ordinal, slot, 1, IDLE))
                del self.timers[slot]
                continue
            ticks = (min(w, IDLE - 1) - due) // period + 1   # firings due, due + p, ... that are <= w and come at all
            nxt = due + ticks * period
            nxt = nxt if nxt < IDLE else IDLE
            out.append((ordinal, slot, ticks, nxt))
            self.timers[slot][0] = nxt
        return out


def random_trace(seed, n_subs, K, n_ops):
    rng = np.random.default_rng(seed)
    n_slots = n_subs * K
    ops, clock, last = [], 0, 0
    if seed % 3 == 0:   # start near the top of the clock
        clock = last = IDLE - int(rng.integers(1, 1 << 40))
        ops.append((nat.DUE_CLOCK, 0, clock))
    for _ in range(n_ops):
        r = rng.random()
        if r < 0.40:
            slot = int(rng.integers(0, n_slots))
            kind = nat.DUE_ONESHOT if rng.random() < 0.25 else nat.DUE_ARM
            q = rng.random()
            if q < 0.75:
                period = int(rng.integers(1, 5000))
            elif q < 0.85:
                period = IDLE - int(rng.integers(0, 1 << 20))           # near 2^64: saturates to "never"
            elif q < 0.95:
                period = max(1, IDLE - clock - int(rng.integers(0, 20_000)))   # first due just short of (or at) the top
            else:
                period = 1 << 63
            ops.append((kind, slot, period))
        elif r < 0.50:
            ops.append((nat.DUE_DISARM, int(rng.integers(0, n_slots)), 0))
        elif r < 0.55:
            ops.append((nat.DUE_UNSUB, int(rng.integers(0, n_subs)), 0))
        else:
            step = int(rng.integers(0, 20_000)) if rng.random() < 0.9 else int(rng.integers(0, 200_000))
            clock = min(IDLE, clock + step)
            w = clock if rng.random() < 0.8 else last + int(rng.integers(0, clock - last + 1))
            last = w
            ops.append((nat.DUE_LAUNCH, 0, w))
            ops.append((nat.DUE_CLOCK, 0, clock))
    return ops, n_slots


def run_model(ops, n_slots, K):
    m, launches, out = TimerModel(n_slots, K), 0, []
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
        else:
            out += m.launch(value, launches)
            launches += 1
    return out


@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("seed", range(6))
def test_due_index_matches_the_model(K, seed):
    ops, n_slots = random_trace(1000 * K + seed, 16, K, 600)
    rc, got = trace(ops, n_slots, K)
    assert rc == 0
    assert got == run_model(ops, n_slots, K)


@pytest.mark.parametrize("seed", range(3))
def test_dense_launches_take_the_one_pass_path(seed):
    """Most of a 4,096-slot table due at once (more than the index pops one by one), mixed with sparse launches."""
    rng = np.random.default_rng(seed)
    K, n_subs = 4, 1024
    n_slots = n_subs * K
    ops = []
    for s in range(n_slots):
        if rng.random() < 0.9:
            ops.append((nat.DUE_ONESHOT if rng.random() < 0.1 else nat.DUE_ARM, s, int(rng.integers(1, 1000))))
    clock = 0
    for i in range(40):
        clock += int(rng.integers(1, 3000)) if i % 4 else 1
        if i % 7 == 3:
            ops.append((nat.DUE_DISARM, int(rng.integers(0, n_slots)), 0))
            ops.append((nat.DUE_UNSUB, int(rng.integers(0, n_subs)), 0))
        ops.append((nat.DUE_LAUNCH, 0, clock))
        ops.append((nat.DUE_CLOCK, 0, clock))
        ops.append((nat.DUE_ARM, int(rng.integers(0, n_slots)), int(rng.integers(1, 1000))))
    rc, got = trace(ops, n_slots, K)
    assert rc == 0
    assert got == run_model(ops, n_slots, K)
    assert max(sum(1 for f in got if f[0] == q) for q in range(40)) > n_slots // 2


def test_generation_reuse_never_fires_a_stale_entry():
    """One slot re-armed and cancelled many times between launches: only its current arming fires."""
    ops = []
    for i in range(200):
        ops.append((nat.DUE_ARM if i % 2 else nat.DUE_ONESHOT, 3, 1 + i % 5))
        if i % 3:
            ops.append((nat.DUE_DISARM, 3, 0))
    ops += [(nat.DUE_ARM, 3, 7), (nat.DUE_LAUNCH, 0, 100), (nat.DUE_CLOCK, 0, 100), (nat.DUE_LAUNCH, 0, 104)]
    rc, got = trace(ops, 8, 1)
    assert rc == 0 and got == run_model(ops, 8, 1)
    assert got == [(0, 3, 14, 105)]   # 7, 14, ..., 98; nothing of the earlier armings, and nothing due by 104


def test_trace_rejects_bad_ops():
    assert trace([(nat.DUE_ARM, 8, 5)], 8, 1)[0] == nat.EINVAL                       # slot out of range
    assert trace([(nat.DUE_ARM, 0, 0)], 8, 1)[0] == nat.EINVAL                       # period 0
    assert trace([(nat.DUE_UNSUB, 4, 0)], 8, 2)[0] == nat.EINVAL                     # subscriber 4 of 4
    assert trace([(nat.DUE_LAUNCH, 0, 9), (nat.DUE_LAUNCH, 0, 8)], 8, 1)[0] == nat.EINVAL   # launch behind the previous one
    assert trace([(9, 0, 0)], 8, 1)[0] == nat.EINVAL
    assert trace([], 8, 3)[0] == nat.EINVAL
