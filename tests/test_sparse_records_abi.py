"""Sparse record delivery (CPBUS_CFG_SPARSE_RECORDS) without a GPU: the flag and the plan export, a plain-C99 caller,
cpbus_create's and the group's refusal of the flag, and the plan (cpbus_sparse_plan, the bus's own planning code) against
a model built on tests/py_model.py's delivery rule on seeded fleets: code masks, exact cases, unsubscribed and mask-0
mailboxes, unicast records and due timer slots, and flushes of due ticks alone.  It gives up exactly at the caps.
The bus itself needs a GPU: tests/test_gpu_sparse_records.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from containerpilot_b200 import _native as nat
from py_model import PyBus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EVENT_DTYPE = np.dtype([("seq", "<u8"), ("ts_ns", "<u8"), ("code", "<u4"), ("source_id", "<u4"),
                        ("target", "<u4"), ("flags", "<u4")])


def test_flag_and_export():
    lib = C.CDLL(nat.LIB_PATH)
    assert hasattr(lib, "cpbus_sparse_plan") and "cpbus_sparse_plan" in nat.SYMBOLS
    others = nat.CFG_LOSSLESS | nat.CFG_DIGEST | nat.CFG_SPARSE_TICKS
    assert nat.CFG_SPARSE_RECORDS == 0x8 and not nat.CFG_SPARSE_RECORDS & others
    hdr = open(os.path.join(ROOT, "include", "cpbus.h")).read()
    assert "#define CPBUS_CFG_SPARSE_RECORDS 0x8u" in hdr
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
    h = C.c_void_p()
    assert lib.cpbus_create(C.byref(_cfg(nat.CFG_SPARSE_RECORDS | lossless)), C.byref(h)) == nat.EINVAL
    assert not h.value


def test_group_refuses_the_flag():
    lib = nat.load()
    devs = (C.c_int32 * 2)(0, 0)
    for flags in (nat.CFG_SPARSE_RECORDS, nat.CFG_SPARSE_RECORDS | nat.CFG_SPARSE_TICKS):
        h = C.c_void_p()
        assert lib.cpbus_group_create(C.byref(_cfg(flags | nat.CFG_LOSSLESS)), devs, 2, C.byref(h)) == nat.EINVAL
        assert not h.value


def test_sparse_records_declarations_from_plain_c99(tmp_path):
    exe = str(tmp_path / "sparse_records_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "sparse_records_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr


def plan(masks, active, pairs, base, rec, due, K, max_m, max_d):
    """cpbus_sparse_plan: (status, [(local, due_bits, [record indices])])"""
    lib = nat.load()
    n = len(masks)
    masks = np.ascontiguousarray(masks, dtype=np.uint32)
    active = np.ascontiguousarray(active, dtype=np.uint8)
    prow = np.zeros((max(n, 1), 16, 2), dtype=np.uint32)
    npairs = np.zeros(max(n, 1), dtype=np.uint32)
    for l, cases in enumerate(pairs):
        npairs[l] = len(cases)
        for j, (c, s) in enumerate(cases[:16]):
            prow[l, j] = (c, s)
    due = np.ascontiguousarray(due, dtype=np.uint32)
    no, ni = C.c_size_t(), C.c_size_t()
    args = (masks.ctypes.data, active.ctypes.data, n, prow.ctypes.data, npairs.ctypes.data, base,
            rec.ctypes.data if len(rec) else None, len(rec), due.ctypes.data if len(due) else None, len(due), K, max_m, max_d)
    rc = lib.cpbus_sparse_plan(*args, None, 0, None, 0, C.byref(no), C.byref(ni))
    if rc:
        return rc, None
    out = np.zeros(max(1, no.value), dtype=nat.PLAN_ENTRY_DTYPE)
    idx = np.zeros(max(1, ni.value), dtype=np.uint32)
    nat.check(lib.cpbus_sparse_plan(*args, out.ctypes.data, no.value, idx.ctypes.data, ni.value, C.byref(no), C.byref(ni)),
              "cpbus_sparse_plan")
    return 0, [(int(e["local"]), int(e["due_bits"]), [int(i) for i in idx[e["first"]: e["first"] + e["count"]]])
               for e in out[: no.value]]


def model(masks, active, pairs, base, rec, due, K):
    """who takes what, by py_model's rule: a PyBus with the same subscribers receives the records one by one (record i
    is the one with seq i); a due slot makes its subscriber a candidate"""
    bus = PyBus()
    for l, m in enumerate(masks):
        bus.subscribe(int(m), pairs[l])
    for l, a in enumerate(active):
        if not a:
            bus.unsubscribe(l)
    for r in rec:
        t = int(r["target"])
        if t == nat.TARGET_ALL:
            bus.publish(int(r["code"]), int(r["source_id"]))
        elif base <= t < base + len(masks) and active[t - base]:
            bus.receive(t - base, int(r["code"]), int(r["source_id"]))
        else:
            bus.seq += 1   # a unicast record nobody takes
    took = {l: [x[0] for x in s["box"]] for l, s in enumerate(bus.subs) if s["box"]}
    bits = {}
    for slot in due:
        bits[slot // K] = bits.get(slot // K, 0) | 1 << (slot % K)
    return [(l, bits.get(l, 0), took.get(l, [])) for l in sorted(set(took) | set(bits))]


def fleet(rng, n, n_rec, K, max_due=11):
    """a seeded fleet: all-ones, sparse and mask-0 subscribers, some with exact cases, a share unsubscribed; a batch of
    broadcast records (a few out-of-range codes) and unicast sends (some to unsubscribed or foreign ids); up to max_due
    due slots"""
    kind = rng.random(n)
    masks = np.where(kind < 0.1, nat.MASK_ALL, np.where(kind < 0.3, 0, 1 << rng.integers(0, 17, n))).astype(np.uint32)
    masks |= np.where(rng.random(n) < 0.3, 1 << rng.integers(0, 17, n), 0).astype(np.uint32)
    active = (rng.random(n) > 0.15).astype(np.uint8)
    srcs = int(rng.integers(2, 12))
    pairs = [[(int(rng.integers(0, 17)), int(rng.integers(0, srcs))) for _ in range(int(rng.integers(1, 17)))]
             if rng.random() < 0.4 else [] for _ in range(n)]
    base = int(rng.integers(0, 1000))
    rec = np.zeros(n_rec, dtype=EVENT_DTYPE)
    rec["seq"] = np.arange(n_rec)
    rec["ts_ns"] = np.sort(rng.integers(0, 10 ** 6, n_rec))
    rec["code"] = np.where(rng.random(n_rec) < 0.03, 17 + rng.integers(0, 5, n_rec), rng.integers(0, 17, n_rec))
    rec["source_id"] = rng.integers(0, srcs, n_rec)
    uni = rng.random(n_rec) < 0.2
    rec["target"] = np.where(uni, base + rng.integers(0, n + 3, n_rec), nat.TARGET_ALL)
    rec["flags"] = np.where(uni, nat.F_UNICAST, 0)
    due = rng.choice(n * K, size=min(n * K, int(rng.integers(0, max_due + 1))), replace=False).tolist() if K else []
    return masks, active, pairs, base, rec, due


@pytest.mark.parametrize("seed", range(400))
def test_plan_against_the_delivery_rule(seed):
    rng = np.random.default_rng(seed)
    K = [0, 1, 2, 4, 8][seed % 5]
    n = int(rng.integers(1, 90))
    if seed % 4 == 3:   # a flush of due ticks alone, up to every slot of the fleet
        masks, active, pairs, base, rec, due = fleet(rng, n, 0, K, max_due=n * K)
    else:
        masks, active, pairs, base, rec, due = fleet(rng, n, int(rng.integers(0, 64)), K)
    want = model(masks, active, pairs, base, rec, due, K)
    n_cand, n_deliv = len(want), sum(len(r) for _, _, r in want)
    max_m = max(n_cand, len(due), 1)
    rc, got = plan(masks, active, pairs, base, rec, due, K, max_m, n_deliv)
    assert rc == nat.OK and got == want
    if not len(rec):                      # one entry per due mailbox, ascending, with its due-slot bits and no record
        bits = {}
        for slot in due:
            bits[slot // K] = bits.get(slot // K, 0) | 1 << (slot % K)
        assert got == [(l, bits[l], []) for l in sorted(bits)]
    assert plan(masks, active, pairs, base, rec, due, K, max_m + 1 + seed % 7, n_deliv + seed % 3) == (nat.OK, want)
    # one mailbox fewer than needed: the full fan-out.  The cap counts due slots as well as mailboxes, so without records
    # (max_m = len(due) >= n_cand) this pins the due-slot cap, the one the bus's due index applies before it plans
    if n_cand > 1 or len(due) > 1:
        assert plan(masks, active, pairs, base, rec, due, K, max_m - 1, n_deliv)[0] == nat.ENOSPC
    if n_deliv:                           # one record fewer than needed
        assert plan(masks, active, pairs, base, rec, due, K, max_m, n_deliv - 1)[0] == nat.ENOSPC


def test_dense_code_ends_planning():
    """an all-ones fleet: the first broadcast record's code has more subscribers than the cap"""
    n = 4096
    masks = np.full(n, nat.MASK_ALL, dtype=np.uint32)
    rec = np.zeros(3, dtype=EVENT_DTYPE)
    rec["code"], rec["target"] = 3, nat.TARGET_ALL
    args = (masks, np.ones(n, np.uint8), [[] for _ in range(n)], 0, rec, [], 1)
    assert plan(*args, 4095, 10 ** 6)[0] == nat.ENOSPC
    assert plan(*args, 4096, 3 * 4096)[0] == nat.OK
    assert plan(*args, 4096, 3 * 4096 - 1)[0] == nat.ENOSPC


def test_bad_arguments():
    rec = np.zeros(1, dtype=EVENT_DTYPE)
    rec["target"] = nat.TARGET_ALL
    masks, active, pairs = np.ones(4, np.uint32), np.ones(4, np.uint8), [[]] * 4
    assert plan(masks, active, pairs, 0, rec, [], 3, 32, 32)[0] == nat.EINVAL        # K = 3
    assert plan(masks, active, pairs, 0, rec, [1], 0, 32, 32)[0] == nat.EINVAL       # due slots without timers
    assert plan(masks, active, pairs, 0, rec, [8], 2, 32, 32)[0] == nat.EINVAL       # slot of subscriber 4 of 4
    assert plan(masks, active, [[(1, 1)] * 17] + [[]] * 3, 0, rec, [], 1, 32, 32)[0] == nat.EINVAL   # 17 cases
