"""Subscriber id reuse (cpbus_release_many, cpbus_subscribe_list and their group twins) without a GPU: the exports and
declarations, a plain-C99 caller, the argument checks, which return before the bus or a device is looked at, and the oracle's
reuse extension (tests/c/reuse_oracle.c) against a Python model of file-descriptor-style ids.  The calls themselves need a
GPU: tests/test_gpu_subscriber_reuse.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import oracle_binding as ob
import reuse_oracle as ro
from containerpilot_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ("release_many", "subscribe_list")


def test_exports_and_declarations():
    lib = C.CDLL(nat.LIB_PATH)
    hdr = open(os.path.join(ROOT, "include", "cpbus.h")).read()
    for name in CALLS:
        for full in (f"cpbus_{name}", f"cpbus_group_{name}"):
            assert hasattr(lib, full) and full in nat.SYMBOLS
            assert re.search(r"\bint " + full + r"\(", hdr), full
    assert nat.load().cpbus_abi_version() == 2


def _fake():
    """a zeroed stand-in handle: every check below returns before the handle is read"""
    fake = C.create_string_buffer(4096)
    return fake, C.c_void_p(C.addressof(fake))


@pytest.mark.parametrize("group", [False, True])
def test_release_many_argument_checks(group):
    fn = getattr(nat.load(), "cpbus_group_release_many" if group else "cpbus_release_many")
    ids = np.arange(4, dtype=np.uint32)
    status = np.full(4, 99, dtype=np.int32)
    applied = C.c_uint32(7)
    fake, handle = _fake()
    for n in (4, 0):
        assert fn(None, ids.ctypes.data, n, status.ctypes.data, C.byref(applied)) == nat.EINVAL
    assert fn(handle, None, 4, status.ctypes.data, C.byref(applied)) == nat.EINVAL
    assert (status == 99).all() and applied.value == 7
    assert fn(handle, None, 0, status.ctypes.data, C.byref(applied)) == nat.OK       # n == 0: the bus is not read
    assert (status == 99).all() and applied.value == 0
    assert fn(handle, None, 0, None, None) == nat.OK
    assert not any(fake.raw), "the handle was written"


@pytest.mark.parametrize("group", [False, True])
def test_subscribe_list_argument_checks(group):
    """The checks of cpbus_subscribe_pairs_many, with NULL pairs / n_pairs meaning no cases; sub_ids is left alone"""
    fn = getattr(nat.load(), "cpbus_group_subscribe_list" if group else "cpbus_subscribe_list")
    masks = np.full(2, nat.MASK_ALL, dtype=np.uint32)
    rows = np.zeros((2, 16, 2), dtype=np.uint32)
    out = np.full(2, 5, dtype=np.uint32)
    fake, handle = _fake()
    p = lambda a: a.ctypes.data  # noqa: E731

    def call(h, pairs, n_pairs, n=2, sub_ids=p(out)):
        return fn(h, p(masks), pairs, n_pairs, n, sub_ids)

    assert call(None, None, None) == nat.EINVAL
    assert call(handle, None, None, n=0) == nat.EINVAL                                  # n == 0, as subscribe_many
    assert call(handle, None, None, sub_ids=None) == nat.EINVAL
    assert call(handle, None, p(np.array([1, 0], dtype=np.uint32))) == nat.EINVAL       # n_pairs without pairs
    assert call(handle, p(rows), p(np.array([17, 0], dtype=np.uint32))) == nat.EINVAL   # > CPBUS_MAX_PAIRS
    rows[1, 0, 0] = 17
    assert call(handle, p(rows), p(np.array([0, 1], dtype=np.uint32))) == nat.EINVAL    # a case's code out of range
    assert (out == 5).all() and not any(fake.raw)


def test_reuse_declarations_from_plain_c99(tmp_path):
    exe = str(tmp_path / "reuse_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "reuse_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "PASS" in r.stdout, r.stdout + r.stderr


class _Model:
    """File-descriptor-style ids in plain Python: live / closed / released slots, lowest free id first, and how many
    broadcast records each slot holds"""

    def __init__(self, n_max):
        self.n_max, self.state, self.mask, self.count = n_max, [], [], []

    def free(self):
        return [i for i, s in enumerate(self.state) if s == "released"] + list(range(len(self.state), self.n_max))

    def subscribe_list(self, masks):
        free = self.free()
        if len(free) < len(masks):
            return ob.ENOSPC, []
        ids = free[:len(masks)]
        for i, m in zip(ids, masks):
            if i == len(self.state):
                self.state.append(None); self.mask.append(0); self.count.append(0)
            self.state[i], self.mask[i], self.count[i] = "live", m, 0
        return 0, ids

    def unsubscribe(self, i):
        if i >= len(self.state) or self.state[i] == "released":
            return ob.ENOENT
        if self.state[i] == "closed":
            return ob.ECLOSED
        self.state[i] = "closed"
        return 0

    def release(self, i):
        if i >= len(self.state) or self.state[i] == "released":
            return ob.ENOENT
        if self.state[i] == "live":
            return ro.EINVAL
        self.state[i], self.mask[i], self.count[i] = "released", 0, 0
        return 0

    def publish(self, code):
        for i, s in enumerate(self.state):
            if s == "live" and (self.mask[i] >> code) & 1:
                self.count[i] += 1

    def send(self, i):
        if i >= len(self.state) or self.state[i] == "released":
            return ob.ENOENT
        if self.state[i] == "closed":
            return ob.ECLOSED
        self.count[i] += 1
        return 0


@pytest.mark.parametrize("seed", range(6))
def test_reuse_oracle_against_python_model(seed):
    """Seeded traces of subscribe_list, unsubscribe, release (repeats, live and never-issued ids), publishes and sends: the
    oracle extension hands out the ids the model does, refuses what it refuses and holds the records it counts"""
    rng = np.random.default_rng(seed)
    n_max = 24
    orc, model = ro.ReuseOracle(n_max, keep_window=0), _Model(n_max)
    for step in range(600):
        r = rng.random()
        hw = len(model.state)
        if r < 0.15:
            masks = [int(rng.integers(0, 1 << 17)) for _ in range(int(rng.integers(1, 6)))]
            assert orc.subscribe_list(masks) == model.subscribe_list(masks), step
        elif r < 0.3 and hw:
            i = int(rng.integers(0, hw + 2))
            assert orc.unsubscribe(i) == model.unsubscribe(i), step
        elif r < 0.45:
            ids = [int(rng.integers(0, hw + 3)) for _ in range(int(rng.integers(1, 5)))]
            ids += ids[:int(rng.integers(0, 2))]
            assert orc.release_many(ids) == [model.release(i) for i in ids], step
        elif r < 0.6 and hw:
            i = int(rng.integers(0, hw + 1))
            assert orc.receive(i, 3, 1) == model.send(i), step
        else:
            code = int(rng.integers(0, 17))
            assert orc.publish(code, 0) == 0
            model.publish(code)
        assert orc.high_water() == len(model.state) <= n_max
        for i in range(len(model.state)):
            assert orc.count(i) == model.count[i], (step, i)
            assert orc.released(i) == (model.state[i] == "released")
            assert len(orc.mailbox(i)) == model.count[i]
