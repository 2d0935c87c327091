"""Acknowledged drains (cpbus_take_ready, cpbus_ack_many and their group twins) without a GPU: the exports and declarations,
a plain-C99 caller, and the argument checks, which return before the bus or a device is looked at.  The calls themselves
need a GPU: tests/test_gpu_take_ack.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import EVENT_DTYPE, READY_DTYPE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ("take_ready", "ack_many")


def test_exports_and_declarations():
    lib = C.CDLL(nat.LIB_PATH)
    hdr = open(os.path.join(ROOT, "include", "cpbus.h")).read()
    for name in CALLS:
        assert name in nat.GROUP_CALLS
        for full in (f"cpbus_{name}", f"cpbus_group_{name}"):
            assert hasattr(lib, full) and full in nat.SYMBOLS
            assert re.search(r"\bint " + full + r"\(", hdr), full
    assert nat.SYMBOLS["cpbus_take_ready"][1] == nat.SYMBOLS["cpbus_drain_ready"][1]
    assert nat.load().cpbus_abi_version() == 2


def _fake_handle():
    fake = C.create_string_buffer(4096)
    return fake, C.c_void_p(C.addressof(fake))


@pytest.mark.parametrize("group", [False, True])
def test_take_ready_argument_checks(group):
    """A NULL bus, a NULL output, n == 0 and ready_cap == 0 are CPBUS_EINVAL, and nothing is written; all but the NULL bus
    are refused before the handle is read, so a zeroed stand-in handle serves on a machine without a GPU."""
    fn = getattr(nat.load(), "cpbus_group_take_ready" if group else "cpbus_take_ready")
    fake, handle = _fake_handle()
    out = np.zeros(64, dtype=EVENT_DTYPE)
    ready = np.zeros(4, dtype=READY_DTYPE)
    n_ready, total, nxt = C.c_size_t(5), C.c_size_t(5), C.c_uint32(5)
    refs = (C.byref(n_ready), C.byref(total), C.byref(nxt))

    def call(h, n=4, ready_cap=4, out_p=out.ctypes.data, ready_p=ready.ctypes.data, r=refs):
        return fn(h, 0, n, 0, out_p, 64, ready_p, ready_cap, *r)

    assert call(None) == nat.EINVAL
    assert call(handle, n=0) == nat.EINVAL
    assert call(handle, ready_cap=0) == nat.EINVAL
    assert call(handle, out_p=None) == nat.EINVAL
    assert call(handle, ready_p=None) == nat.EINVAL
    for j in range(3):
        assert call(handle, r=tuple(None if k == j else refs[k] for k in range(3))) == nat.EINVAL
    assert (n_ready.value, total.value, nxt.value) == (5, 5, 5)
    assert not any(out.tobytes()) and not any(ready.tobytes())
    assert not any(fake.raw), "the handle was written"


@pytest.mark.parametrize("group", [False, True])
def test_ack_many_argument_checks(group):
    """A NULL bus is CPBUS_EINVAL (also with n == 0); a NULL array with n > 0 is CPBUS_EINVAL; n == 0 is CPBUS_OK with
    applied = 0 and no status written, and the handle is not read."""
    fn = getattr(nat.load(), "cpbus_group_ack_many" if group else "cpbus_ack_many")
    fake, handle = _fake_handle()
    ids, counts = np.arange(4, dtype=np.uint32), np.ones(4, dtype=np.uint32)
    status = np.full(4, 99, dtype=np.int32)
    applied = C.c_uint32(7)
    for n in (4, 0):
        assert fn(None, ids.ctypes.data, counts.ctypes.data, n, status.ctypes.data, C.byref(applied)) == nat.EINVAL
    assert fn(handle, None, counts.ctypes.data, 4, status.ctypes.data, C.byref(applied)) == nat.EINVAL
    assert fn(handle, ids.ctypes.data, None, 4, status.ctypes.data, C.byref(applied)) == nat.EINVAL
    assert (status == 99).all() and applied.value == 7
    assert fn(handle, None, None, 0, status.ctypes.data, C.byref(applied)) == nat.OK
    assert (status == 99).all() and applied.value == 0
    assert fn(handle, None, None, 0, None, None) == nat.OK
    assert not any(fake.raw), "the handle was written"


def test_take_ack_declarations_from_plain_c99(tmp_path):
    exe = str(tmp_path / "take_ack_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "take_ack_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "PASS" in r.stdout, r.stdout + r.stderr
