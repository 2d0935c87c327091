"""The bulk membership calls (cpbus_unsubscribe_many, cpbus_set_mask_many, cpbus_timer_cancel_many and their group twins)
without a GPU: the exports and declarations, a plain-C99 caller, and the argument checks, which return before the bus or a
device is looked at.  The calls themselves need a GPU: tests/test_gpu_bulk_membership.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from containerpilot_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ("unsubscribe_many", "set_mask_many", "timer_cancel_many")


def test_exports_and_declarations():
    lib = C.CDLL(nat.LIB_PATH)
    hdr = open(os.path.join(ROOT, "include", "cpbus.h")).read()
    for name in CALLS:
        for full in (f"cpbus_{name}", f"cpbus_group_{name}"):
            assert hasattr(lib, full) and full in nat.SYMBOLS
            assert re.search(r"\bint " + full + r"\(", hdr), full
    assert nat.load().cpbus_abi_version() == 2


def _call(name, handle, arrays, n, status, applied):
    fn = getattr(nat.load(), name)
    return fn(handle, *arrays, n, status, applied)


def _arrays(name, ids):
    return [ids, ids] if name.endswith("set_mask_many") else [ids]


@pytest.mark.parametrize("group", [False, True])
@pytest.mark.parametrize("name", CALLS)
def test_null_bus_is_einval(name, group):
    full = f"cpbus_group_{name}" if group else f"cpbus_{name}"
    ids = np.arange(4, dtype=np.uint32)
    status = np.full(4, 99, dtype=np.int32)
    applied = C.c_uint32(7)
    for n in (4, 0):
        assert _call(full, None, [a.ctypes.data for a in _arrays(name, ids)], n, status.ctypes.data, C.byref(applied)) == nat.EINVAL
    assert (status == 99).all() and applied.value == 7


@pytest.mark.parametrize("group", [False, True])
@pytest.mark.parametrize("name", CALLS)
def test_null_arrays_and_empty_lists(name, group):
    """A NULL array with n > 0 is CPBUS_EINVAL; n == 0 is CPBUS_OK with applied = 0 and no status written.  Both return
    before the handle is read, so a zeroed stand-in handle serves on a machine without a GPU."""
    full = f"cpbus_group_{name}" if group else f"cpbus_{name}"
    fake = C.create_string_buffer(4096)
    handle = C.c_void_p(C.addressof(fake))
    ids = np.arange(4, dtype=np.uint32)
    status = np.full(4, 99, dtype=np.int32)
    applied = C.c_uint32(7)
    n_arrays = len(_arrays(name, ids))
    for null_at in range(n_arrays):
        arrays = [None if j == null_at else ids.ctypes.data for j in range(n_arrays)]
        assert _call(full, handle, arrays, 4, status.ctypes.data, C.byref(applied)) == nat.EINVAL
    assert (status == 99).all() and applied.value == 7
    assert _call(full, handle, [None] * n_arrays, 0, status.ctypes.data, C.byref(applied)) == nat.OK
    assert (status == 99).all() and applied.value == 0
    assert _call(full, handle, [None] * n_arrays, 0, None, None) == nat.OK
    assert not any(fake.raw), "the handle was written"


def test_bulk_membership_declarations_from_plain_c99(tmp_path):
    exe = str(tmp_path / "bulk_membership_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "bulk_membership_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "PASS" in r.stdout, r.stdout + r.stderr
