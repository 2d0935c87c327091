"""Bulk timer arming (cpbus_timer_add_list and cpbus_group_timer_add_list) without a GPU: the exports and declarations,
cpbus_timer_spec's layout from a plain-C99 caller and from Python, and the argument checks, which return before the bus or
a device is looked at.  The calls themselves need a GPU: tests/test_gpu_timer_add_list.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from containerpilot_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("cpbus_timer_add_list", "cpbus_group_timer_add_list")
LAYOUT = [24, 0, 8, 12, 16, 20]   # sizeof, then offsetof period_ns, sub_id, source_id, oneshot, pad


def test_exports_and_declarations():
    lib = C.CDLL(nat.LIB_PATH)
    hdr = open(os.path.join(ROOT, "include", "cpbus.h")).read()
    for full in NAMES:
        assert hasattr(lib, full) and full in nat.SYMBOLS
        assert re.search(r"\bint " + full + r"\(", hdr), full
    assert "timer_add_list" in nat.GROUP_CALLS
    assert re.search(r"typedef struct cpbus_timer_spec \{", hdr)
    assert nat.load().cpbus_abi_version() == 2


def test_spec_dtype_matches_the_header():
    d = nat.TIMER_SPEC_DTYPE
    assert [d.itemsize] + [d.fields[f][1] for f in ("period_ns", "sub_id", "source_id", "oneshot", "pad")] == LAYOUT


def _specs(n):
    s = np.zeros(n, dtype=nat.TIMER_SPEC_DTYPE)
    s["period_ns"], s["sub_id"], s["source_id"] = 1000, np.arange(n), 7
    return s


@pytest.mark.parametrize("name", NAMES)
def test_null_bus_is_einval(name):
    fn = getattr(nat.load(), name)
    specs = _specs(4)
    ids = np.full(4, 5, dtype=np.uint32)
    status = np.full(4, 99, dtype=np.int32)
    applied = C.c_uint32(7)
    for n in (4, 0):
        assert fn(None, specs.ctypes.data, n, ids.ctypes.data, status.ctypes.data, C.byref(applied)) == nat.EINVAL
    assert (status == 99).all() and (ids == 5).all() and applied.value == 7


@pytest.mark.parametrize("name", NAMES)
def test_null_specs_and_empty_lists(name):
    """NULL specs with n > 0 is CPBUS_EINVAL; n == 0 is CPBUS_OK with applied = 0 and no id or status written.  Both return
    before the handle is read, so a zeroed stand-in handle serves on a machine without a GPU."""
    fn = getattr(nat.load(), name)
    fake = C.create_string_buffer(4096)
    handle = C.c_void_p(C.addressof(fake))
    ids = np.full(4, 5, dtype=np.uint32)
    status = np.full(4, 99, dtype=np.int32)
    applied = C.c_uint32(7)
    assert fn(handle, None, 4, ids.ctypes.data, status.ctypes.data, C.byref(applied)) == nat.EINVAL
    assert (status == 99).all() and (ids == 5).all() and applied.value == 7
    assert fn(handle, None, 0, ids.ctypes.data, status.ctypes.data, C.byref(applied)) == nat.OK
    assert (status == 99).all() and (ids == 5).all() and applied.value == 0
    assert fn(handle, _specs(4).ctypes.data, 0, None, None, None) == nat.OK
    assert not any(fake.raw), "the handle was written"


def test_timer_add_list_from_plain_c99(tmp_path):
    exe = str(tmp_path / "timer_add_list_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "timer_add_list_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "PASS" in r.stdout, r.stdout + r.stderr
    layout = re.search(r"layout ([\d ]+)", r.stdout).group(1).split()
    assert [int(x) for x in layout] == LAYOUT
