"""Device batches on the group (cpbus_group_publish_device, cpbus_group_publish_device_staged) without a GPU: the exports,
declarations and bindings, a plain-C99 caller, and the argument checks, which return CPBUS_EINVAL before a device is
looked at.  The calls themselves need a GPU: tests/test_gpu_group_device.py."""
import ctypes as C
import os
import re
import subprocess

import pytest

from containerpilot_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ("publish_device", "publish_device_staged")


def test_exports_declarations_and_bindings():
    lib = C.CDLL(nat.LIB_PATH)
    hdr = open(os.path.join(ROOT, "include", "cpbus.h")).read()
    for name in CALLS:
        assert name in nat.GROUP_CALLS
        full = f"cpbus_group_{name}"
        assert hasattr(lib, full) and full in nat.SYMBOLS
        assert nat.SYMBOLS[full] == nat.SYMBOLS[f"cpbus_{name}"]
        assert re.search(r"\bint " + full + r"\(cpbus_group_t\* g,", hdr), full
    assert nat.load().cpbus_abi_version() == 2


def _fake():
    """a zeroed stand-in handle: every check below returns before a device is touched or the handle is written"""
    fake = C.create_string_buffer(1 << 16)
    return fake, C.c_void_p(C.addressof(fake))


@pytest.mark.parametrize("group", [False, True])
@pytest.mark.parametrize("name", CALLS)
def test_argument_checks(name, group):
    """NULL handle, NULL batch with n > 0, a batch not 32-byte aligned, a misaligned or oversized next-batch hint"""
    fn = getattr(nat.load(), ("cpbus_group_" if group else "cpbus_") + name)
    batch = C.create_string_buffer(32 * 9 + 64)
    aligned = (C.addressof(batch) + 31) & ~31
    fake, handle = _fake()

    def call(h, ptr, n, nxt=0, n_next=0):
        args = (h, C.c_void_p(ptr), n, 1000)
        return fn(*args, C.c_void_p(nxt), n_next) if name == "publish_device_staged" else fn(*args)

    assert call(None, aligned, 4) == nat.EINVAL
    assert call(None, 0, 0) == nat.EINVAL
    assert call(handle, 0, 4) == nat.EINVAL
    for off in (1, 8, 16):
        assert call(handle, aligned + off, 4) == nat.EINVAL
    if name == "publish_device_staged":
        assert call(handle, aligned, 4, aligned + 8, 4) == nat.EINVAL
        assert call(handle, aligned, 4, aligned, 1) == nat.EINVAL          # n_next > batch_cap (0 in the zeroed handle)
    assert not any(fake.raw), "the handle was written"


def test_group_device_declarations_from_plain_c99(tmp_path):
    exe = str(tmp_path / "group_device_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "group_device_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
