"""Drain tickets (cpbus_drain_ready_begin, cpbus_take_ready_begin, cpbus_drain_ready_end; Bus.drain_ready_begin,
.take_ready_begin, .drain_ready_end) without a GPU: the exports and declarations, the output layout they share with
cpbus_drain_ready, a plain-C99 caller, and the argument checks that return before the bus or a device is looked at.  The
calls themselves need a GPU: tests/test_gpu_drain_tickets.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE, READY_DTYPE
from containerpilot_b200.group import GroupBus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "cpbus.h")).read()
BEGINS = ("cpbus_drain_ready_begin", "cpbus_take_ready_begin")
END = "cpbus_drain_ready_end"


def _decl(name):
    """the parameter list of `int name(...)` in the header, whitespace normalised"""
    m = re.search(r"\bint " + name + r"\(([^;{]*?)\)\s*;", HEADER, re.S)
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def test_exports_and_declarations():
    lib = C.CDLL(nat.LIB_PATH)
    for name in BEGINS + (END,):
        assert hasattr(lib, name) and name in nat.SYMBOLS, name
        assert not hasattr(lib, name.replace("cpbus_", "cpbus_group_")), "the group has no drain tickets"
        assert len(_decl(name)) == len(nat.SYMBOLS[name][1]), name
    assert nat.SYMBOLS[BEGINS[0]] == nat.SYMBOLS[BEGINS[1]]
    assert _decl(BEGINS[0])[1:] == _decl(BEGINS[1])[1:]
    assert _decl(BEGINS[0])[-3:] == ["size_t cap", "size_t ready_cap", "uint32_t* ticket"]
    assert nat.load().cpbus_abi_version() == 2


def test_end_shares_the_output_layout_of_drain_ready():
    """_end's outputs are cpbus_drain_ready's, parameter for parameter: (out, cap, ready, ready_cap, n_ready, total,
    next_sub), and its ctypes binding takes the same types there."""
    sync, end = _decl("cpbus_drain_ready"), _decl(END)
    assert end[0] == "cpbus_t* bus" and end[1] == "uint32_t ticket"
    assert end[2:] == sync[4:]
    assert nat.SYMBOLS[END][1][2:] == nat.SYMBOLS["cpbus_drain_ready"][1][4:]
    assert nat.SYMBOLS[END][0] == nat.SYMBOLS["cpbus_drain_ready"][0]


def test_python_methods_are_the_single_bus_ones():
    for name in ("drain_ready_begin", "take_ready_begin", "drain_ready_end"):
        assert callable(getattr(Bus, name)), name
        assert not hasattr(GroupBus, name), name
    for name in ("drain_ready_begin", "take_ready_begin", "drain_ready_end"):
        assert name not in nat.GROUP_CALLS


def _fake_handle():
    fake = C.create_string_buffer(4096)
    return fake, C.c_void_p(C.addressof(fake))


@pytest.mark.parametrize("name", BEGINS)
def test_begin_argument_checks(name):
    """A NULL bus, a NULL ticket, n == 0 and ready_cap == 0 are CPBUS_EINVAL and write no ticket; all but the NULL bus are
    refused before the handle is read, so a zeroed stand-in handle serves on a machine without a GPU."""
    fn = getattr(nat.load(), name)
    fake, handle = _fake_handle()
    ticket = C.c_uint32(77)

    def call(h, n=4, ready_cap=4, t=C.byref(ticket)):
        return fn(h, 0, n, 0, 1024, ready_cap, t)

    assert call(None) == nat.EINVAL
    assert call(handle, t=None) == nat.EINVAL
    assert call(handle, n=0) == nat.EINVAL
    assert call(handle, ready_cap=0) == nat.EINVAL
    assert ticket.value == 77
    assert not any(fake.raw), "the handle was written"


def test_end_argument_checks():
    """A NULL bus or any NULL output is CPBUS_EINVAL, and nothing is written."""
    fn = getattr(nat.load(), END)
    fake, handle = _fake_handle()
    out = np.zeros(64, dtype=EVENT_DTYPE)
    ready = np.zeros(4, dtype=READY_DTYPE)
    n_ready, total, nxt = C.c_size_t(5), C.c_size_t(5), C.c_uint32(5)
    refs = (C.byref(n_ready), C.byref(total), C.byref(nxt))

    def call(h, out_p=out.ctypes.data, ready_p=ready.ctypes.data, r=refs):
        return fn(h, 0, out_p, 64, ready_p, 4, *r)

    assert call(None) == nat.EINVAL
    assert call(handle, out_p=None) == nat.EINVAL
    assert call(handle, ready_p=None) == nat.EINVAL
    for j in range(3):
        assert call(handle, r=tuple(None if k == j else refs[k] for k in range(3))) == nat.EINVAL
    assert (n_ready.value, total.value, nxt.value) == (5, 5, 5)
    assert not any(out.tobytes()) and not any(ready.tobytes())
    assert not any(fake.raw), "the handle was written"


def test_drain_tickets_declarations_from_plain_c99(tmp_path):
    exe = str(tmp_path / "drain_tickets_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "drain_tickets_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "PASS" in r.stdout, r.stdout + r.stderr
