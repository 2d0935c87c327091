"""The oracle's side of the consumer backlog queries: `backlog` and `blockers` on an `oracle_binding.Oracle`.

tests/c/lag_oracle.c includes the oracle's source whole and adds the two observers on top of its own rules; it is compiled
once per process into a temporary directory (the source tree may be read-only) and called on the handles that
oracle/libcpbus_oracle.so creates.  Test infrastructure only."""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

import oracle_binding as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "c", "lag_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="lag_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "liblag_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=gnu11", "-Wall", "-Wextra", "-shared", SRC, "-o", so])
        l = C.CDLL(so)
        l.orc_backlog.restype, l.orc_backlog.argtypes = C.c_uint64, [C.c_void_p, C.c_uint32]
        l.orc_blockers.restype = C.c_size_t
        l.orc_blockers.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_size_t]
        _lib = l
    return _lib


def backlog(orc: ob.Oracle, sub: int) -> int:
    """records subscriber `sub`'s mailbox holds (at most mailbox_cap when the oracle has one)"""
    return int(lib().orc_backlog(orc.h, sub))


def blockers(orc: ob.Oracle, t: int, code=None, source_id: int = 0, target: int = 0xFFFFFFFF) -> np.ndarray:
    """ids that would block the next sends: the ticks due by t, then {code, source_id} to target (code None: ticks only)"""
    rec = None
    if code is not None:
        rec = np.zeros(1, dtype=ob.EVENT_DTYPE)
        rec["ts_ns"], rec["code"], rec["source_id"], rec["target"] = t, code, source_id, target
    ptr = None if rec is None else rec.ctypes.data
    n = lib().orc_blockers(orc.h, ptr, t, None, 0)
    out = np.zeros(max(1, n), dtype=np.uint32)
    lib().orc_blockers(orc.h, ptr, t, out.ctypes.data, n)
    return out[:n]
