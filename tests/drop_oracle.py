"""The oracle with missed periodic ticks dropped (CPBUS_CFG_DROP_MISSED_TICKS): `DropOracle`, an `oracle_binding.Oracle`
whose `advance` catches each periodic timer up to its last firing in the step before the oracle's firing loop runs.

tests/c/drop_oracle.c includes the oracle's source whole and adds that catch-up on top of its own timer state; it is compiled
once per process into a temporary directory (the source tree may be read-only) and called on the handles that
oracle/libcpbus_oracle.so creates.  Test infrastructure only."""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import oracle_binding as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "c", "drop_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="drop_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libdrop_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=gnu11", "-Wall", "-Wextra", "-shared", SRC, "-o", so])
        l = C.CDLL(so)
        l.orc_advance_drop_missed.restype, l.orc_advance_drop_missed.argtypes = C.c_int, [C.c_void_p, C.c_uint64]
        _lib = l
    return _lib


class DropOracle(ob.Oracle):
    def advance(self, now_ns):
        return lib().orc_advance_drop_missed(self.h, now_ns)
