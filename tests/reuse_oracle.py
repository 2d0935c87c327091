"""The oracle with subscriber id reuse: `ReuseOracle`, an `oracle_binding.Oracle` with `release_many` and `subscribe_list`, and
with the bus's rules for ids that name a released slot.

tests/c/reuse_oracle.c includes the oracle's source whole and adds the release and the lowest-free subscribe on top of its own
state; it is compiled once per process into a temporary directory (the source tree may be read-only) and called on the handles
that oracle/libcpbus_oracle.so creates.  The oracle's timer ids carry no generation; this wrapper adds the bus's 6-bit one per
timer slot (advanced by every arming, kept by a release), so that a stale id of a slot's previous occupant is refused here as
on the bus.  Test infrastructure only."""
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
SRC = os.path.join(ROOT, "tests", "c", "reuse_oracle.c")
OK, EINVAL = 0, -1
SLOT_BITS, MAX_PAIRS = 26, 16
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="reuse_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libreuse_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=gnu11", "-Wall", "-Wextra", "-shared", SRC, "-o", so])
        l = C.CDLL(so)
        vp, u32 = C.c_void_p, C.c_uint32
        l.orc_released.restype, l.orc_released.argtypes = C.c_int, [vp, u32]
        l.orc_high_water.restype, l.orc_high_water.argtypes = u32, [vp]
        l.orc_active.restype, l.orc_active.argtypes = C.c_int, [vp, u32]
        l.orc_n_timers.restype, l.orc_n_timers.argtypes = u32, [vp]
        l.orc_release.restype, l.orc_release.argtypes = C.c_int, [vp, u32]
        l.orc_subscribe_list.restype = C.c_int
        l.orc_subscribe_list.argtypes = [vp, vp, vp, vp, vp, u32, vp]
        _lib = l
    return _lib


class ReuseOracle(ob.Oracle):
    def __init__(self, n_max_subs, timers_per_sub=0, keep_window=0, mailbox_cap=0, sub_id_base=0):
        super().__init__(n_max_subs, timers_per_sub, keep_window, mailbox_cap, sub_id_base)
        self.K, self.gen = timers_per_sub, {}

    def released(self, sub) -> bool:
        return bool(lib().orc_released(self.h, sub))

    def high_water(self) -> int:
        return int(lib().orc_high_water(self.h))

    def active(self, sub) -> bool:
        return bool(lib().orc_active(self.h, sub))

    def n_timers(self) -> int:
        return int(lib().orc_n_timers(self.h))

    def release_many(self, ids):
        return [int(lib().orc_release(self.h, int(i))) for i in ids]

    def subscribe_list(self, masks, pairs=None):
        """(status, ids)"""
        m = np.ascontiguousarray(masks, dtype=np.uint32)
        n = m.size
        codes = np.zeros((max(n, 1), MAX_PAIRS), dtype=np.uint32)
        srcs = np.zeros_like(codes)
        cnt = np.zeros(max(n, 1), dtype=np.uint32)
        for i, pr in enumerate(pairs or []):
            cnt[i] = len(pr)
            for j, (c, s) in enumerate(pr):
                codes[i, j], srcs[i, j] = c, s
        out = np.zeros(max(n, 1), dtype=np.uint32)
        rc = lib().orc_subscribe_list(self.h, m.ctypes.data, codes.ctypes.data, srcs.ctypes.data,
                                      cnt.ctypes.data if pairs is not None else None, n, out.ctypes.data)
        return int(rc), ([int(x) for x in out[:n]] if rc == OK else [])

    # ids of released slots are refused as never handed out
    def unsubscribe(self, sub):
        return ob.ENOENT if self.released(sub) else super().unsubscribe(sub)

    def receive(self, sub, code, source_id=0):
        return ob.ENOENT if self.released(sub) else super().receive(sub, code, source_id)

    def timer_add(self, sub, period_ns, source_id, oneshot=False):
        """(status, timer id with the bus's generation)"""
        if self.released(sub):
            return ob.ENOENT, None
        out = C.c_uint32()
        rc = self.l.orc_timer_add(self.h, sub, period_ns, source_id, int(oneshot), C.byref(out))
        if rc:
            return int(rc), None
        slot = out.value
        self.gen[slot] = (self.gen.get(slot, 0) + 1) & 0x3F
        return OK, slot | self.gen[slot] << SLOT_BITS

    def timer_cancel(self, tid):
        slot = tid & ((1 << SLOT_BITS) - 1)
        if not self.K or slot // self.K >= self.high_water() or self.gen.get(slot, 0) != tid >> SLOT_BITS:
            return ob.ENOENT
        return super().timer_cancel(slot)
