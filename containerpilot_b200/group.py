"""`GroupBus`: one bus handle over several GPUs (or several shards of one GPU), through the `cpbus_group_*` C-ABI.

It has `Bus`'s method names and return conventions for the calls the group supports, and gives the same results as one
`Bus` with the same configuration (include/cpbus.h, "the group").  Shard g lives on `devices[g]`; devices may repeat.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as nat
from .bus import Bus


class _GroupCalls:
    """`lib.cpbus_<name>` -> `lib.cpbus_group_<name>` for the calls the group has; any other call is an error."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name: str):
        short = name[len("cpbus_"):] if name.startswith("cpbus_") else name
        if short in nat.GROUP_CALLS or short == "destroy":
            return getattr(self._lib, "cpbus_group_" + short)
        raise AttributeError(f"{name} has no cpbus_group_* counterpart")


class GroupBus(Bus):
    _GROUP = True   # hides the single-bus-only methods (the drain tickets)

    def __init__(self, n_max_subs: int, devices, ring_cap: int = 1024, batch_cap: int = 256, timers_per_sub: int = 0,
                 lossless: bool = False, digest: bool = True, sub_id_base: int = 0, store_path: int = nat.STORE_AUTO,
                 grid_ctas: int = 0, drop_missed_ticks: bool = False):
        """`drop_missed_ticks`: CPBUS_CFG_DROP_MISSED_TICKS, as on `Bus`"""
        self._h = C.c_void_p()
        lib = nat.load()
        self._lib = _GroupCalls(lib)
        cfg = nat.Config()
        cfg.n_max_subs, cfg.ring_cap, cfg.batch_cap, cfg.timers_per_sub = n_max_subs, ring_cap, batch_cap, timers_per_sub
        cfg.flags = ((nat.CFG_LOSSLESS if lossless else 0) | (nat.CFG_DIGEST if digest else 0)
                     | (nat.CFG_DROP_MISSED_TICKS if drop_missed_ticks else 0))
        cfg.device, cfg.sub_id_base, cfg.store_path, cfg.grid_ctas = -1, sub_id_base, store_path, grid_ctas
        devs = np.ascontiguousarray(list(devices), dtype=np.int32)
        nat.check(lib.cpbus_group_create(C.byref(cfg), devs.ctypes.data, devs.size, C.byref(self._h)), "cpbus_group_create")
        self.devices = [int(d) for d in devs]
        self.ring_cap, self.batch_cap, self.sub_id_base = ring_cap, batch_cap, sub_id_base
