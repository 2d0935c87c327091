"""cpbus — an H100-native event bus behind ContainerPilot's `events` API.

Package layout (only what the hot path needs):
  csrc/cpbus_kernels.cuh   sm_90a kernels (fan-out, admission, digest fold)
  csrc/cpbus.cu            C-ABI implementation (include/cpbus.h) -> libcpbus.so: the bus, its streams, every launch
  csrc/cpbus_group.cpp     the group (cpbus_group_*), host C++ over the bus
  csrc/cpbus_host.cpp      host-only planners and exports; host_index.hpp: the due and subscription indexes
  csrc/cpbus_internal.hpp  what those three files share (struct cpbus, struct cpbus_group, the host front end)
  _native.py               ctypes binding of the C-ABI (no fallback)
  bus.py                   numpy-friendly `Bus` wrapper, 1:1 with cpbus_*
  events.py                mirror of the Go `events` package API
"""
from . import _native  # noqa: F401

__all__ = ["_native", "bus", "events"]
