"""The owners of the bus's CUDA memory, events and streams (containerpilot_b200/csrc/cuda_owned.hpp): a small C++ program
built with g++ against the header and the CUDA runtime checks their failure rule without a device and their growth on the
GPU; on the GPU a bus whose drain staging was refused keeps working and returns what the oracle expects."""
import os
import subprocess

import numpy as np
import pytest

import oracle_binding as ob
from containerpilot_b200 import _native as nat
from containerpilot_b200.bus import Bus, EVENT_DTYPE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.path.dirname(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")))


def _run(tmp_path, mode, env=None):
    exe = str(tmp_path / "owned_buffers")
    lib = os.path.join(CUDA, "lib64")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror",
                           "-I", os.path.join(ROOT, "containerpilot_b200", "csrc"), "-I", os.path.join(CUDA, "include"),
                           os.path.join(ROOT, "tests", "c", "owned_buffers.cc"), "-o", exe,
                           "-L", lib, "-lcudart", "-Wl,-rpath," + lib])
    r = subprocess.run([exe, mode], capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stdout + r.stderr


def test_refused_allocations_leave_owners_empty(tmp_path):
    """No visible device: grow and alloc return the error and leave {nullptr, 0}; events and streams stay null; empty and
    moved-from owners are destroyed harmlessly."""
    _run(tmp_path, "nodevice", env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})


@pytest.mark.gpu
def test_owners_on_the_device(tmp_path):
    """grow applies the floor and keeps a buffer that fits; a request larger than the device is refused with
    cudaErrorMemoryAllocation, leaves {nullptr, 0} and no last error, and a small grow then succeeds; a move hands an
    allocation over exactly once."""
    _run(tmp_path, "device")


def _publish(bus, orc, rng, n_events):
    ev = np.zeros(n_events, dtype=EVENT_DTYPE)
    ev["code"] = rng.integers(1, 17, n_events)
    ev["source_id"] = rng.integers(0, 64, n_events)
    nat.check(bus.publish_many(ev), "publish")
    nat.check(bus.flush(), "flush")
    for c, s in zip(ev["code"], ev["source_id"]):
        assert orc.publish(int(c), int(s)) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("lossless", [True, False])
def test_refused_drain_staging_leaves_the_bus_usable(lossless):
    """A drain_many whose staging the device cannot hold returns CPBUS_ECUDA and leaves the buffer empty, so later drains
    with smaller caps regrow it instead of writing through a null pointer, and later calls do not see the refusal."""
    N, R = 32, 1024
    rng = np.random.default_rng(0x0B0FF)
    masks = np.where(rng.random(N) < 0.5, nat.MASK_ALL, rng.integers(0, 1 << 17, N)).astype(np.uint32)
    orc = ob.Oracle(N)
    with Bus(N, ring_cap=R, batch_cap=256, lossless=lossless, digest=True, device=0) as bus:
        bus.subscribe_many(masks)
        for m in masks:
            orc.subscribe(int(m))

        def check_many(cap):
            rec, offs, cnts = bus.drain_many(0, N, cap)
            for s in range(N):
                got = rec[int(offs[s]):int(offs[s]) + int(cnts[s])]
                assert got.tobytes() == orc.consume(s, R).tobytes(), s

        _publish(bus, orc, rng, 100)
        check_many(8192)
        _publish(bus, orc, rng, 100)
        out = np.zeros(N * R, dtype=EVENT_DTYPE)                # room for every record the mailboxes can hold
        with pytest.raises(nat.CpbusError) as e:
            bus.drain_many(0, N, 0xFFFFFFFF, out=out)           # 128 GiB of staging
        assert e.value.status == nat.ECUDA
        check_many(4096)
        _publish(bus, orc, rng, 100)
        runs, start = {}, 0
        while True:
            rec, ready, start = bus.drain_ready(0, N, start, 2048, N)
            if len(ready) == 0:
                break
            for r in ready:
                runs.setdefault(int(r["sub_id"]), []).append(rec[int(r["offset"]):int(r["offset"]) + int(r["count"])])
        for s in range(N):
            got = np.concatenate(runs[s]) if s in runs else np.zeros(0, dtype=EVENT_DTYPE)
            assert got.tobytes() == orc.consume(s, R).tobytes(), s
        d = bus.digests(0, N)
        for s in range(N):
            assert int(d["count"][s]) == orc.count(s) and int(d["digest"][s]) == orc.digest(s), s
