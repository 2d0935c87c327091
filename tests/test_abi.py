"""The C-ABI boundary: libcpbus.so loads here (no GPU) and exports every symbol
include/cpbus.h declares; host-only entry points agree with the golden vectors; and
without a device the library refuses to run (no CPU fallback)."""
import ctypes as C
import json
import os
import subprocess
import re

import numpy as np

import oracle_binding as ob
from containerpilot_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "cpbus.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(cpbus_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = C.CDLL(nat.LIB_PATH)
    names = declared_symbols()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), f"libcpbus.so does not export {n}"
    assert set(names) == set(nat.SYMBOLS), set(names) ^ set(nat.SYMBOLS)
    assert nat.load().cpbus_abi_version() == 2


def test_record_layout_is_32_bytes():
    assert C.sizeof(nat.Event) == 32 and ob.EVENT_DTYPE.itemsize == 32
    assert [f[0] for f in nat.Event._fields_] == list(ob.EVENT_DTYPE.names)


def test_names_agree_with_reference_vectors():
    G = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_vectors.json")))
    lib = nat.load()
    for i, n in enumerate(G["code_names"]["names"]):
        assert lib.cpbus_code_name(i).decode() == n
    assert lib.cpbus_code_name(17) is None
    for name, code in G["from_string"]["accepted"].items():
        assert lib.cpbus_code_from_string(name.encode()) == code
    for name in G["from_string"]["rejected"]:
        assert lib.cpbus_code_from_string(name.encode()) == -1


def test_record_hash_spec_matches_oracle():
    lib = nat.load()
    rng = np.random.default_rng(3)
    for _ in range(200):
        e = nat.Event(int(rng.integers(0, 1 << 62)), int(rng.integers(0, 1 << 62)), int(rng.integers(0, 17)),
                      int(rng.integers(0, 1 << 32)), int(rng.integers(0, 1 << 32)), int(rng.integers(0, 4)))
        assert lib.cpbus_record_hash(C.byref(e)) == ob.lib().orc_record_hash(bytes(e))
    assert lib.cpbus_digest_multiplier() == ob.lib().orc_digest_multiplier()


def test_no_cpu_fallback_without_a_device():
    import torch
    if torch.cuda.is_available():
        return
    cfg = nat.Config(); cfg.n_max_subs = 8; cfg.device = -1
    h = C.c_void_p()
    assert nat.load().cpbus_create(C.byref(cfg), C.byref(h)) == nat.ENODEV
    assert not h.value
    assert b"no CPU fallback" in nat.load().cpbus_strerror(nat.ENODEV)


def test_product_never_touches_the_oracle():
    """The oracle is test infrastructure: nothing under containerpilot_b200/ or include/ may reference it."""
    for base in ("containerpilot_b200", "include"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, base)):
            for fn in files:
                if fn.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cc", ".cpp")):
                    txt = open(os.path.join(dirpath, fn), errors="ignore").read()
                    assert "oracle_binding" not in txt and "libcpbus_oracle" not in txt and "orc_" not in txt, fn


def test_create_rejects_bad_configs_before_touching_the_device():
    """Argument validation is host logic: the same status codes with or without a GPU."""
    lib = nat.load()
    def create(**kw):
        cfg = nat.Config(); cfg.n_max_subs = 8; cfg.device = -1
        for k, v in kw.items():
            setattr(cfg, k, v)
        h = C.c_void_p()
        rc = lib.cpbus_create(C.byref(cfg), C.byref(h))
        if rc == 0:
            lib.cpbus_destroy(h)
        return rc
    assert create(n_max_subs=0) == nat.EINVAL
    assert create(ring_cap=1000) == nat.EINVAL            # not a power of two
    assert create(ring_cap=32) == nat.EINVAL              # < 64
    assert create(ring_cap=1024, batch_cap=1024) == nat.EINVAL   # > ring_cap / 2
    assert create(ring_cap=1024, batch_cap=100) == nat.EINVAL    # not a multiple of 32
    assert create(ring_cap=8192, batch_cap=2048) == nat.EINVAL   # > 1024
    assert create(timers_per_sub=3) == nat.EINVAL
    assert create(store_path=9) == nat.EINVAL
    assert lib.cpbus_create(None, None) == nat.EINVAL
    assert lib.cpbus_destroy(None) == nat.EINVAL
    assert lib.cpbus_strerror(nat.EAGAIN).startswith(b"mailbox full")


C_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "c")


def build_c_smoke(out_dir):
    """tests/c/abi_smoke.c: the C-ABI called from plain C99 (what cgo-generated code does), -Wall -Wextra -Werror -pedantic.
    The program is written to out_dir: the source tree may be read-only to the user running the tests."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(str(out_dir), "abi_smoke")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(root, "include"),
                           os.path.join(C_DIR, "abi_smoke.c"), "-L", os.path.join(root, "containerpilot_b200"), "-lcpbus",
                           "-Wl,-rpath," + os.path.join(root, "containerpilot_b200"), "-o", exe])
    return exe


def test_header_is_plain_c99_and_a_c_caller_links(tmp_path):
    exe = build_c_smoke(tmp_path)
    assert os.path.exists(exe)
    import torch
    if not torch.cuda.is_available():            # without a device the program must stop at cpbus_create with ENODEV, loudly
        r = subprocess.run([exe], capture_output=True, text=True)
        assert r.returncode == 1 and "no CUDA device" in r.stdout


def _mask_order(masks, active, ring_cap, block, heavy):
    lib = nat.load()
    masks = np.ascontiguousarray(masks, dtype=np.uint32)
    act = None if active is None else np.ascontiguousarray(active, dtype=np.uint8)
    out = np.zeros(len(masks), dtype=np.uint32)
    k = lib.cpbus_mask_order(masks.ctypes.data, act.ctypes.data if act is not None else None, len(masks), ring_cap, block, int(heavy), out.ctypes.data)
    return out[:k]


def test_mask_order_host_logic():
    """The walk order of the filtered fan-out (host-only): a permutation of the active subscribers, block by block of
    consecutive ids, equal masks adjacent inside a block, masks with more codes first when asked."""
    import trace as tr
    n = 20_000
    masks = tr.zipf_masks(n, 1.0, 5)
    active = (np.random.default_rng(9).random(n) < 0.9).astype(np.uint8)
    for block, heavy in ((0, False), (0, True), (0xFFFFFFFF, True), (4096, False), (4096, True), (1000, True)):
        o = _mask_order(masks, active, 1024, block, heavy)
        assert sorted(o.tolist()) == np.flatnonzero(active).tolist()                 # exactly the active ones, once each
        blk = n if block in (0, 0xFFFFFFFF) else block                                # 20,000 x 32 KiB < 16 GiB: policy = one block
        bid = o // blk
        assert (np.diff(bid.astype(np.int64)) >= 0).all()                             # blocks in id order
        for b in np.unique(bid):
            m = masks[o[bid == b]] & 0x1FFFF
            runs = np.flatnonzero(np.diff(m.astype(np.int64)) != 0).size + 1
            assert runs == np.unique(m).size                                          # every mask is ONE run inside the block
            if heavy:
                pc = np.array([bin(int(x)).count("1") for x in m])
                assert (np.diff(pc) <= 0).all()                                       # more codes first
            else:
                assert (np.diff(m.astype(np.int64)) >= 0).all()                       # plain mask order
            ids = o[bid == b]
            for mv in np.unique(m)[:20]:
                assert (np.diff(ids[m == mv].astype(np.int64)) > 0).all()             # stable: ids ascending inside a run
    # the footprint policy: 1,048,576 rings of 32 KiB = 32 GiB -> blocks of 8 GiB = 262,144 subscribers
    big = np.full(1 << 20, 0x1FFFF, dtype=np.uint32); big[1::2] = 0x2
    o = _mask_order(big, None, 1024, 0, True)
    assert len(o) == 1 << 20
    first = o[: 1 << 18]
    assert first.max() < (1 << 18) and (first[: 1 << 17] % 2 == 0).all() and (first[1 << 17:] % 2 == 1).all()
    o2 = _mask_order(big[: 1 << 19], None, 1024, 0, True)                            # 16 GiB: one global block
    assert (o2[: 1 << 18] % 2 == 0).all()


def _split_plan(ts, B, now, wm, window):
    lib = nat.load()
    ts = np.ascontiguousarray(ts, dtype=np.uint64)
    n_sl = C.c_size_t()
    rc = lib.cpbus_split_plan(ts.ctypes.data if len(ts) else None, len(ts), B, now, wm, window, None, None, 0, C.byref(n_sl))
    if rc:
        return rc, None, None
    ends = np.zeros(n_sl.value, dtype=np.uintp); wms = np.zeros(n_sl.value, dtype=np.uint64)
    assert lib.cpbus_split_plan(ts.ctypes.data if len(ts) else None, len(ts), B, now, wm, window, ends.ctypes.data, wms.ctypes.data, n_sl.value, C.byref(n_sl)) == 0
    return 0, ends.astype(np.int64), wms


def test_split_plan_host_logic():
    """How an oversize / wide-window device batch is cut (host-only): slices are contiguous, at most batch_cap long, their
    watermarks never decrease, step at most one window, cover their records, end exactly at the caller's watermark, and no
    record older than a slice's watermark is left for a later slice."""
    UMAX = (1 << 64) - 1
    rng = np.random.default_rng(11)
    for trial in range(300):
        B = int(rng.choice([32, 64, 256, 1024]))
        n = int(rng.choice([0, 1, B - 1, B, B + 1, 3 * B + 7, int(rng.integers(0, 5 * B))]))
        now = int(rng.integers(0, 10_000))
        span = int(rng.choice([0, 1, 50, 100_000]))
        window = [UMAX, 1, 7, 1000, 33_000][int(rng.integers(0, 5))]                            # (a Python int: numpy would make 2^64-1 a float)
        ts = np.sort(rng.integers(max(0, now - 20), now + span + 1, n)).astype(np.uint64)     # a few records older than the clock are legal
        wm = now + span + int(rng.choice([0, 0, 5, 40_000]))
        if window == 1 and wm - now > 5000:
            window = 7                                                                         # (keep the number of slices sane)
        rc, ends, wms = _split_plan(ts, B, now, wm, window)
        assert rc == 0
        begins = np.concatenate(([0], ends[:-1]))
        assert (ends >= begins).all() and ends[-1] == n and (ends - begins <= B).all()
        assert (np.diff(wms.astype(object)) >= 0).all() and int(wms[-1]) == wm and int(wms[0]) >= now
        steps = np.diff(np.concatenate(([now], wms)).astype(object))
        if window != UMAX:
            assert max(steps) <= window
        prev = now
        for b0, e0, w in zip(begins, ends, wms):
            if e0 > b0:
                assert int(ts[e0 - 1]) <= int(w)                                               # the slice's records are not beyond its watermark
            if e0 < n and int(ts[e0]) < int(w):
                # a record older than a slice's watermark may only be left behind by a SIZE cut among records that were
                # already older than the clock (they ride with it: the watermark did not move)
                assert e0 - b0 == B and int(w) == prev
            prev = int(w)
        if n <= B and (window == UMAX or wm - now <= window):
            assert len(ends) == 1                                                              # nothing to cut
    # refusals
    assert _split_plan(np.array([5, 4], dtype=np.uint64), 32, 0, 10, UMAX)[0] == nat.EORDER    # unsorted
    assert _split_plan(np.array([5, 11], dtype=np.uint64), 32, 0, 10, UMAX)[0] == nat.EORDER   # beyond the watermark
    assert _split_plan(np.array([], dtype=np.uint64), 32, 10, 9, UMAX)[0] == nat.EORDER        # clock would move backwards
    assert _split_plan(np.array([1], dtype=np.uint64), 32, 0, 10, 0)[0] == nat.EINVAL
