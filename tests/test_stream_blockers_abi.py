"""C-ABI of cpbus_stream_blockers without a GPU: the export and its binding, a plain-C99 caller, and the CPBUS_EINVAL cases
that need no device.  The query itself needs a lossless stream, hence a GPU: tests/test_gpu_stream_blockers.py."""
import ctypes as C
import os
import subprocess

from containerpilot_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_stream_blockers_with_the_blockers_signature():
    lib = C.CDLL(nat.LIB_PATH)
    assert hasattr(lib, "cpbus_stream_blockers")
    assert nat.SYMBOLS["cpbus_stream_blockers"] == nat.SYMBOLS["cpbus_blockers"]
    assert "stream_blockers" not in nat.GROUP_CALLS
    lib = nat.load()
    n, one = C.c_size_t(), (C.c_uint32 * 1)()
    assert lib.cpbus_stream_blockers(None, one, 1, C.byref(n)) == nat.EINVAL
    assert lib.cpbus_stream_blockers(None, None, 0, C.byref(n)) == nat.EINVAL
    assert lib.cpbus_stream_blockers(None, one, 1, None) == nat.EINVAL
    assert lib.cpbus_abi_version() == 2


def test_stream_blockers_declaration_from_plain_c99(tmp_path):
    exe = str(tmp_path / "stream_blockers_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "stream_blockers_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
