"""C-ABI of the lossless stream rounds (cpbus_stream_round_next / cpbus_stream_progress): exported, bound, and NULL
arguments are refused with CPBUS_EINVAL before anything touches a device.  The rounds themselves need a bus, hence a GPU:
tests/test_gpu_stream_rounds.py."""
import ctypes as C

from containerpilot_b200 import _native as nat


def test_round_next_and_progress_are_exported_and_bound():
    lib = C.CDLL(nat.LIB_PATH)
    for name in ("cpbus_stream_round_next", "cpbus_stream_progress"):
        assert hasattr(lib, name)
        assert name in nat.SYMBOLS
    assert nat.load().cpbus_abi_version() == 2


def test_null_arguments_give_einval():
    lib = nat.load()
    b, off, stalled = C.c_uint64(7), C.c_size_t(7), C.c_uint64(7)
    assert lib.cpbus_stream_round_next(None) == nat.EINVAL
    assert lib.cpbus_stream_progress(None, C.byref(b), C.byref(off), C.byref(stalled)) == nat.EINVAL
    assert lib.cpbus_stream_progress(None, None, None, None) == nat.EINVAL
    assert (b.value, off.value, stalled.value) == (7, 7, 7)
