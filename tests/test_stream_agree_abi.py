"""C-ABI of the cross-process lossless stream (cpbus_stream_offer / cpbus_stream_agree): exported, bound, and NULL
arguments are refused with CPBUS_EINVAL before anything touches a device.  The throughput-mode and round-state checks
need a bus, hence a GPU: tests/test_gpu_stream_agree.py."""
import ctypes as C

from containerpilot_b200 import _native as nat


def test_offer_and_agree_are_exported_and_bound():
    lib = C.CDLL(nat.LIB_PATH)
    for name in ("cpbus_stream_offer", "cpbus_stream_agree"):
        assert hasattr(lib, name)
        assert name in nat.SYMBOLS
    assert nat.load().cpbus_abi_version() == 2


def test_null_arguments_give_einval():
    lib = nat.load()
    m = C.c_size_t(7)
    assert lib.cpbus_stream_offer(None, 0, 0) == nat.EINVAL
    assert lib.cpbus_stream_offer(None, 5, 1) == nat.EINVAL
    assert lib.cpbus_stream_agree(None, C.byref(m)) == nat.EINVAL
    assert lib.cpbus_stream_agree(None, None) == nat.EINVAL
