"""C-ABI of the stream follower (cpbus_stream_fanout_next): exported, bound, and a NULL stream is refused with
CPBUS_EINVAL before anything touches a device.  The lossless refusal and the launches themselves need a bus, hence a GPU:
tests/test_gpu_stream_follow.py."""
import ctypes as C

from containerpilot_b200 import _native as nat


def test_fanout_next_is_exported_and_bound():
    lib = C.CDLL(nat.LIB_PATH)
    assert hasattr(lib, "cpbus_stream_fanout_next")
    assert "cpbus_stream_fanout_next" in nat.SYMBOLS
    assert nat.load().cpbus_abi_version() == 2


def test_null_stream_gives_einval():
    assert nat.load().cpbus_stream_fanout_next(None) == nat.EINVAL
