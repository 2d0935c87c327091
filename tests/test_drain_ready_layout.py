"""cpbus_ready (the entry of cpbus_drain_ready's ready list) is a frozen 24-byte C layout; the Python dtype mirrors it."""
import os
import shutil
import subprocess

import pytest

from containerpilot_b200.bus import READY_DTYPE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_numpy_dtype_is_24_bytes_with_the_c_offsets():
    assert READY_DTYPE.itemsize == 24
    assert [READY_DTYPE.fields[f][1] for f in ("sub_id", "count", "offset", "pad", "lost")] == [0, 4, 8, 12, 16]


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_layout_is_24_bytes(tmp_path):
    src = tmp_path / "ready_layout.c"
    src.write_text(
        '#include <stddef.h>\n#include "cpbus.h"\n'
        "_Static_assert(sizeof(cpbus_ready) == 24, \"size\");\n"
        "_Static_assert(offsetof(cpbus_ready, sub_id) == 0 && offsetof(cpbus_ready, count) == 4, \"ids\");\n"
        "_Static_assert(offsetof(cpbus_ready, offset) == 8 && offsetof(cpbus_ready, pad) == 12, \"offsets\");\n"
        "_Static_assert(offsetof(cpbus_ready, lost) == 16, \"lost\");\n")
    subprocess.check_call(["cc", "-std=c11", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)])
