"""C-ABI of the group (cpbus_group_*): every entry point is exported and bound, each twin declares the arguments of its
single-bus entry point with the group handle in front, and the declarations compile and run from plain C99.  The group
itself needs a bus, hence a GPU: tests/test_gpu_group.py."""
import ctypes as C
import os
import re
import subprocess

from containerpilot_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "cpbus.h")).read()


def _decls():
    """{name: [parameter types]} of every `int cpbus_*(...)` declaration in the header"""
    out = {}
    for name, args in re.findall(r"\bint (cpbus_\w+)\(([^;{]*?)\)\s*;", HEADER, re.S):
        types = []
        for p in " ".join(args.split()).split(","):
            p = p.strip()
            p = re.sub(r"\s*\b\w+\[\d*\]$", "*", p)                   # out[4] / handle[64] -> pointer
            types.append(re.sub(r"\s*\b\w+$", "", p) if not p.endswith("*") else p)
        out[name] = types
    return out


def test_every_group_call_is_exported_and_bound():
    lib = C.CDLL(nat.LIB_PATH)
    decls = _decls()
    names = {n for n in decls if n.startswith("cpbus_group_")}
    assert names == {"cpbus_group_create", "cpbus_group_destroy"} | {f"cpbus_group_{x}" for x in nat.GROUP_CALLS}
    for name in names:
        assert hasattr(lib, name), name
        assert name in nat.SYMBOLS, name
    assert nat.load().cpbus_abi_version() == 2


def test_each_twin_takes_the_single_bus_arguments():
    decls = _decls()
    for x in nat.GROUP_CALLS:
        one, grp = decls[f"cpbus_{x}"], decls[f"cpbus_group_{x}"]
        assert one[0] == "cpbus_t*" and grp[0] == "cpbus_group_t*", x
        assert one[1:] == grp[1:], (x, one, grp)
        assert nat.SYMBOLS[f"cpbus_group_{x}"] == nat.SYMBOLS[f"cpbus_{x}"], x
    assert decls["cpbus_group_create"] == ["const cpbus_config*", "const int32_t*", "uint32_t", "cpbus_group_t**"]


def test_group_declarations_from_plain_c99(tmp_path):
    exe = str(tmp_path / "group_abi")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "group_abi.c"), "-L", os.path.join(ROOT, "containerpilot_b200"),
                           "-lcpbus", "-Wl,-rpath," + os.path.join(ROOT, "containerpilot_b200"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
