"""libcpbus's host code is split across translation units: the files that hold no device code compile as plain C++17,
and the internals they share stay out of the library's dynamic symbol table, with one definition of the thread's CUDA
error text (cpbus_last_cuda_error) however many files record into it."""
import os
import shutil
import subprocess

import pytest

from containerpilot_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "containerpilot_b200", "csrc")


def cuda_include():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")
    assert os.path.exists(os.path.join(inc, "cuda_runtime.h")), f"no CUDA headers next to {nvcc}"
    return inc


@pytest.mark.parametrize("name", ["cpbus_host.cpp", "cpbus_group.cpp", "host_index.hpp"])
def test_host_files_compile_as_plain_cpp(name):
    cxx = shutil.which(os.environ.get("CXX", "g++"))
    assert cxx, "no C++ compiler"
    r = subprocess.run([cxx, "-std=c++17", "-fsyntax-only", "-x", "c++", "-I", os.path.join(ROOT, "include"), "-I", CSRC,
                        "-I", cuda_include(), os.path.join(CSRC, name)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def nm(*args):
    return subprocess.run(["nm", *args, nat.LIB_PATH], capture_output=True, text=True, check=True).stdout.splitlines()


def test_library_exports_no_internal_symbol():
    exported = nm("-D", "-C", "--defined-only")
    assert any(line.endswith(" cpbus_create") for line in exported)
    leaked = [line for line in exported if "cpbus_host::" in line]
    assert not leaked, leaked[:10]


def test_cuda_error_text_is_defined_once():
    defs = [line for line in nm("-C") if line.endswith("g_cuda_err") and line.split()[-2] in "bBdD"]
    assert len(defs) == 1, defs
