#!/bin/bash
# Registers / spills of every kernel variant (cross-compiles without a GPU).  usage: scripts/ptxas_summary.sh [extra nvcc flags]
cd "$(dirname "$0")/.."
# (compiled, not linked: the host internals that cpbus.cu calls live in the library's other files, hidden)
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -c -Xcompiler -fPIC -Xptxas -v "$@" \
  -o /tmp/cpbus_ptxas.o containerpilot_b200/csrc/cpbus.cu 2>&1 | python3 -c '
import re, sys, subprocess
txt = sys.stdin.read()
for m in re.finditer(r"Compiling entry function .(\S+?). for .sm_90a.\n.*?\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\nptxas info\s+: Used (\d+) registers", txt):
    name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
    print(f"{name:70s} regs={m.group(5):>3s} stack={m.group(2):>3s} spill_st={m.group(3):>3s} spill_ld={m.group(4):>3s}")
errs = [l for l in txt.splitlines() if "error" in l.lower()]
print("\n".join(errs))
'
