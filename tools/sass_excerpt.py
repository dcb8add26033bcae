#!/usr/bin/env python
"""SASS evidence for the two-pass ingest kernels: the TMA bulk copies (UBLKCP.S.G) and mbarrier operations (SYNCS.*) of
agg_kernel's per-warp rings, the shared-memory atomics (ATOMS.*) of both passes, the 128-bit shared / global accesses.

    python tools/sass_excerpt.py > profiles/r02_sass_excerpt.txt      (needs cuobjdump, no GPU)
"""
import os
import re
import subprocess
import sys
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "arroyo_b200", "libarroyo_b200.so")
PAT = re.compile(r"UBLKCP|SYNCS|ATOMS|ATOMG|\bRED\.|LDS\.128|STS\.128|STG\.E\.128|LDG\.E\.(64|128)")


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    print("# cuobjdump -sass arroyo_b200/libarroyo_b200.so (sm_90a): opcode counts and first occurrences per kernel")
    for kernel in ("agg_kernelILi1", "agg_kernelILi0", "part_kernelILi1ELi1", "part_kernelILi0ELi0"):
        inside, ops, first = False, Counter(), {}
        for line in sass.splitlines():
            if "Function :" in line:
                inside = kernel in line
                continue
            if not inside:
                continue
            m = re.search(r"/\*([0-9a-f]{4})\*/\s+(.*?);", line)
            if not m or not PAT.search(m.group(2)):
                continue
            text = re.sub(r"\s+", " ", m.group(2)).strip()
            op = next(t for t in text.split() if not t.startswith("@"))
            ops[op] += 1
            first.setdefault(op, f"/*{m.group(1)}*/ {text}")
        print(f"\n## {kernel}")
        for op, n in sorted(ops.items()):
            print(f"{n:4d} x {op:36s} first: {first[op]}")


if __name__ == "__main__":
    sys.exit(main())
