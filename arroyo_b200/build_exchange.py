"""Builds the opt-in native Shuffle edge (csrc/exchange.cu -> libarroyo_b200_xchg.so): NCCL called from C++.
Separate from build.py on purpose: nothing on the measured paths loads this library.  Skipped (returns None) when the
NCCL headers / library that ship with torch are not there."""
import glob
import os
import subprocess
import sys

from . import build as main_build

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "exchange.cu")
LIB = os.path.join(HERE, "libarroyo_b200_xchg.so")


def nccl_paths():
    for base in sys.path:
        inc = os.path.join(base, "nvidia", "nccl", "include")
        libs = glob.glob(os.path.join(base, "nvidia", "nccl", "lib", "libnccl.so*"))
        if os.path.exists(os.path.join(inc, "nccl.h")) and libs:
            return inc, sorted(libs)[0]
    return None, None


def build(force: bool = False):
    inc, lib = nccl_paths()
    if inc is None:
        return None
    main_lib = main_build.build()
    deps = [SRC, main_lib, os.path.abspath(__file__)]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(d) for d in deps):
        return LIB
    tmp = LIB + ".tmp"
    cmd = [main_build.nvcc_path(), *main_build.GENCODE, "-O3", "-std=c++17", "-lineinfo",
           "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function", "--expt-relaxed-constexpr", "-I" + inc, "-shared", "-o", tmp, SRC,
           "-L" + HERE, "-l:" + os.path.basename(main_lib), "-L" + os.path.dirname(lib), "-l:" + os.path.basename(lib),
           "-Xlinker", "-rpath=$ORIGIN", "-Xlinker", "-rpath=" + os.path.dirname(lib), "-lcudart"]
    subprocess.check_call(cmd)
    os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
