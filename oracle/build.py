"""Build recipe for the CPU oracle (TEST INFRASTRUCTURE ONLY -- see oracle/xq_oracle.c).

    python oracle/build.py        -> oracle/libxq_oracle.so

Flags: -ffp-contract=off so that only the fmaf() calls written in the source fuse
(canonical arithmetic); -mfma -mavx2 (x86-64-v3, present on every current x86 GPU host) so fmaf
is a single instruction; OpenMP for the row-parallel loops.  The reference is pure Python,
so there is no `oracle/_ref` to compile (DESIGN.md "Oracle").
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "xq_oracle.c")
OUT = os.path.join(HERE, "libxq_oracle.so")


def build(force: bool = False) -> str:
    if (not force and os.path.exists(OUT)
            and os.path.getmtime(OUT) >= os.path.getmtime(SRC)):
        return OUT
    cmd = ["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-fopenmp",
           "-ffp-contract=off", "-fno-fast-math", "-mavx2", "-mfma",
           "-o", OUT, SRC, "-lm"]
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
