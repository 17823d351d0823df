"""Build libjsmpeg_b200.so (hand-written CUDA for sm_90a, H100 + the C ABI) in-tree with nvcc.

    python -m jsmpeg_b200.build

The library is self-contained (static cudart); it is git-ignored but travels with the tree.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["engine.cu", "parse.cu", "recon.cu", "scan.cu", "tsdemux.cu", "psdemux.cu", "macroblocks.cu", "coefficients.cu", "residuals.cu", "accumulate.cu", "conceal.cu"]
OUT = os.path.join(HERE, "libjsmpeg_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def nvcc_path():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "jsmpeg_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    cmd = [nvcc_path(), *ARCH, "-O3", "-std=c++17", "-lineinfo", "--shared", "-Xcompiler", "-fPIC",
           "-Xptxas", "-v" if verbose else "-O3", *os.environ.get("JSMPEG_B200_NVCC_FLAGS", "").split(),
           "-o", OUT, *srcs]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed")
    if verbose:
        print(res.stdout + res.stderr)
    return OUT


if __name__ == "__main__":
    print(build(force=True, verbose="-v" in sys.argv))
