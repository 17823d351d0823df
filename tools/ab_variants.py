#!/usr/bin/env python
"""Build compile-time variants of the product library side by side and print the one-call A/B command.

    python tools/ab_variants.py                      # builds variants/lib_<name>.so for the candidates below
    <the printed command>                            # on the GPU: tools/time_stages.py per library (JSMPEG_B200_LIB), twice, interleaved

The candidates are the compile-time tuning constants: the occupancy bounds of the lane-parallel walk and of
the reconstruct kernel, and the runs per CTA of the expand kernel.  The in-tree library is left alone.
"""
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from jsmpeg_b200 import build  # noqa: E402

CANDIDATES = {
    "default": "",
    "lanes_ctas3": "-DJSMPEG_LANES_MIN_CTAS=3",
    "lanes_ctas5": "-DJSMPEG_LANES_MIN_CTAS=5",
    "expand_groups1": "-DJSMPEG_EXPAND_GROUPS=1",
    "expand_groups8": "-DJSMPEG_EXPAND_GROUPS=8",
    "recon_ctas4": "-DJSMPEG_RECON_MIN_CTAS=4",
    "recon_ctas6": "-DJSMPEG_RECON_MIN_CTAS=6",
}


def main():
    out_dir = os.path.join(ROOT, "variants")
    os.makedirs(out_dir, exist_ok=True)
    keep = build.OUT + ".keep"
    if os.path.exists(build.OUT):
        shutil.copy2(build.OUT, keep)
    cmds = []
    try:
        for name, flags in CANDIDATES.items():
            os.environ["JSMPEG_B200_NVCC_FLAGS"] = flags
            build.build(force=True)
            dst = os.path.join(out_dir, f"lib_{name}.so")
            shutil.copy2(build.OUT, dst)
            cmds.append(f"echo {name}; JSMPEG_B200_LIB=$PWD/variants/lib_{name}.so timeout 100 python tools/time_stages.py 64 60 2 2>&1 | tail -1")
    finally:
        os.environ.pop("JSMPEG_B200_NVCC_FLAGS", None)
        if os.path.exists(keep):
            os.replace(keep, build.OUT)
    print("; ".join(cmds + cmds))
    print("\n# parity first, per variant:  JSMPEG_B200_LIB=$PWD/variants/lib_<name>.so python -m pytest tests/test_gpu_parity.py -m gpu -x -q",
          file=sys.stderr)


if __name__ == "__main__":
    main()
