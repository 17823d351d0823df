#!/usr/bin/env python
"""md5 of the SASS instruction stream of every product kernel (addresses and encodings stripped).
Used to show that a source change left the machine code of a GPU-verified kernel untouched
(profiles/sass_hashes_sm90a.txt lists the hashes of the build the H100 numbers were taken with).

    python tools/sass_hash.py [--csrc DIR] [extra nvcc flags...]
"""
import hashlib
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "jsmpeg_b200", "csrc")
FILES = ("parse.cu", "recon.cu", "scan.cu", "tsdemux.cu")


def kernel_hashes(cu, csrc=CSRC, flags=()):
    """{kernel name: (md5, instruction count)} for one .cu file."""
    with tempfile.TemporaryDirectory() as tmp:
        cubin = os.path.join(tmp, "k.cubin")
        subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", *flags,
                               "-cubin", "-o", cubin, os.path.join(csrc, cu)])
        sass = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True, check=True).stdout
    out, name, lines = {}, None, []

    def close():
        if name is not None:
            out[name] = (hashlib.md5(("\n".join(lines) + "\n").encode()).hexdigest(), len(lines))

    for l in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", l)
        if m:
            close()
            name, lines = m.group(1), []
        elif re.match(r"^\s+/\*[0-9a-f]{4,5}\*/", l):
            lines.append(re.sub(r"^\s+/\*[0-9a-f]{4,5}\*/\s*", "", l).split("/*")[0].rstrip())
    close()
    return out


def demangle(name):
    r = subprocess.run(["cu++filt", name], capture_output=True, text=True)
    s = r.stdout.strip() if r.returncode == 0 and r.stdout.strip() else name
    return s.split("(")[0].split("::")[-1]


if __name__ == "__main__":
    args = sys.argv[1:]
    csrc = CSRC
    if args[:1] == ["--csrc"]:
        csrc, args = args[1], args[2:]
    for cu in FILES:
        if not os.path.exists(os.path.join(csrc, cu)):
            continue
        for name, (h, n) in sorted(kernel_hashes(cu, csrc, args).items(), key=lambda kv: demangle(kv[0])):
            print(f"{cu:12s} {demangle(name):34s} {h}  ({n} instructions)")
