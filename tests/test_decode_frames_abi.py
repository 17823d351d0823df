"""decode_frames' contract without a GPU: the call is declared and bound with its arity, jsmpeg_b200_frame_t's size and
offsets are the ctypes mirror's, the wrapper refuses a negative count before it asks the library (over a stand-in for
it) and turns the library's refusals into errors, and the four FRAME variants of the reconstruct kernels are the machine
code whose H100 numbers are recorded (profiles/sass_hashes_sm90a.txt)."""
import ctypes
import os
import re
import shutil
import subprocess
import sys
import tempfile

import pytest

import helpers
from jsmpeg_b200 import batch

HEADER = open(os.path.join(helpers.ROOT, "include", "jsmpeg_b200.h")).read()
FRAME_KERNELS = ["reconstruct_frame_kernel", "reconstruct_rgba_frame_kernel", "reconstruct_frame_b_kernel",
                 "reconstruct_rgba_frame_b_kernel"]


def test_the_call_is_declared_and_bound_with_its_arity():
    code = re.sub(r"/\*.*?\*/", "", HEADER, flags=re.S)
    m = re.search(r"\blong\s+jsmpeg_b200_batch_decode_frames\s*\(([^)]*)\)\s*;", code)
    assert m
    restype, args = batch._BATCH_ABI["jsmpeg_b200_batch_decode_frames"]
    assert restype is ctypes.c_long and len(args) == len(m.group(1).split(",")) == 9
    assert args[7] == ctypes.POINTER(batch.Frame)


def test_the_frame_struct_matches_the_mirror():
    """sizeof and offsetof of jsmpeg_b200_frame_t as a C compiler lays it out, against the ctypes mirror"""
    cc = shutil.which("cc") or shutil.which("gcc")
    if not cc:
        pytest.skip("no C compiler")
    fields = [name for name, _ in batch.Frame._fields_]
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "jsmpeg_b200.h"\nint main(void) {\n'
           '\tprintf("%zu", sizeof(jsmpeg_b200_frame_t));\n' +
           "".join(f'\tprintf(" %zu", offsetof(jsmpeg_b200_frame_t, {f}));\n' for f in fields) + "\treturn 0;\n}\n")
    with tempfile.TemporaryDirectory() as tmp:
        c, exe = os.path.join(tmp, "layout.c"), os.path.join(tmp, "layout")
        with open(c, "w") as f:
            f.write(src)
        subprocess.check_call([cc, "-I", os.path.join(helpers.ROOT, "include"), "-o", exe, c])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [ctypes.sizeof(batch.Frame)] + [getattr(batch.Frame, f).offset for f in fields]
    assert got[0] == 16


class FakeLib:
    """Two streams, 320 x 240 with a sequence header; decode_frames answers `answer`."""

    def __init__(self, answer):
        self.answer = answer
        self.calls = []

    def jsmpeg_b200_batch_create(self, n, device, max_slots):
        return 1

    def jsmpeg_b200_batch_last_error(self, handle):
        return None

    def jsmpeg_b200_batch_destroy(self, handle):
        pass

    def jsmpeg_b200_batch_stream_info(self, handle, s, w, h, cs, fr):
        w.value, h.value, cs.value = 320, 240, 320 * 240
        return 1

    def jsmpeg_b200_batch_decode_frames(self, handle, n, flags, planes, rgba, res, mb, info, n_frames):
        self.calls.append((n, flags))
        return self.answer


def test_wrapper_argument_errors():
    lib = FakeLib(-2)
    bd = batch.BatchDecoder(2, lib=lib)
    with pytest.raises(ValueError):
        bd.decode_frames(-1)
    assert lib.calls == []  # refused before the library is asked
    with pytest.raises(ValueError):  # the library's -2
        bd.decode_frames(0, planes=False)
    lib.answer = -1
    with pytest.raises(RuntimeError):  # a dead batch is no ValueError
        bd.decode_frames(0, batch.OUT_RGBA, planes=False)
    assert lib.calls == [(0, 0), (0, batch.OUT_RGBA)]


def test_the_frame_kernels_are_the_measured_ones():
    """profiles/sass_hashes_sm90a.txt records the SASS md5 (tools/sass_hash.py) of the four FRAME variants on the build
    their H100 numbers were taken with; recompiling recon.cu must give the same machine code."""
    if not (shutil.which("nvcc") and shutil.which("cuobjdump")):
        pytest.skip("nvcc / cuobjdump not available")
    sys.path.insert(0, os.path.join(helpers.ROOT, "tools"))
    import sass_hash
    recorded = {}
    for line in open(os.path.join(helpers.ROOT, "profiles", "sass_hashes_sm90a.txt")):
        parts = line.split()
        if len(parts) >= 3 and parts[0] == "recon.cu" and parts[1] in FRAME_KERNELS:
            recorded[parts[1]] = next(p for p in parts[2:] if len(p) == 32)
    assert sorted(recorded) == sorted(FRAME_KERNELS)
    now = {sass_hash.demangle(k): md5 for k, (md5, _) in sass_hash.kernel_hashes("recon.cu").items()}
    assert {k: now.get(k) for k in FRAME_KERNELS} == recorded
