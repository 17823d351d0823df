"""decode_frames_into's contract without a GPU: the call is declared and bound with its arity, jsmpeg_b200_frame_dst_t's
size and offsets are the ctypes mirror's, and the wrapper refuses map frames without OUT_ACCUMULATED (and a negative
count) before it asks the library or allocates anything, and makes decode_frames' own call when no new kind is asked
for (over a stand-in for the library)."""
import ctypes
import os
import re
import shutil
import subprocess
import tempfile

import pytest

import helpers
from jsmpeg_b200 import batch

HEADER = open(os.path.join(helpers.ROOT, "include", "jsmpeg_b200.h")).read()


def test_the_call_is_declared_and_bound_with_its_arity():
    code = re.sub(r"/\*.*?\*/", "", HEADER, flags=re.S)
    m = re.search(r"\blong\s+jsmpeg_b200_batch_decode_frames_into\s*\(([^)]*)\)\s*;", code)
    assert m
    restype, args = batch._BATCH_ABI["jsmpeg_b200_batch_decode_frames_into"]
    assert restype is ctypes.c_long and len(args) == len(m.group(1).split(",")) == 6
    assert args[3] == ctypes.POINTER(batch.FrameDst) and args[4] == ctypes.POINTER(batch.Frame)
    assert "const jsmpeg_b200_frame_dst_t *dst" in m.group(1)


def test_the_destination_struct_matches_the_mirror():
    """sizeof and offsetof of jsmpeg_b200_frame_dst_t as a C compiler lays it out, against the ctypes mirror"""
    cc = shutil.which("cc") or shutil.which("gcc")
    if not cc:
        pytest.skip("no C compiler")
    fields = [name for name, _ in batch.FrameDst._fields_]
    assert fields == ["planes", "rgba", "res", "mb", "coef", "acc"]
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "jsmpeg_b200.h"\nint main(void) {\n'
           '\tprintf("%zu", sizeof(jsmpeg_b200_frame_dst_t));\n' +
           "".join(f'\tprintf(" %zu", offsetof(jsmpeg_b200_frame_dst_t, {f}));\n' for f in fields) +
           # every member is an array of per-stream pointers: `void *const *`
           "".join(f"\t{{ void *const **p = &((jsmpeg_b200_frame_dst_t *)0)->{f}; (void)p; }}\n" for f in fields) +
           "\treturn 0;\n}\n")
    with tempfile.TemporaryDirectory() as tmp:
        c, exe = os.path.join(tmp, "layout.c"), os.path.join(tmp, "layout")
        with open(c, "w") as f:
            f.write(src)
        subprocess.check_call([cc, "-Wall", "-Werror", "-I", os.path.join(helpers.ROOT, "include"), "-o", exe, c])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [ctypes.sizeof(batch.FrameDst)] + [getattr(batch.FrameDst, f).offset for f in fields]
    assert got == [48, 0, 8, 16, 24, 32, 40]


class FakeLib:
    """Two streams, 320 x 240 with a sequence header; both frame calls answer `answer`."""

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
        self.calls.append(("frames", n, flags))
        return self.answer

    def jsmpeg_b200_batch_decode_frames_into(self, handle, n, flags, dst, info, n_frames):
        self.calls.append(("into", n, flags))
        return self.answer


def test_wrapper_argument_errors():
    """Refused before the library is asked and before anything is allocated (no device is touched here)"""
    lib = FakeLib(0)
    bd = batch.BatchDecoder(2, lib=lib)
    with pytest.raises(ValueError, match="OUT_ACCUMULATED"):
        bd.decode_frames(0, planes=False, accumulated=True)
    with pytest.raises(ValueError, match="OUT_ACCUMULATED"):
        bd.decode_frames(1, batch.OUT_RGBA | batch.OUT_HOST | batch.OUT_RESIDUALS, accumulated=True, coefficients=True)
    with pytest.raises(ValueError):
        bd.decode_frames(-1, batch.OUT_ACCUMULATED, accumulated=True)
    with pytest.raises(ValueError):
        bd.decode_frames(-1, coefficients=True)
    assert lib.calls == [] and bd.last_frames_batch == {}


def test_the_old_kinds_make_the_old_call():
    lib = FakeLib(0)
    bd = batch.BatchDecoder(2, lib=lib)
    assert [o["n_frames"] for o in bd.decode_frames(0, planes=False)] == [0, 0]
    bd.decode_frames(0, batch.OUT_ACCUMULATED, planes=False)
    assert lib.calls == [("frames", 0, 0), ("frames", 0, batch.OUT_ACCUMULATED)]
    lib.answer = -2
    with pytest.raises(ValueError):
        bd.decode_frames(0, planes=False)
