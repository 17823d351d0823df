"""decode_frames_display's and flush_frames' contract without a GPU: both calls are declared and bound with their arity,
the wrapper refuses its bad arguments before it asks the library or allocates anything, sizes its info rows for
n_pictures + 1 frames and calls the display entry point (over a stand-in for the library), and the existing kernels'
SASS is what profiles/sass_hashes_sm90a.txt records: display order is host bookkeeping, no kernel changed."""
import ctypes
import os
import re

import pytest

import helpers
from jsmpeg_b200 import batch

HEADER = re.sub(r"/\*.*?\*/", "", open(os.path.join(helpers.ROOT, "include", "jsmpeg_b200.h")).read(), flags=re.S)


@pytest.mark.parametrize("name,arity,dst_at,info_at", [("jsmpeg_b200_batch_decode_frames_display", 6, 3, 4),
                                                       ("jsmpeg_b200_batch_flush_frames", 4, 1, 2)])
def test_the_calls_are_declared_and_bound_with_their_arity(name, arity, dst_at, info_at):
    m = re.search(r"\blong\s+" + name + r"\s*\(([^)]*)\)\s*;", HEADER)
    assert m
    restype, args = batch._BATCH_ABI[name]
    assert restype is ctypes.c_long and len(args) == len(m.group(1).split(",")) == arity
    assert args[dst_at] == ctypes.POINTER(batch.FrameDst) and args[info_at] == ctypes.POINTER(batch.Frame)
    assert "const jsmpeg_b200_frame_dst_t *dst" in m.group(1) and "int32_t *n_frames_out" in m.group(1)


class FakeLib:
    """Two streams, 320 x 240 with a sequence header; the display calls answer `answer` and report one frame each."""

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

    def _frames(self, info, n_frames, stride):
        for s in range(2):
            n_frames[s] = 1
            info[s * stride].picture_type = 1 + s

    def jsmpeg_b200_batch_decode_frames_display(self, handle, n, flags, dst, info, n_frames):
        self.calls.append(("display", n, flags))
        self._frames(info, n_frames, n + 1)
        return self.answer

    def jsmpeg_b200_batch_flush_frames(self, handle, dst, info, n_frames):
        self.calls.append(("flush",))
        self._frames(info, n_frames, 1)
        return self.answer

    def jsmpeg_b200_batch_decode_frames(self, handle, n, flags, planes, rgba, res, mb, info, n_frames):
        self.calls.append(("frames", n, flags))
        return self.answer


def test_wrapper_argument_errors():
    """Refused before the library is asked and before anything is allocated (no device is touched here)"""
    lib = FakeLib(0)
    bd = batch.BatchDecoder(2, lib=lib)
    with pytest.raises(ValueError):
        bd.decode_frames(-1, planes=False, display_order=True)
    with pytest.raises(ValueError, match="OUT_ACCUMULATED"):
        bd.decode_frames(2, batch.OUT_RGBA, planes=False, accumulated=True, display_order=True)
    assert lib.calls == [] and bd.last_frames_batch == {}
    lib.answer = -2
    with pytest.raises(ValueError):
        bd.decode_frames(0, planes=False, display_order=True)
    with pytest.raises(ValueError):
        bd.flush_frames(planes=False)
    lib.answer = -1
    with pytest.raises(RuntimeError):
        bd.flush_frames(planes=False)


def test_the_wrapper_makes_the_display_call_with_rows_of_n_plus_one():
    lib = FakeLib(3)
    bd = batch.BatchDecoder(2, lib=lib)
    out = bd.decode_frames(4, batch.OUT_MACROBLOCKS, planes=False, display_order=True)
    assert lib.calls == [("display", 4, batch.OUT_MACROBLOCKS)]
    assert [(o["n_frames"], [i["type"] for i in o["info"]]) for o in out] == [(1, [1]), (1, [2])]
    out = bd.flush_frames(planes=False)
    assert lib.calls[-1] == ("flush",) and [o["info"][0]["type"] for o in out] == [1, 2]
    bd.decode_frames(4, planes=False)  # (coded order: not the display call)
    assert lib.calls[-1] == ("frames", 4, 0)


def test_the_existing_kernels_keep_their_sass():
    """Every kernel profiles/sass_hashes_sm90a.txt records, from any product source (tools/sass_hash.py FILES), is still
    there and compiles to the recorded SASS"""
    import shutil
    if not (shutil.which("nvcc") and shutil.which("cuobjdump")):
        pytest.skip("nvcc / cuobjdump not available")
    import sass_hash
    recorded = {}
    for line in open(os.path.join(helpers.ROOT, "profiles", "sass_hashes_sm90a.txt")):
        parts = line.split()
        if len(parts) >= 3 and parts[0].endswith(".cu") and parts[1].endswith("_kernel"):  # (the project's own kernels)
            recorded[(parts[0], parts[1])] = next(p for p in parts[2:] if len(p) == 32)
    now = {}
    for cu in sass_hash.FILES:
        for name, (md5, _) in sass_hash.kernel_hashes(cu).items():
            now[(cu, sass_hash.demangle(name))] = md5
    assert len(recorded) > 20 and {k: now.get(k) for k in recorded} == recorded
