"""The OUT_RESIDUALS contract without a GPU: the flag is a bit of its own, the two calls are declared and bound with
their arity, the wrappers refuse a stream out of range or without a sequence header before they ask the library (over a
stand-in for it), and the four RES variants of the reconstruct kernels are the machine code whose H100 numbers are
recorded (profiles/sass_hashes_sm90a.txt)."""
import ctypes
import os
import re
import shutil
import sys

import numpy as np
import pytest

import helpers
from jsmpeg_b200 import batch

HEADER = open(os.path.join(helpers.ROOT, "include", "jsmpeg_b200.h")).read()
NEW = ["jsmpeg_b200_batch_get_residuals", "jsmpeg_b200_batch_read_residuals"]
RES_KERNELS = ["reconstruct_res_kernel", "reconstruct_rgba_res_kernel", "reconstruct_res_b_kernel",
               "reconstruct_rgba_res_b_kernel"]


def header_flags():
    """{name: value} of every JSMPEG_B200_OUT_* macro of the header: a number, a parenthesised shift or a parenthesised
    hexadecimal number"""
    out = {}
    for name, value in re.findall(r"#define JSMPEG_B200_(OUT_\w+)\s+(\d+|\(\s*\d+\s*<<\s*\d+\s*\)|\(\s*0x[0-9a-fA-F]+\s*\))",
                                  HEADER):
        if "0x" in value:
            out[name] = int(value.strip("() "), 16)
        else:
            terms = [int(x) for x in re.findall(r"\d+", value)]
            out[name] = terms[0] << terms[1] if len(terms) == 2 else terms[0]
    return out


def test_the_flag_is_a_bit_of_its_own():
    flags = header_flags()
    assert flags == {"OUT_DEVICE": 0, "OUT_HOST": 1, "OUT_RGBA": 2, "OUT_MACROBLOCKS": 4, "OUT_ACCUMULATED": 8,
                     "OUT_RESIDUALS": 16}
    assert batch.OUT_RESIDUALS == flags["OUT_RESIDUALS"]
    others = batch.OUT_HOST | batch.OUT_RGBA | batch.OUT_MACROBLOCKS | batch.OUT_ACCUMULATED
    assert batch.OUT_RESIDUALS & others == 0 and bin(batch.OUT_RESIDUALS).count("1") == 1


def test_the_new_calls_are_declared_and_bound_with_their_arity():
    code = re.sub(r"/\*.*?\*/", "", HEADER, flags=re.S)
    for name in NEW:
        m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", code)
        assert m, name
        assert len(batch._BATCH_ABI[name][1]) == len(m.group(1).split(",")), name
        assert batch._BATCH_ABI[name][0] is ctypes.c_int, name


class FakeLib:
    """Stream 0 is 320 x 240 with a sequence header, stream 1 has none."""

    N = 320 * 240 * 3 // 2

    def __init__(self):
        self.calls = []

    def jsmpeg_b200_batch_create(self, n, device, max_slots):
        return 1

    def jsmpeg_b200_batch_last_error(self, handle):
        return None

    def jsmpeg_b200_batch_destroy(self, handle):
        pass

    def jsmpeg_b200_batch_stream_info(self, handle, s, w, h, cs, fr):
        w.value, h.value, cs.value = (320, 240, 320 * 240) if s == 0 else (0, 0, 0)
        return 1 if s == 0 else 0

    def jsmpeg_b200_batch_get_residuals(self, handle, s, out):
        self.calls.append(s)
        return -1

    def jsmpeg_b200_batch_read_residuals(self, handle, s, dst):
        self.calls.append(s)
        ctypes.memset(dst, 0xff, self.N * 2)
        return 0


def test_wrappers_refuse_streams_out_of_range_or_without_a_sequence_header():
    lib = FakeLib()
    bd = batch.BatchDecoder(2, lib=lib)
    for s in (-1, 1, 2):
        for call in (bd.device_residuals, bd.read_residuals):
            with pytest.raises(ValueError):
                call(s)
    assert lib.calls == []  # refused before the library is asked
    got = bd.read_residuals(0)
    assert got.shape == (FakeLib.N,) and got.dtype == np.int16 and (got == -1).all()
    with pytest.raises(RuntimeError):  # a failing library call is no ValueError
        bd.device_residuals(0)
    assert lib.calls == [0, 0]


def test_the_residual_kernels_are_the_measured_ones():
    """profiles/sass_hashes_sm90a.txt records the SASS md5 (tools/sass_hash.py) of the four RES variants on the build
    their H100 numbers were taken with; recompiling recon.cu must give the same machine code."""
    if not (shutil.which("nvcc") and shutil.which("cuobjdump")):
        pytest.skip("nvcc / cuobjdump not available")
    sys.path.insert(0, os.path.join(helpers.ROOT, "tools"))
    import sass_hash
    recorded = {}
    for line in open(os.path.join(helpers.ROOT, "profiles", "sass_hashes_sm90a.txt")):
        parts = line.split()
        if len(parts) >= 3 and parts[0] == "recon.cu" and parts[1] in RES_KERNELS:
            recorded[parts[1]] = next(p for p in parts[2:] if len(p) == 32)
    assert sorted(recorded) == sorted(RES_KERNELS)
    now = {sass_hash.demangle(k): md5 for k, (md5, _) in sass_hash.kernel_hashes("recon.cu").items()}
    assert {k: now.get(k) for k in RES_KERNELS} == recorded
