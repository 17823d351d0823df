"""The OUT_ACCUMULATED contract without a GPU: the output flags are bits of their own, the two calls are declared and
bound with their arity, and the wrappers refuse a stream out of range or without a sequence header before they ask the
library (over a stand-in for it)."""
import ctypes
import os
import re

import numpy as np
import pytest

import helpers
from jsmpeg_b200 import batch

HEADER = open(os.path.join(helpers.ROOT, "include", "jsmpeg_b200.h")).read()
NEW = ["jsmpeg_b200_batch_get_accumulated", "jsmpeg_b200_batch_read_accumulated"]


def header_flags():
    """{name: value} of every JSMPEG_B200_OUT_* macro of the header: a number, or a parenthesised shift of two"""
    out = {}
    for name, value in re.findall(r"#define JSMPEG_B200_(OUT_\w+)\s+(\d+|\(\s*\d+\s*<<\s*\d+\s*\))", HEADER):
        terms = [int(x) for x in re.findall(r"\d+", value)]
        out[name] = terms[0] << terms[1] if len(terms) == 2 else terms[0]
    return out


def test_the_flag_is_a_bit_of_its_own():
    flags = header_flags()
    assert flags == {"OUT_DEVICE": 0, "OUT_HOST": 1, "OUT_RGBA": 2, "OUT_MACROBLOCKS": 4, "OUT_ACCUMULATED": 8}
    assert batch.OUT_ACCUMULATED == flags["OUT_ACCUMULATED"]
    assert batch.OUT_MACROBLOCKS == flags["OUT_MACROBLOCKS"]
    assert batch.OUT_ACCUMULATED & (batch.OUT_HOST | batch.OUT_RGBA | batch.OUT_MACROBLOCKS) == 0


def test_the_new_calls_are_declared_and_bound_with_their_arity():
    code = re.sub(r"/\*.*?\*/", "", HEADER, flags=re.S)
    for name in NEW:
        m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", code)
        assert m, name
        assert len(batch._BATCH_ABI[name][1]) == len(m.group(1).split(",")), name
        assert batch._BATCH_ABI[name][0] is ctypes.c_int, name


class FakeLib:
    """Stream 0 is 320 x 240 with a sequence header, stream 1 has none."""

    N_REC = 320 * 240 * 3 // 2

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

    def jsmpeg_b200_batch_get_accumulated(self, handle, s, out):
        self.calls.append(s)
        return -1

    def jsmpeg_b200_batch_read_accumulated(self, handle, s, dst):
        self.calls.append(s)
        ctypes.memset(dst, 0xff, self.N_REC * 8)
        return 0


def test_wrappers_refuse_streams_out_of_range_or_without_a_sequence_header():
    lib = FakeLib()
    bd = batch.BatchDecoder(2, lib=lib)
    for s in (-1, 1, 2):
        for call in (bd.device_accumulated, bd.read_accumulated):
            with pytest.raises(ValueError):
                call(s)
    assert lib.calls == []  # refused before the library is asked
    got = bd.read_accumulated(0)
    assert got.shape == (FakeLib.N_REC, 4) and got.dtype == np.int16 and (got == -1).all()
    with pytest.raises(RuntimeError):  # a failing library call is no ValueError
        bd.device_accumulated(0)
    assert lib.calls == [0, 0]
