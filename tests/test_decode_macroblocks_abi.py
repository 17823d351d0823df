"""The OUT_MACROBLOCKS contract without a GPU: the flag's value, the declarations and their Python prototypes, and the
wrappers' argument errors (over a stand-in for the library)."""
import ctypes
import os
import re

import pytest

import helpers
from jsmpeg_b200 import batch, decoder

HEADER = open(os.path.join(helpers.ROOT, "include", "jsmpeg_b200.h")).read()
NEW = ["jsmpeg_b200_batch_get_macroblocks", "jsmpeg_b200_batch_read_macroblocks", "jsmpeg_b200_batch_get_host_macroblocks",
       "jsmpeg_b200_decoder_get_macroblocks"]


def test_the_flag_is_a_bit_of_its_own():
    flags = {name: int(value) for name, value in re.findall(r"#define JSMPEG_B200_(OUT_\w+)\s+(\d+)", HEADER)}
    assert flags == {"OUT_DEVICE": 0, "OUT_HOST": 1, "OUT_RGBA": 2, "OUT_MACROBLOCKS": 4}
    assert batch.OUT_MACROBLOCKS == flags["OUT_MACROBLOCKS"]
    assert batch.OUT_MACROBLOCKS & (batch.OUT_HOST | batch.OUT_RGBA) == 0


def test_the_new_calls_are_declared_and_bound_with_their_arity():
    code = re.sub(r"/\*.*?\*/", "", HEADER, flags=re.S)
    for name in NEW:
        m = re.search(r"\b" + name + r"\s*\(([^)]*)\)\s*;", code)
        assert m, name
        assert len(batch._BATCH_ABI[name][1]) == len(m.group(1).split(",")), name
    assert batch._BATCH_ABI["jsmpeg_b200_decoder_get_macroblocks"][0] is ctypes.c_void_p


class FakeLib:
    """Stream 0 is 320 x 240 with a sequence header, stream 1 has none; the entries are a host buffer."""

    def __init__(self):
        self.entries = (ctypes.c_uint8 * (15 * 20 * 16))()
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

    def jsmpeg_b200_batch_get_host_macroblocks(self, handle, s, out):
        self.calls.append(s)
        out._obj.value = ctypes.addressof(self.entries)
        return 0

    def jsmpeg_b200_batch_read_macroblocks(self, handle, s, dst):
        self.calls.append(s)
        ctypes.memset(dst, 7, 15 * 20 * 16)
        return 0


def test_wrappers_refuse_streams_out_of_range_or_without_a_sequence_header():
    lib = FakeLib()
    bd = batch.BatchDecoder(2, lib=lib)
    for s in (-1, 1, 2):
        for call in (bd.device_macroblocks, bd.read_macroblocks, bd.host_macroblocks):
            with pytest.raises(ValueError):
                call(s)
    assert lib.calls == []  # refused before the library is asked
    assert bd.host_macroblocks(0).shape == (15, 20, 16)
    got = bd.read_macroblocks(0)
    assert got.shape == (15, 20, 16) and (got == 7).all()


def test_decoder_surface_without_the_option_has_no_entries():
    class Lib:
        def mpeg1_decoder_create(self, size, mode):
            return 1

        def jsmpeg_b200_decoder_get_macroblocks(self, d):
            raise AssertionError("not asked without exportMacroblocks")

    d = decoder.MPEG1Video({}, lib=Lib())
    assert d.macroblocks() is None
