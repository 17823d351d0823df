"""The coefficient export of decode_coefficients WITHOUT a GPU: the row conversion of the compact records
(coef_record_row, jsmpeg_b200/csrc/coef_records.h) built with g++ against numpy unpacking; the oracle's fresh decode of
every listed picture pinned to its own sequential decode() through macroblock_model.coefficients (the coefficient twin
of test_macroblock_index.py's record test); and the export kernel's recorded SASS hash."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import helpers
import macroblock_model
from jsmpeg_b200 import decoder
from test_compact_records import RECORD, ZIG_ZAG
from test_macroblock_index import GOLDEN, MINI_ENC, corpus_stream, pictures


def numpy_unpack(rec):
    """[n, 64] raster values of n compact records: the k-th set bit of the mask takes level[k]"""
    out = np.zeros((len(rec), 64), np.int16)
    for i, r in enumerate(rec):
        pos = [k for k in range(64) if (int(r["mask"]) >> k) & 1]
        out[i, ZIG_ZAG[pos]] = r["level"][:len(pos)]
    return out


def random_records(rng, n=3000):
    """Compact records with 0 to 12 positions at random zig-zag places (position 63 and the full twelve included), any
    level values, and garbage in the unused levels (the conversion must not read them)"""
    rec = np.zeros(n, RECORD)
    rec["level"] = rng.integers(-32768, 32768, size=(n, 12))
    for i in range(n):
        k = i % 13
        pos = rng.choice(64, size=k, replace=False)
        if i % 5 == 0 and k and 63 not in pos:
            pos[0] = 63
        rec["mask"][i] = sum(1 << int(p) for p in pos)
    rec["mask"][-3] = sum(1 << p for p in range(52, 64))  # twelve positions ending at 63
    rec["mask"][-2] = (1 << 63) | 1
    rec["mask"][-1] = 0
    return rec


def test_the_row_conversion_compiled_for_the_host_equals_numpy_unpacking(tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not available")
    exe = tmp_path / "coefficients_check"
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", "-o", str(exe),
                        os.path.join(helpers.ROOT, "tests", "emu", "coefficients_check.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    rec = random_records(np.random.default_rng(3))
    path = tmp_path / "records.bin"
    path.write_bytes(rec.tobytes())
    out = subprocess.run([str(exe), str(path)], capture_output=True, check=True).stdout
    got = np.frombuffer(out, np.int16).reshape(-1, 64)
    assert np.array_equal(got, numpy_unpack(rec))


def oracle_coefficients(es, stop=None):
    """The oracle (B pictures on) fed `es`: [(start code position, picture_info, records, int16 coefficient plane)] of
    every picture its decode() consumes, up to the one whose start code is at `stop`."""
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(1)
    try:
        d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=lib)
        d.write(0.0, [es])
        mb = lib.oracle_seq_params(d.decoder).contents.mb_size
        out = []
        while d.decode():
            info = helpers.PictureInfo.from_buffer_copy(lib.oracle_last_picture_info(d.decoder).contents)
            rec = np.ctypeslib.as_array(ctypes.cast(lib.oracle_last_mb_records(d.decoder), ctypes.POINTER(ctypes.c_uint8)),
                                        shape=(mb * 16,)).reshape(mb, 16).copy()
            coef = np.ctypeslib.as_array(ctypes.cast(lib.oracle_last_coefficients(d.decoder), ctypes.POINTER(ctypes.c_int16)),
                                         shape=(mb * 6 * 64,)).copy()
            out.append((info.start_byte - 4, info, rec, coef))
            if stop is not None and info.start_byte - 4 >= stop:
                break
        d.destroy()
    finally:
        lib.oracle_set_decode_b(0)
    return out


def oracle_fresh_coefficients(es, entry):
    """(picture_info, records, int16 [mb_size, 6, 64]) of the oracle fed macroblock_model.fresh_bytes(es, entry): its
    first picture, through macroblock_model.coefficients."""
    fresh = macroblock_model.fresh_bytes(es, entry)
    at = len(fresh) - (entry["close"] + 4 - entry["byte_pos"])
    got = oracle_coefficients(fresh, stop=at)
    assert got and got[-1][0] == at
    _, info, rec, coef = got[-1]
    return info, rec, macroblock_model.coefficients(rec, coef)


@pytest.mark.parametrize("name", GOLDEN + ["ffmpeg_320x240", "ffmpeg_1280x720"] + sorted(MINI_ENC))
def test_fresh_coefficients_equal_the_sequential_decode(name):
    """For every picture the oracle's decode() consumes and decodes, the fresh decoder of that picture gives the same
    coefficients (zero outside coded blocks); the listed pictures are exactly the decoded ones that are closed."""
    es = corpus_stream(name)
    by_pos = {e["byte_pos"]: e for e in macroblock_model.macroblock_index(es)}
    checked = coded = 0
    for pos, info, rec, coef in oracle_coefficients(es):
        if info.status != 1 or pos not in by_pos:
            assert info.status != 1 or pos == pictures(es)[-1], (name, pos)  # only the unclosed tail
            continue
        want = macroblock_model.coefficients(rec, coef)
        _, _, got = oracle_fresh_coefficients(es, by_pos[pos])
        assert np.array_equal(got, want), (name, by_pos[pos]["picture"])
        checked += 1
        coded += int(want.any())
    assert checked == len(by_pos) > 0 and coded > 0, name


def test_the_model_zeroes_uncoded_blocks_and_absent_macroblocks():
    rec = np.zeros((3, 16), np.uint8)
    rec[0, 4], rec[0, 5] = macroblock_model.MBF_PRESENT, 0b100001  # blocks 0 and 5 coded
    rec[1, 4], rec[1, 5] = 0, 0x3F                                  # absent: cbp ignored
    rec[2, 4], rec[2, 5] = macroblock_model.MBF_PRESENT | macroblock_model.MBF_INTRA, 0x3F
    coef = np.arange(3 * 6 * 64, dtype=np.int16) + 1
    got = macroblock_model.coefficients(rec, coef)
    want = coef.reshape(3, 6, 64).copy()
    want[0, 1:5] = 0
    want[1] = 0
    assert got.dtype == np.int16 and np.array_equal(got, want)


def test_the_export_kernel_is_the_measured_one():
    """profiles/sass_hashes_sm90a.txt records the coefficient export kernel's SASS md5 (tools/sass_hash.py) on the build
    its H100 numbers were taken with; recompiling coefficients.cu must give the same machine code."""
    import sys
    if not (shutil.which("nvcc") and shutil.which("cuobjdump")):
        pytest.skip("nvcc / cuobjdump not available")
    sys.path.insert(0, os.path.join(helpers.ROOT, "tools"))
    import sass_hash
    line = next(x for x in open(os.path.join(helpers.ROOT, "profiles", "sass_hashes_sm90a.txt"))
                if "coefficients.cu" in x and "export_coefficients_kernel" in x)
    recorded = next(p for p in line.split() if len(p) == 32)
    now = {sass_hash.demangle(k): md5 for k, (md5, _) in sass_hash.kernel_hashes("coefficients.cu").items()}
    assert now == {"export_coefficients_kernel": recorded}
