"""The macroblock index and the record conversion of tools/macroblock_model.py: literal index expectations (I/P
streams, B pictures without a chain start, f_code-0 P / D pictures, pictures before the sequence header, the unclosed
tail), the oracle's fresh decode of every listed picture pinned to its own sequential decode() (the records decode()
uses for that picture), and the device's conversion (jsmpeg_b200/csrc/macroblocks.cuh) built for the host against the
model's."""
import functools
import glob
import os
import shutil
import subprocess

import numpy as np
import pytest

import chain_model
import helpers
import intra_model
import macroblock_model
import synth_es
from jsmpeg_b200 import decoder


def pictures(es):
    return [p for p in intra_model.prefixes(es) if p + 3 < len(es) and es[p + 3] == 0]


def index_pairs(es):
    return [(e["picture"], e["type"]) for e in macroblock_model.macroblock_index(es)]


def ffmpeg_es(w, h, n, seed=1234):
    return b"".join(p for _, p in helpers.clip_packets(w, h, n, seed=seed))


@functools.lru_cache(maxsize=None)
def mini_enc_clip(f_codes=(3, 3), full_pel=(0, 0), gop_refs=None):
    """mini_enc I/P/B, 176x144, two B pictures per reference (gop_refs=2: an open GOP, coded I P B B I B B P ...)."""
    pytest.importorskip("cv2")
    import mini_enc
    if gop_refs:
        return mini_enc.make_b_clip(176, 144, 13, 2, gop_refs=gop_refs)[0]
    return mini_enc.make_b_clip(176, 144, 10, 2, f_codes=f_codes, full_pel=full_pel)[0]


def test_i_p_streams_literal():
    assert index_pairs(synth_es.make_case("rows_ip")) == \
        [(0, 1), (1, 2), (2, 2), (3, 2), (4, 1), (5, 2), (6, 2), (7, 2), (8, 1), (9, 2)]
    # FFmpeg, GOP 12: the last picture is never closed (no sequence end code)
    assert index_pairs(ffmpeg_es(320, 240, 24)) == [(k, 1 if k % 12 == 0 else 2) for k in range(23)]


def test_b_pictures_without_a_chain_start_are_listed():
    """b_rows: I B B P B B I B B P B B I.  Every picture is listed; the first two B pictures (one reference before them)
    have no chain start, so decode_pictures cannot reach them, with decode_b on or off."""
    es = synth_es.make_case("b_rows")
    assert index_pairs(es) == list(enumerate([1, 3, 3, 2, 3, 3, 1, 3, 3, 2, 3, 3, 1]))
    assert {1, 2}.isdisjoint(e["picture"] for e in chain_model.picture_index(es, True))
    assert not any(e["type"] == 3 for e in chain_model.picture_index(es, False))
    # an open GOP: coded I P B B I B B P B B I B B, every picture listed
    assert index_pairs(mini_enc_clip(gop_refs=2)) == list(enumerate([1, 2, 3, 3, 1, 3, 3, 2, 3, 3, 1, 3, 3]))


def test_ignored_pictures_are_not_listed():
    """ignored_pictures_userdata: I P P(forward_f_code 0) P I P D P I P D P -- the walks decode neither the f_code-0
    P picture nor the D pictures."""
    es = synth_es.make_case("ignored_pictures_userdata")
    assert index_pairs(es) == [(0, 1), (1, 2), (3, 2), (4, 1), (5, 2), (7, 2), (8, 1), (9, 2), (11, 2)]


def test_pictures_before_the_sequence_header_and_the_unclosed_tail_are_not_listed():
    es = synth_es.make_case("rows_ip")
    pics = pictures(es)
    lead = es[pics[1]:pics[2]]  # a P picture in front of the sequence header: picture 0, never listed
    assert index_pairs(lead + es) == [(k + 1, t) for k, t in index_pairs(es)]
    last = macroblock_model.macroblock_index(es)[-1]
    for cut in (last["close"], last["close"] + 3):
        assert last["picture"] not in [e["picture"] for e in macroblock_model.macroblock_index(es[:cut])]
    assert last in macroblock_model.macroblock_index(es[:last["close"] + 4])


@pytest.mark.parametrize("name", sorted(synth_es.CASES) + sorted(synth_es.B_CASES))
def test_the_index_holds_the_picture_index_with_b_pictures(name):
    """Every picture decode_pictures can reach (B pictures on) is listed here, with the same position and type."""
    es = synth_es.make_case(name)
    mine = {e["picture"]: (e["byte_pos"], e["type"], e["temporal_reference"], e["close"])
            for e in macroblock_model.macroblock_index(es)}
    for e in chain_model.picture_index(es, True):
        assert mine[e["picture"]] == (e["byte_pos"], e["type"], e["temporal_reference"], e["close"])


def _oracle():
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(1)
    return lib


def oracle_records(es, stop=None):
    """The oracle (B pictures on) fed `es`: [(start code position, picture_info, uint8 [mb_size, 16] records)] of every
    picture its decode() consumes, up to the one whose start code is at `stop`."""
    import ctypes
    lib = _oracle()
    try:
        d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=lib)
        d.write(0.0, [es])
        mb = lib.oracle_seq_params(d.decoder).contents.mb_size
        out = []
        while d.decode():
            info = lib.oracle_last_picture_info(d.decoder).contents
            rec = np.ctypeslib.as_array(ctypes.cast(lib.oracle_last_mb_records(d.decoder), ctypes.POINTER(ctypes.c_uint8)),
                                        shape=(mb * 16,)).reshape(mb, 16).copy()
            info = helpers.PictureInfo.from_buffer_copy(info)
            out.append((info.start_byte - 4, info, rec))
            if stop is not None and info.start_byte - 4 >= stop:
                break
        d.destroy()
    finally:
        lib.oracle_set_decode_b(0)
    return out


def oracle_fresh(es, entry):
    """(picture_info, records) of the oracle fed macroblock_model.fresh_bytes(es, entry): its first picture."""
    fresh = macroblock_model.fresh_bytes(es, entry)
    at = len(fresh) - (entry["close"] + 4 - entry["byte_pos"])
    got = oracle_records(fresh, stop=at)
    assert got and got[-1][0] == at
    return got[-1][1], got[-1][2]


GOLDEN = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(helpers.GOLDEN, "*.es")))


@functools.lru_cache(maxsize=None)
def corpus_stream(name):
    if name == "ffmpeg_320x240":
        return ffmpeg_es(320, 240, 24)
    if name == "ffmpeg_1280x720":
        return ffmpeg_es(1280, 720, 6)
    if name.startswith("mini_enc"):
        return mini_enc_clip(**MINI_ENC[name])
    return open(os.path.join(helpers.GOLDEN, name + ".es"), "rb").read()


MINI_ENC = {"mini_enc_open_gop": dict(gop_refs=2), "mini_enc_fcodes_2_4_fullpel_bwd": dict(f_codes=(2, 4), full_pel=(0, 1)),
            "mini_enc_fcodes_4_2_fullpel_fwd": dict(f_codes=(4, 2), full_pel=(1, 0))}


@pytest.mark.parametrize("name", GOLDEN + ["ffmpeg_320x240", "ffmpeg_1280x720"] + sorted(MINI_ENC))
def test_fresh_records_equal_the_sequential_decode(name):
    """For every picture the oracle's decode() consumes and decodes, the fresh decoder of that picture gives the same
    records and the same picture info; and the listed pictures are exactly the decoded ones that are closed."""
    es = corpus_stream(name)
    entries = macroblock_model.macroblock_index(es)
    by_pos = {e["byte_pos"]: e for e in entries}
    checked = 0
    for pos, info, rec in oracle_records(es):
        if info.status != 1:
            assert pos not in by_pos, (name, pos)
            continue
        if pos not in by_pos:  # only the unclosed tail
            assert pos == pictures(es)[-1], (name, pos)
            continue
        e = by_pos[pos]
        f_info, f_rec = oracle_fresh(es, e)
        assert (f_info.status, f_info.picture_type, f_info.n_present, f_info.error) == \
            (info.status, info.picture_type, info.n_present, info.error), (name, e["picture"])
        assert f_info.picture_type == e["type"]
        assert np.array_equal(macroblock_model.export(f_rec, e["type"]), macroblock_model.export(rec, e["type"])), \
            (name, e["picture"])
        checked += 1
    assert checked == len(entries) > 0, name


def test_the_conversion_compiled_for_the_host_equals_the_model(tmp_path):
    """macroblocks.cuh is the device's conversion; built with g++ it must give the model's entries for random records
    of all three picture types (every flag combination, any vector and field values)."""
    if not shutil.which("g++"):
        pytest.skip("g++ not available")
    exe = tmp_path / "macroblocks_check"
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", "-o", str(exe),
                        os.path.join(helpers.ROOT, "tests", "emu", "macroblocks_check.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    rng = np.random.default_rng(11)
    rec = rng.integers(0, 256, size=(4096, 16), dtype=np.uint8)
    rec[:32, 4] = np.arange(32)  # every combination of the five flags
    rec[32:, 4] &= 0x1f
    path = tmp_path / "records.bin"
    path.write_bytes(rec.tobytes())
    for picture_type in (1, 2, 3):
        out = subprocess.run([str(exe), str(path), str(picture_type)], capture_output=True, check=True).stdout
        got = np.frombuffer(out, np.uint8).reshape(-1, 16)
        want = macroblock_model.export(rec, picture_type)
        assert np.array_equal(got, want), picture_type
        flags = want[:, 8]
        assert not (want[(flags & 1) == 0] != 0).any()  # absent: all zero
        assert not want[:, 11:].any()  # reserved
        if picture_type != 3:
            assert ((flags & macroblock_model.MB_BACKWARD) == 0).all()
            assert (((flags & 0x03) == 0x01) == ((flags & macroblock_model.MB_FORWARD) != 0)).all()


def test_the_export_kernel_is_the_measured_one():
    """profiles/sass_hashes_sm90a.txt records the export kernel's SASS md5 (tools/sass_hash.py) on the build its H100
    numbers were taken with; recompiling macroblocks.cu must give the same machine code."""
    import sys
    if not (shutil.which("nvcc") and shutil.which("cuobjdump")):
        pytest.skip("nvcc / cuobjdump not available")
    sys.path.insert(0, os.path.join(helpers.ROOT, "tools"))
    import sass_hash
    line = next(x for x in open(os.path.join(helpers.ROOT, "profiles", "sass_hashes_sm90a.txt"))
                if "macroblocks.cu" in x and "export_macroblocks_kernel" in x)
    recorded = next(p for p in line.split() if len(p) == 32)
    now = {sass_hash.demangle(k): md5 for k, (md5, _) in sass_hash.kernel_hashes("macroblocks.cu").items()}
    assert now == {"export_macroblocks_kernel": recorded}
