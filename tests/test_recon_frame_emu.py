"""Stage 2's decode_frames variant (reconstruct_at<..., FRAME = true>, jsmpeg_b200/csrc/recon.cuh, DESIGN 3.16) WITHOUT a
GPU.  tests/emu/recon_frame_check.cpp builds the device code for the host (the emulation of test_compact_records) and
runs walk -> expand -> reconstruct for I, P and B pictures through the plain code, the RES variant and the FRAME
variant, in the plain kernel's numbering and in the RGBA kernel's, on every kind of stream the suite has, clean and
bit-flipped:
  * the FRAME variant's planes are the plain ones, with a planar frame, a residual, both or neither;
  * its planar frame is the planes, every byte of it, absent macroblocks included (the rows the set keeps);
  * its residual is the RES variant's;
  * in the RGBA kernel's numbering the rows it hands the epilogue are the RES variant's;
  * P pictures whose vectors are pushed out of the plane take the per-tap path.
"""
import os
import subprocess

import numpy as np
import pytest

import helpers
import macroblock_model
from test_compact_records import GOLDEN, RECORD, stream_geometry
from test_recon_residual_emu import outside_blocks

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_SRC = os.path.join(HERE, "emu", "recon_frame_check.cpp")
CSRC = os.path.join(HERE, "..", "jsmpeg_b200", "csrc")
SENTINEL = 0x5A  # what a destination holds before the variant writes it


def frame_lib():
    import ctypes
    out = os.path.join(HERE, "emu", "librecon_frame_check.so")
    deps = [EMU_SRC, os.path.join(HERE, "emu", "compact_emu.cpp"), os.path.join(HERE, "emu", "walk_emu.cpp")] + \
        [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        tmp = out + ".%d.tmp" % os.getpid()
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-Wno-attributes",
                               "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-o", tmp, EMU_SRC])
        os.replace(tmp, out)
    lib = ctypes.CDLL(out)
    vp, i, u32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32
    lib.emu_walk_picture.argtypes = [vp, u32, u32, i, i, vp, vp, vp, i]
    lib.emu_walk_picture_b.argtypes = [vp, u32, u32, i, i, vp, vp, vp]
    lib.emu_expand_picture_compact.argtypes = [vp, u32, i, i, vp, vp, vp, vp, vp]
    lib.emu_reconstruct_picture_compact.argtypes = [vp, vp, vp, vp, vp, vp, i, i]
    lib.emu_reconstruct_picture_frame.argtypes = [vp, vp, vp, vp, vp, vp, i, i, vp, vp, i, vp]
    return lib


def ptr(a):
    return None if a is None else a.ctypes.data


def frame_pipeline(es, name, push_out=False):
    """The emulated pipeline with the product's plane bookkeeping (test_recon_residual_emu.residual_pipeline), every
    decoded picture reconstructed by the plain code and by the FRAME variant in both numberings.  push_out: as there.
    Returns per-kind counts."""
    from jsmpeg_b200 import decoder
    olib = helpers.oracle_lib()
    olib.oracle_set_decode_b(1)
    lib = frame_lib()
    seen = {"pictures": 0, "b": 0, "absent": 0, "outside": 0}
    try:
        d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=olib)
        d.write(0, [es])
        seq = olib.oracle_seq_params(d.decoder).contents
        mb = seq.mb_size
        lib.emu_set_quant(bytes(seq.intra_q), bytes(seq.non_intra_q))
        mbw, mbh = stream_geometry(es)
        buf = np.frombuffer(es + b"\0" * 16, dtype=np.uint8).copy()
        ysize = mb * 256
        n = ysize * 3 // 2
        size = n + mbw * 16 + 64
        planes = [np.zeros(size, dtype=np.uint8) for _ in range(2)]
        planes_b = np.zeros(size, dtype=np.uint8)
        cur = 0
        while d.decode():
            info = olib.oracle_last_picture_info(d.decoder).contents
            is_b = ((es[info.start_byte + 1] >> 3) & 7) == 3
            hdr = np.zeros(mb * 4, dtype=np.uint32)
            park = np.zeros(mb * 6 * 2, dtype=np.uint32)
            pinfo = np.zeros(12, dtype=np.int32)
            if is_b:
                lib.emu_walk_picture_b(buf.ctypes.data, len(es), info.start_byte, mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                                       pinfo.ctypes.data)
            else:
                lib.emu_walk_picture(buf.ctypes.data, len(es), info.start_byte, mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                                     pinfo.ctypes.data, 1)
            if pinfo[2] != 1:
                continue
            coef = np.zeros(mb * 6 * 64, dtype=np.int16)
            compact = np.zeros(mb * 6, dtype=RECORD)
            lib.emu_expand_picture_compact(buf.ctypes.data, len(es), mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                                           coef.ctypes.data, compact.ctypes.data, pinfo.ctypes.data)
            if push_out and info.picture_type == 2:
                rows = (np.arange(mb) // mbw) % 2 == 0
                hdr.reshape(mb, 4)[rows, 0] = np.uint32((0xFFC0 << 16) | 0xFFC0)  # (int16 -64, int16 -64)
            if is_b:
                out, fwd, bwd = planes_b, planes[cur], planes[cur ^ 1]
            else:
                out, fwd, bwd = planes[cur], planes[cur ^ 1], None
            before = out.copy()
            lib.emu_reconstruct_picture_compact(hdr.ctypes.data, coef.ctypes.data, compact.ctypes.data, out.ctypes.data,
                                                fwd.ctypes.data, ptr(bwd), mbw, mbh)
            label = f"{name}: picture {seen['pictures']} (type {info.picture_type})"

            def run(variant, with_res, with_frame, rows=None):
                o = before.copy()
                res = np.full(n, SENTINEL, dtype=np.int16) if with_res else None
                frame = np.full(n, SENTINEL, dtype=np.uint8) if with_frame else None
                lib.emu_reconstruct_picture_frame(hdr.ctypes.data, coef.ctypes.data, compact.ctypes.data, o.ctypes.data,
                                                  fwd.ctypes.data, ptr(bwd), mbw, mbh, ptr(res), ptr(frame), variant, ptr(rows))
                return o, res, frame

            _, want_res, _ = run(0, True, False)  # the RES variant
            for with_res in (False, True):
                for with_frame in (False, True):
                    o, res, frame = run(1, with_res, with_frame)
                    assert np.array_equal(o, out), (label, "planes", with_res, with_frame)
                    if with_res:
                        assert np.array_equal(res, want_res), (label, "residual", with_frame)
                    if with_frame:
                        assert np.array_equal(frame, out[:n]), (label, "frame", with_res)
            keep_rows = np.zeros(mb * 6 * 8 * 2, dtype=np.uint32)
            o_keep, res_keep, _ = run(0, True, False, keep_rows)  # the RGBA kernel's numbering, RES variant
            assert np.array_equal(o_keep, out) and np.array_equal(res_keep, want_res), label
            frame_rows = np.zeros_like(keep_rows)
            o, res, frame = run(1, True, True, frame_rows)
            assert np.array_equal(o, out), (label, "planes, RGBA numbering")
            assert np.array_equal(frame_rows, keep_rows), (label, "the epilogue's rows")
            assert np.array_equal(res, want_res), (label, "residual, RGBA numbering")
            assert np.array_equal(frame, out[:n]), (label, "frame, RGBA numbering")
            if not is_b:
                cur ^= 1
            flags = hdr.view(np.uint8).reshape(mb, 16)[:, 4]
            seen["absent"] += int(((flags & macroblock_model.MBF_PRESENT) == 0).sum())
            if info.picture_type == 2:
                seen["outside"] += outside_blocks(hdr, mbw, mbh)
            seen["b"] += int(is_b)
            seen["pictures"] += 1
        d.destroy()
    finally:
        olib.oracle_set_decode_b(0)
    assert seen["pictures"] > 0, name
    return seen


def _sum(a, b):
    return {k: a.get(k, 0) + b[k] for k in b}


@pytest.mark.parametrize("name", GOLDEN)
def test_frame_variant_on_golden_streams(name):
    frame_pipeline(open(os.path.join(HERE, "golden", name + ".es"), "rb").read(), name)


def test_frame_variant_on_synth_cases_covers_absent_macroblocks():
    import synth_es
    total = {}
    for name in list(synth_es.CASES) + list(synth_es.B_CASES):
        total = _sum(total, frame_pipeline(synth_es.make_case(name), name))
    assert total["b"] > 0 and total["absent"] > 0, total


def test_frame_variant_with_vectors_that_leave_the_plane():
    import synth_es
    total = {}
    for name in ("rows_ip", "b_rows"):
        total = _sum(total, frame_pipeline(synth_es.make_case(name), name, push_out=True))
    assert total["outside"] > 0, total


def test_frame_variant_on_encoder_clips_clean_and_damaged():
    pytest.importorskip("cv2")
    es = b"".join(p for _, p in helpers.clip_packets(320, 240, 8))
    frame_pipeline(es, "ffmpeg 320x240")
    rng = np.random.default_rng(7)
    for trial in range(4):
        bad = bytearray(es)
        for pos in rng.integers(200, len(es), size=4):
            bad[pos] ^= 1 << int(rng.integers(0, 8))
        frame_pipeline(bytes(bad), f"ffmpeg 320x240 damaged {trial}")


def test_frame_variant_on_mini_enc_streams():
    pytest.importorskip("cv2")
    import mini_enc
    es, types, _, _ = mini_enc.make_b_clip(frames=10)
    seen = frame_pipeline(es, "mini_enc 176x144 I/P/B")
    assert seen["pictures"] == len(types) and seen["b"] > 0
