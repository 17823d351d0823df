"""Stage 2's OUT_RESIDUALS variant (reconstruct_block<..., RES = true>, jsmpeg_b200/csrc/recon.cuh, DESIGN 3.15) WITHOUT
a GPU.  tests/emu/recon_residual_check.cpp builds the device code for the host (the emulation of test_compact_records)
and runs walk -> expand -> reconstruct for I, P and B pictures, once through the plain kernel's code and once through
the RES variant, on every kind of stream the suite has, clean and bit-flipped:
  * the RES variant's planes are the plain ones, with and without a residual destination;
  * its residual is macroblock_model.residuals of the oracle's records and coefficients on clean streams, and on every
    stream the numpy transform of the emulated expand's own coefficient blocks, every in-picture sample written;
  * the corpus has pictures with absent macroblocks, and P pictures whose vectors are pushed out of the plane take the
    per-tap path.
"""
import os
import subprocess

import numpy as np
import pytest

import helpers
import macroblock_model
from test_compact_records import GOLDEN, RECORD, stream_geometry

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_SRC = os.path.join(HERE, "emu", "recon_residual_check.cpp")
CSRC = os.path.join(HERE, "..", "jsmpeg_b200", "csrc")
SENTINEL = 0x5A5A  # what the residual holds before the RES variant writes it


def residual_lib():
    import ctypes
    out = os.path.join(HERE, "emu", "librecon_residual_check.so")
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
    lib.emu_expand_picture.argtypes = [vp, u32, i, i, vp, vp, vp, vp]
    lib.emu_expand_picture_compact.argtypes = [vp, u32, i, i, vp, vp, vp, vp, vp]
    lib.emu_reconstruct_picture_compact.argtypes = [vp, vp, vp, vp, vp, vp, i, i]
    lib.emu_reconstruct_picture_res.argtypes = [vp, vp, vp, vp, vp, vp, i, i, vp]
    return lib


def outside_blocks(hdr, mbw, mbh):
    """Luma blocks of present predicted macroblocks whose forward prediction leaves the plane (stage 2's flat-index
    rule, PREDICTION_INSIDE in common.cuh)"""
    h = hdr.reshape(-1, 4)
    mh = (h[:, 0] & 0xFFFF).astype(np.uint16).view(np.int16).astype(np.int64)
    mv = (h[:, 0] >> 16).astype(np.uint16).view(np.int16).astype(np.int64)
    flags = h[:, 1] & 0xFF
    pred = ((flags & macroblock_model.MBF_PRESENT) != 0) & ((flags & macroblock_model.MBF_INTRA) == 0)
    stride, ysize = mbw * 16, mbw * mbh * 256
    row, col = np.divmod(np.arange(mbw * mbh), mbw)
    n = 0
    for b in range(4):
        origin = (row * 16 + (b >> 1) * 8) * stride + col * 16 + (b & 1) * 8
        src = origin + (mv >> 1) * stride + (mh >> 1)
        inside = (src >= 0) & (src + 7 * stride + 7 + (mv & 1) * stride + (mh & 1) < ysize)
        n += int((pred & ~inside).sum())
    return n


def residual_pipeline(es, name, damaged=False, push_out=False):
    """The emulated pipeline with the product's plane bookkeeping (test_compact_records.compact_pipeline), every
    decoded picture reconstructed by the plain code and by the RES variant.  push_out: the present predicted
    macroblocks of every other macroblock row of a P picture get the vector (-64, -64) (luma half-samples) before stage
    2, so that the blocks of the first row read outside the plane.  Returns per-kind counts."""
    import ctypes
    from jsmpeg_b200 import decoder
    olib = helpers.oracle_lib()
    olib.oracle_set_decode_b(1)
    lib = residual_lib()
    seen = {"pictures": 0, "b": 0, "absent": 0, "outside": 0, "oracle_checked": 0}
    try:
        d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=olib)
        d.write(0, [es])
        seq = olib.oracle_seq_params(d.decoder).contents
        mb = seq.mb_size
        lib.emu_set_quant(bytes(seq.intra_q), bytes(seq.non_intra_q))
        mbw, mbh = stream_geometry(es)
        buf = np.frombuffer(es + b"\0" * 16, dtype=np.uint8).copy()
        ysize = mb * 256
        size = ysize * 3 // 2 + mbw * 16 + 64
        planes = [np.zeros(size, dtype=np.uint8) for _ in range(2)]  # the plain path's sets
        planes_b = np.zeros(size, dtype=np.uint8)
        cur = 0
        clean = True
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
            dense = np.zeros(mb * 6 * 64, dtype=np.int16)
            lib.emu_expand_picture(buf.ctypes.data, len(es), mbw, mbh, hdr.ctypes.data, park.ctypes.data, dense.ctypes.data,
                                   pinfo.ctypes.data)
            coef = np.zeros(mb * 6 * 64, dtype=np.int16)
            compact = np.zeros(mb * 6, dtype=RECORD)
            lib.emu_expand_picture_compact(buf.ctypes.data, len(es), mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                                           coef.ctypes.data, compact.ctypes.data, pinfo.ctypes.data)
            if push_out and info.picture_type == 2:
                rows = (np.arange(mb) // mbw) % 2 == 0
                h4 = hdr.reshape(mb, 4)
                h4[rows, 0] = np.uint32((0xFFC0 << 16) | 0xFFC0)  # (int16 -64, int16 -64)
            if is_b:
                out, fwd, bwd = planes_b, planes[cur], planes[cur ^ 1]
            else:
                out, fwd, bwd = planes[cur], planes[cur ^ 1], None
            before = out.copy()
            lib.emu_reconstruct_picture_compact(hdr.ctypes.data, coef.ctypes.data, compact.ctypes.data, out.ctypes.data,
                                                fwd.ctypes.data, None if bwd is None else bwd.ctypes.data, mbw, mbh)
            for with_res in (False, True):  # (the RES variant without and with a residual task: the same planes)
                out_r = before.copy()
                res = np.full(ysize * 3 // 2, SENTINEL, dtype=np.int16)
                lib.emu_reconstruct_picture_res(hdr.ctypes.data, coef.ctypes.data, compact.ctypes.data, out_r.ctypes.data,
                                                fwd.ctypes.data, None if bwd is None else bwd.ctypes.data, mbw, mbh,
                                                res.ctypes.data if with_res else None)
                assert np.array_equal(out_r, out), f"{name}: picture {seen['pictures']}: planes (residual {with_res})"
                assert with_res or (res == SENTINEL).all(), f"{name}: a task without a residual stored one"
            if not is_b:
                cur ^= 1
            # every sample written, and the transform of the expand's own blocks (the walk's cbp bits decide)
            hb = hdr.view(np.uint8).reshape(mb, 16).copy()
            want = macroblock_model.residuals(hb, dense, mbw, mbh)
            assert np.array_equal(res, want), f"{name}: picture {seen['pictures']} (type {info.picture_type}): residual"
            if damaged and info.error:
                clean = False
            if clean and not push_out:  # the oracle's own records and coefficients of the picture (= its fresh decoder's on a clean stream)
                orec = np.ctypeslib.as_array(ctypes.cast(olib.oracle_last_mb_records(d.decoder), ctypes.POINTER(ctypes.c_uint8)),
                                             shape=(mb * 16,)).reshape(mb, 16).copy()
                ocoef = np.ctypeslib.as_array(ctypes.cast(olib.oracle_last_coefficients(d.decoder), ctypes.POINTER(ctypes.c_int16)),
                                              shape=(mb * 6 * 64,)).copy()
                assert np.array_equal(res, macroblock_model.residuals(orec, ocoef, mbw, mbh)), \
                    f"{name}: picture {seen['pictures']} (type {info.picture_type}): residual against the oracle"
                seen["oracle_checked"] += 1
            flags = hb[:, 4]
            seen["absent"] += int(((flags & macroblock_model.MBF_PRESENT) == 0).sum())
            if info.picture_type == 2:
                seen["outside"] += outside_blocks(hdr, mbw, mbh)
            seen["b"] += int(is_b)
            seen["pictures"] += 1
        d.destroy()
    finally:
        olib.oracle_set_decode_b(0)
    assert seen["pictures"] > 0 and (seen["oracle_checked"] > 0 or push_out or damaged), name
    return seen


def _sum(a, b):
    return {k: a.get(k, 0) + b[k] for k in b}


@pytest.mark.parametrize("name", GOLDEN)
def test_residual_variant_on_golden_streams(name):
    residual_pipeline(open(os.path.join(HERE, "golden", name + ".es"), "rb").read(), name)


def test_residual_variant_on_synth_cases_covers_absent_macroblocks():
    import synth_es
    total = {}
    for name in list(synth_es.CASES) + list(synth_es.B_CASES):
        total = _sum(total, residual_pipeline(synth_es.make_case(name), name))
    assert total["b"] > 0 and total["absent"] > 0, total


def test_residual_variant_with_vectors_that_leave_the_plane():
    """The per-tap path of stage 2 (a prediction outside the plane) in the RES variant: the vectors of a P picture's
    records pushed out of the plane (the records' coefficients, so the residual, unchanged)"""
    import synth_es
    total = {}
    for name in ("rows_ip", "b_rows"):
        total = _sum(total, residual_pipeline(synth_es.make_case(name), name, push_out=True))
    assert total["outside"] > 0, total


def test_residual_variant_on_encoder_clips_clean_and_damaged():
    pytest.importorskip("cv2")
    es = b"".join(p for _, p in helpers.clip_packets(320, 240, 8))
    residual_pipeline(es, "ffmpeg 320x240")
    rng = np.random.default_rng(7)
    for trial in range(4):
        bad = bytearray(es)
        for pos in rng.integers(200, len(es), size=4):
            bad[pos] ^= 1 << int(rng.integers(0, 8))
        residual_pipeline(bytes(bad), f"ffmpeg 320x240 damaged {trial}", damaged=True)


def test_residual_variant_on_mini_enc_streams():
    pytest.importorskip("cv2")
    import mini_enc
    es, types, _, _ = mini_enc.make_b_clip(frames=10)
    seen = residual_pipeline(es, "mini_enc 176x144 I/P/B")
    assert seen["pictures"] == len(types) and seen["b"] > 0
    es, types, _, _ = mini_enc.make_b_clip(frames=7, qscale=(1, 1, 1))  # mostly dense records
    assert residual_pipeline(es, "mini_enc qscale 1")["pictures"] == len(types)
