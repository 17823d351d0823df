"""Stage 1b builds a block's compact record in code order and its warp stores the records (jsmpeg_b200/csrc/walk.cuh:
expand_warp_run, tests/emu/expand_warp_emu.cpp: a warp as 32 coroutines).

Without a GPU: a stream written block by block, with the shapes the random streams do not pin -- exactly 12, exactly 13
and 64 values, an intra block that is its DC alone, a non-intra block that starts with the peeled dct_coeff_first and
one that does not, a run that passes position 63, and a picture in which every second block slot is uncoded -- through
the emulated walk and the warp's expand: the compact and the dense plane against the oracle's blocks, every byte
outside the coded blocks' records untouched, and the dense-only mode.
On the GPU: decode_coefficients of pictures of 1080p bench clips, the crafted stream and small streams in one batch
against the oracle's blocks.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers  # noqa: F401  (adds tools/ to sys.path)
import synth_es
from synth_es import CBP_CODE, DC_LUMA_CODE, DC_CHROMA_CODE, MBA_CODE, TYPE_I_CODE, TYPE_P_CODE, V
from test_coefficient_export import oracle_coefficients
from test_compact_records import DENSE, LEVELS, RECORD, ZIG_ZAG, stream_geometry

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_SRC = os.path.join(HERE, "emu", "expand_warp_emu.cpp")
CSRC = os.path.join(HERE, "..", "jsmpeg_b200", "csrc")
FILL = 0x5A  # what the planes hold before stage 1b: a slot it must not write keeps it


def warp_lib():
    out = os.path.join(HERE, "emu", "libexpand_warp_emu.so")
    deps = [os.path.join(HERE, "emu", f) for f in ("expand_warp_emu.cpp", "compact_emu.cpp", "walk_emu.cpp")]
    deps += [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        tmp = out + ".%d.tmp" % os.getpid()
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wno-attributes", "-Wno-unknown-pragmas",
                               "-I/usr/local/cuda/include", "-o", tmp, EMU_SRC])
        os.replace(tmp, out)
    lib = ctypes.CDLL(out)
    vp, i, u32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32
    lib.emu_walk_picture.argtypes = [vp, u32, u32, i, i, vp, vp, vp, i]
    lib.emu_expand_picture_warps.argtypes = [vp, u32, i, i, vp, vp, vp, vp, vp]
    return lib


# ---- a stream written block by block --------------------------------------------------------------------------------

def put_codes(w, codes, first):
    """(run, level) pairs as dct_coeff_first / dct_coeff_next codes, then end_of_block"""
    for run, level in codes:
        code = V.DCT_RUN_LEVEL_CODE.get((run, abs(level)))
        if code is None:  # escape, one-byte level
            w.code(V.DCT_ESCAPE_CODE)
            w.put(run, 6)
            w.put(level & 255, 8)
        else:
            w.code("1" if first and code == "1" else ("11" if code == "1" else code))
            w.put(1 if level < 0 else 0, 1)
        first = False
    w.code(V.DCT_EOB_CODE)


def ones(n, level=1):
    """n values at consecutive positions, signs alternating"""
    return [(0, level if k % 2 == 0 else -level) for k in range(n)]


# per picture: (picture type, [(intra, coded block pattern, [codes of each coded block])] per macroblock)
PAST_63 = [(5, 2), (60, 1), (0, 1), (3, -2)]          # 6, then 67: dropped, like everything behind it
INTRA_BLOCKS = [[], ones(11), ones(12), ones(63), [(0, 3), (1, -1)], [(62, 1)]]  # DC alone, 12, 13, 64 values, ..., position 63
INTER_BLOCKS = [ones(12), ones(13, 2), ones(64)]      # peeled first code; first code (0, 2): not peeled
INTER_MORE = [[(0, 1)], [(2, 3), (0, -1)], [(0, -1), (62, 2)]]


def crafted_pictures(mb_count):
    intra_mb = (True, 0x3F, INTRA_BLOCKS)
    pics = [(1, [intra_mb] * mb_count)]
    # every second slot uncoded: pattern 101010 in every macroblock, so the coded slots are the even ones
    pics.append((2, [(False, 0x2A, INTER_BLOCKS if m % 2 == 0 else INTER_MORE) for m in range(mb_count)]))
    # mixed: intra macroblocks between coded ones, all six blocks coded (a dense block beside compact ones in a warp)
    pics.append((2, [intra_mb if m % 3 == 0 else (False, 0x3F, INTER_BLOCKS + INTER_MORE) for m in range(mb_count)]))
    # a picture with runs that pass position 63 (the walk flags it; the stores past 63 are dropped)
    pics.append((2, [(False, 0x30, [PAST_63, [(0, 1)] + PAST_63]) for m in range(mb_count)]))
    return pics


def crafted_stream(width=96, height=64):
    s = synth_es.SynthStream(synth_es.Knobs(width=width, height=height), 1)
    s.sequence_header()
    for index, (ptype, mbs) in enumerate(crafted_pictures(s.mbw * s.mbh)):
        if ptype == 1:
            s.gop_header()
        s.picture_header(index, ptype, 0, 1)
        w = synth_es.BitWriter()
        w.start_code(1)
        w.put(3 + index, 5)  # quantiser scale
        w.put(0, 1)
        for intra, cbp, blocks in mbs:
            w.code(MBA_CODE[1])
            w.code(TYPE_I_CODE[0x01] if ptype == 1 else TYPE_P_CODE[0x01 if intra else 0x02])
            if not intra:
                w.code(CBP_CODE[cbp])
            coded = [b for b in range(6) if cbp & (0x20 >> b)]
            assert len(coded) == len(blocks)
            for b, codes in zip(coded, blocks):
                if intra:
                    w.code((DC_LUMA_CODE if b < 4 else DC_CHROMA_CODE)[0])  # dc differential 0
                put_codes(w, codes, first=not intra)
        w.align()
        body = w.tobytes()[4:]
        assert not any(body[i] == 0 and body[i + 1] == 0 and body[i + 2] <= 1 for i in range(len(body) - 2))
        s.out.align()
        s.out.bits.extend(synth_es.BitWriter_bits(w.tobytes()))
    s.out.start_code(0xB7)
    return s.out.tobytes()


# ---- the warp's expand against the oracle ---------------------------------------------------------------------------

def unpack(rec):
    out = np.zeros(64, np.int16)
    pos = [k for k in range(64) if (int(rec["mask"]) >> k) & 1]
    out[ZIG_ZAG[pos]] = rec["level"][:len(pos)]
    return out


def check_stream(es, name, with_compact=True):
    """Every decoded picture: emulated walk, then the warp's expand into planes pre-filled with FILL.  Returns
    (coded blocks, dense blocks, value counts seen)."""
    lib = warp_lib()
    olib = helpers.oracle_lib()
    mbw, mbh = stream_geometry(es)
    mb = mbw * mbh
    buf = np.frombuffer(es + b"\0" * 16, dtype=np.uint8).copy()
    want_all = oracle_coefficients(es)
    seq = None
    from jsmpeg_b200 import decoder
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=olib)
    d.write(0, [es])
    seq = olib.oracle_seq_params(d.decoder).contents
    lib.emu_set_quant(bytes(seq.intra_q), bytes(seq.non_intra_q))
    d.destroy()
    coded_blocks = dense_blocks = 0
    counts = set()
    assert want_all
    for pos, info, _, want in want_all:
        want = want.reshape(mb * 6, 64)
        hdr = np.zeros(mb * 4, dtype=np.uint32)
        park = np.zeros(mb * 6 * 2, dtype=np.uint32)
        pinfo = np.zeros(12, dtype=np.int32)
        lib.emu_walk_picture(buf.ctypes.data, len(es), info.start_byte, mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                             pinfo.ctypes.data, 1)
        assert pinfo[2] == 1, (name, pos)
        coef = np.full(mb * 6 * 128, FILL, dtype=np.uint8)
        compact = np.full(mb * 6 * 32, FILL, dtype=np.uint8)
        lib.emu_expand_picture_warps(buf.ctypes.data, len(es), mbw, mbh, hdr.ctypes.data, park.ctypes.data, coef.ctypes.data,
                                     compact.ctypes.data if with_compact else None, pinfo.ctypes.data)
        hb = hdr.view(np.uint8).reshape(mb, 16)
        coded = np.zeros(mb * 6, dtype=bool)
        for blk in range(6):
            coded[blk::6] = ((hb[:, 4] & 1) != 0) & ((hb[:, 5] & (0x20 >> blk)) != 0)
        records = compact.view(RECORD)
        dense_rows = coef.view(np.int16).reshape(mb * 6, 64)
        for slot in range(mb * 6):
            is_dense = coded[slot] and (not with_compact or int(records["mask"][slot]) == DENSE)
            if coded[slot] and not is_dense:
                n = bin(int(records["mask"][slot])).count("1")
                assert n <= LEVELS
                assert not records["level"][slot][n:].any(), f"{name} @{pos} slot {slot}: unused levels are zero"
                assert np.array_equal(unpack(records[slot]), want[slot]), f"{name} @{pos} slot {slot}: compact record"
                counts.add(n)
            elif with_compact and not coded[slot]:
                assert (compact[slot * 32:slot * 32 + 32] == FILL).all(), f"{name} @{pos} slot {slot}: uncoded, yet written"
            if is_dense:
                assert np.array_equal(dense_rows[slot], want[slot]), f"{name} @{pos} slot {slot}: dense record"
                if with_compact:
                    assert (compact[slot * 32 + 8:slot * 32 + 32] == FILL).all(), f"{name} @{pos} slot {slot}: dense, levels written"
                counts.add(int(np.count_nonzero(want[slot])))
                dense_blocks += 1
            else:
                assert (coef[slot * 128:slot * 128 + 128] == FILL).all(), f"{name} @{pos} slot {slot}: dense plane written"
        coded_blocks += int(coded.sum())
    return coded_blocks, dense_blocks, counts


def test_crafted_blocks_through_the_warp_expand_equal_the_oracle():
    es = crafted_stream()
    coded, dense, counts = check_stream(es, "crafted")
    assert {1, 2, 12, 13, 64} <= counts and dense > 0 and coded > dense
    # every second slot of the second picture is uncoded (and so every second lane of its warps)
    _, _, rec, _ = oracle_coefficients(es)[1]
    assert (rec[:, 4] & 1).all() and (rec[:, 5] == 0x2A).all()


def test_a_task_without_a_compact_plane_gets_dense_records():
    coded, dense, _ = check_stream(crafted_stream(), "crafted, dense only", with_compact=False)
    assert coded == dense > 0


def test_an_odd_sized_picture_whose_last_warp_is_partial():
    """176 x 144: 594 block slots, the last warp holds 18"""
    coded, dense, _ = check_stream(crafted_stream(176, 144), "crafted 176x144")
    assert dense > 0 and coded > dense


@pytest.mark.parametrize("name", ["escapes_matrices", "odd_size", "skips_stuffing_escape_mba"])
def test_synthetic_streams_through_the_warp_expand(name):
    es = synth_es.make_case(name)
    # (these cases hold I and P pictures the reference decodes; ignored pictures are not in the oracle's list)
    coded, _, _ = check_stream(es, name)
    assert coded > 0


# ---- on the GPU -----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_mixed_sizes_in_one_batch_equal_the_oracle_on_the_gpu():
    """Pictures of four 1080p bench clips, the crafted stream at two sizes and a synthetic stream in one
    decode_coefficients call: every block equals the oracle's (fresh decode of each picture)."""
    import random

    import macroblock_model
    from jsmpeg_b200.batch import BatchDecoder
    from test_coefficient_export import oracle_fresh_coefficients
    sys.path.insert(0, helpers.ROOT)
    import bench
    clips = list(bench.load_streams(bench.rank_seeds(0)[:4]))
    clips += [crafted_stream(), crafted_stream(176, 144), synth_es.make_case("escapes_matrices")]
    bd = BatchDecoder(len(clips))
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    rng = random.Random(5)
    reqs = []
    for s in range(len(clips)):
        listed = [e["picture"] for e in bd.macroblock_index(s)]
        reqs += [(s, k) for k in sorted(rng.sample(listed, min(6, len(listed))))]
    rng.shuffle(reqs)
    got = bd.decode_coefficients(reqs)
    assert bd.last_error() is None
    sizes = set()
    for (s, k), t in zip(reqs, got):
        entry = next(e for e in macroblock_model.macroblock_index(clips[s]) if e["picture"] == k)
        want = oracle_fresh_coefficients(clips[s], entry)[2]
        have = t.cpu().numpy().reshape(-1, 6, 64)
        assert np.array_equal(have, want), (s, k)
        sizes.add(have.shape[0])
    assert len(sizes) >= 3
    bd.close()
