"""The compact coefficient records (jsmpeg_b200/csrc/coef_records.h) WITHOUT a GPU.

Stage 1b hands stage 2 a 32-byte record per coded block -- a 64-bit mask of the zig-zag positions its codes wrote
and up to 12 values in zig-zag order -- and a dense 128-byte record only for blocks with more positions.
tests/emu/compact_emu.cpp compiles the header and the device code (walk, expand, reconstruct) for the host:
  * the format, as g++ builds it, against a numpy model, on random blocks of 0 to 64 positions;
  * the emulated pipeline walk -> expand (compact) -> reconstruct against the oracle's planes, and every compact
    record unpacked against the dense expand's block, on every kind of stream the suite has, clean and damaged,
    I, P and B pictures, and a stream coded at quantiser scale 1, where most blocks take the dense form;
  * the same under AddressSanitizer with compact planes of exact size.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers  # noqa: F401  (adds tools/ to sys.path)

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_SRC = os.path.join(HERE, "emu", "compact_emu.cpp")
CSRC = os.path.join(HERE, "..", "jsmpeg_b200", "csrc")
DENSE = 0xFFFFFFFFFFFFFFFF
LEVELS = 12
# ISO 11172-2 2.4.4.1: raster index of zig-zag position k
ZIG_ZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                    7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                    39, 46, 53, 60, 61, 54, 47, 55, 62, 63])
RECORD = np.dtype([("mask", "<u8"), ("level", "<i2", (LEVELS,))])
assert RECORD.itemsize == 32


def build_compact_lib(asan=False):
    out = os.path.join(HERE, "emu", "libcompact_emu_asan.so" if asan else "libcompact_emu.so")
    deps = [EMU_SRC, os.path.join(HERE, "emu", "walk_emu.cpp")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        tmp = out + ".%d.tmp" % os.getpid()
        flags = ["-O1", "-g", "-fsanitize=address", "-fno-omit-frame-pointer"] if asan else ["-O2"]
        subprocess.check_call(["g++", *flags, "-std=c++17", "-shared", "-fPIC", "-Wno-attributes", "-Wno-unknown-pragmas",
                               "-I/usr/local/cuda/include", "-o", tmp, EMU_SRC])
        os.replace(tmp, out)
    return out


def compact_lib(asan=False):
    """The emulation library (asan: the AddressSanitizer build, loadable only where libasan was preloaded)"""
    lib = ctypes.CDLL(build_compact_lib(asan))
    vp, i, u32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32
    lib.emu_walk_picture.argtypes = [vp, u32, u32, i, i, vp, vp, vp, i]
    lib.emu_walk_picture_b.argtypes = [vp, u32, u32, i, i, vp, vp, vp]
    lib.emu_expand_picture.argtypes = [vp, u32, i, i, vp, vp, vp, vp]
    lib.emu_expand_picture_compact.argtypes = [vp, u32, i, i, vp, vp, vp, vp, vp]
    lib.emu_reconstruct_picture_compact.argtypes = [vp, vp, vp, vp, vp, vp, i, i]
    lib.emu_coef_pack.argtypes = [ctypes.c_uint64, vp, vp]
    lib.emu_coef_unpack.argtypes = [vp, vp]
    lib.emu_coef_nonzero_positions.argtypes = [vp]
    lib.emu_coef_nonzero_positions.restype = ctypes.c_uint64
    return lib


# ---- the format ---------------------------------------------------------------------------------------------------

def model_pack(positions, raster):
    """numpy model of coef_record_pack: positions = sorted zig-zag positions"""
    rec = np.zeros(1, dtype=RECORD)
    rec["mask"] = sum(1 << int(p) for p in positions)
    rec["level"][0, :len(positions)] = raster[ZIG_ZAG[np.asarray(positions, dtype=int)]]
    return rec


def random_blocks(rng):
    """(positions, raster block) pairs: 0 to 64 positions, the level extremes, a written zero (intra DC 0), exactly
    12 and 13 positions, position 63"""
    out = []
    for n in list(range(65)) + [12, 13, 12, 13, 1, 1]:
        pos = np.sort(rng.choice(64, size=n, replace=False))
        raster = np.zeros(64, dtype=np.int16)
        vals = rng.integers(-2048, 2048, size=n).astype(np.int16)
        vals[vals == 0] = 1
        raster[ZIG_ZAG[pos]] = vals
        out.append((pos, raster))
    pos = np.array([0, 5, 63])
    raster = np.zeros(64, dtype=np.int16)
    raster[ZIG_ZAG[pos]] = [0, -2048, 2047]  # intra DC 0: written, but zero
    out.append((pos, raster))
    pos = np.arange(52, 64)  # twelve positions ending at 63
    raster = np.zeros(64, dtype=np.int16)
    raster[ZIG_ZAG[pos]] = np.arange(1, 13)
    out.append((pos, raster))
    return out


def test_zigzag_map_is_the_standards():
    lib = compact_lib()
    assert [lib.emu_coef_zigzag_raster(k) for k in range(64)] == ZIG_ZAG.tolist()


def test_format_round_trip_against_the_numpy_model():
    lib = compact_lib()
    rng = np.random.default_rng(11)
    fits = too_big = 0
    for pos, raster in random_blocks(rng):
        mask = sum(1 << int(p) for p in pos)
        rec = np.zeros(1, dtype=RECORD)
        ok = lib.emu_coef_pack(mask, raster.ctypes.data, rec.ctypes.data)
        assert ok == (len(pos) <= LEVELS), len(pos)
        if not ok:
            too_big += 1
            continue
        fits += 1
        assert rec.tobytes() == model_pack(pos, raster).tobytes(), pos
        back = np.full(64, 7, dtype=np.int16)
        lib.emu_coef_unpack(rec.ctypes.data, back.ctypes.data)
        assert np.array_equal(back, raster), pos
        # the debug hook's form: positions taken from the nonzero values reproduce the block as well
        nz = lib.emu_coef_nonzero_positions(raster.ctypes.data)
        assert nz == sum(1 << int(p) for p in pos if raster[ZIG_ZAG[p]] != 0)
        rec2 = np.zeros(1, dtype=RECORD)
        assert lib.emu_coef_pack(nz, raster.ctypes.data, rec2.ctypes.data)
        lib.emu_coef_unpack(rec2.ctypes.data, back.ctypes.data)
        assert np.array_equal(back, raster)
    assert fits >= 15 and too_big >= 50


# ---- the emulated pipeline ----------------------------------------------------------------------------------------

def stream_geometry(es):
    i = es.find(b"\x00\x00\x01\xb3")
    w = (es[i + 4] << 4) | (es[i + 5] >> 4)
    h = ((es[i + 5] & 15) << 8) | es[i + 6]
    return (w + 15) >> 4, (h + 15) >> 4


def compact_pipeline(es, name, lib=None, damaged=False):
    """walk (I/P: lane-parallel, B: walk_b) -> expand, dense and compact -> reconstruct from the compact records, with
    the product's plane bookkeeping, against the oracle's planes (B pictures decoded).  damaged: planes are compared up
    to the first picture whose walk reports an error (outside the parity domain, DESIGN.md section 6); the records
    are compared throughout.  Returns (pictures decoded, coded blocks, blocks in dense form)."""
    from jsmpeg_b200 import decoder
    olib = helpers.oracle_lib()
    olib.oracle_set_decode_b(1)
    try:
        d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=olib)
        d.write(0, [es])
        seq = olib.oracle_seq_params(d.decoder).contents
        mb = seq.mb_size
        lib = lib or compact_lib()
        lib.emu_set_quant(bytes(seq.intra_q), bytes(seq.non_intra_q))
        mbw, mbh = stream_geometry(es)
        buf = np.frombuffer(es + b"\0" * 16, dtype=np.uint8).copy()
        ysize = mb * 256
        size = ysize * 3 // 2 + mbw * 16 + 64
        planes = [np.zeros(size, dtype=np.uint8) for _ in range(2)]
        planes_b = np.zeros(size, dtype=np.uint8)
        cur = 0
        decoded = coded_blocks = dense_blocks = 0
        compare = True
        while d.decode():
            info = olib.oracle_last_picture_info(d.decoder).contents
            hdr = np.zeros(mb * 4, dtype=np.uint32)
            park = np.zeros(mb * 6 * 2, dtype=np.uint32)
            pinfo = np.zeros(12, dtype=np.int32)
            is_b = ((es[info.start_byte + 1] >> 3) & 7) == 3
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
            compact = np.zeros(mb * 6, dtype=RECORD)  # exact size: the product's plane holds mb_size * 6 records
            lib.emu_expand_picture_compact(buf.ctypes.data, len(es), mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                                           coef.ctypes.data, compact.ctypes.data, pinfo.ctypes.data)
            hb = hdr.view(np.uint8).reshape(mb, 16)
            coded = np.zeros(mb * 6, dtype=bool)
            for blk in range(6):
                coded[blk::6] = ((hb[:, 4] & 1) != 0) & ((hb[:, 5] & (0x20 >> blk)) != 0)
            dense = dense.reshape(-1, 64)
            coef = coef.reshape(-1, 64)
            for slot in np.nonzero(coded)[0]:
                if int(compact["mask"][slot]) == DENSE:
                    dense_blocks += 1
                    assert np.array_equal(coef[slot], dense[slot]), f"{name}: picture {decoded} slot {slot}: dense record"
                else:
                    back = np.zeros(64, dtype=np.int16)
                    lib.emu_coef_unpack(compact[slot:slot + 1].ctypes.data, back.ctypes.data)
                    assert bin(int(compact["mask"][slot])).count("1") <= LEVELS
                    assert np.array_equal(back, dense[slot]), f"{name}: picture {decoded} slot {slot}: compact record"
            coded_blocks += int(coded.sum())
            if is_b:
                out = planes_b
                lib.emu_reconstruct_picture_compact(hdr.ctypes.data, coef.ctypes.data, compact.ctypes.data, out.ctypes.data,
                                                    planes[cur].ctypes.data, planes[cur ^ 1].ctypes.data, mbw, mbh)
            else:
                out = planes[cur]
                lib.emu_reconstruct_picture_compact(hdr.ctypes.data, coef.ctypes.data, compact.ctypes.data, out.ctypes.data,
                                                    planes[cur ^ 1].ctypes.data, None, mbw, mbh)
                cur ^= 1
            if damaged and info.error:
                compare = False
            if compare:
                y, cr, cb = d.planes()
                got = np.concatenate([out[:ysize], out[ysize:ysize + ysize // 4], out[ysize + ysize // 4:ysize * 3 // 2]])
                assert np.array_equal(got, np.concatenate([y, cr, cb])), f"{name}: picture {decoded} (type {info.picture_type})"
            decoded += 1
        d.destroy()
    finally:
        olib.oracle_set_decode_b(0)
    assert decoded > 0
    return decoded, coded_blocks, dense_blocks


GOLDEN = sorted(f[:-3] for f in os.listdir(os.path.join(HERE, "golden")) if f.endswith(".es"))


@pytest.mark.parametrize("name", GOLDEN)
def test_compact_pipeline_on_golden_streams(name):
    compact_pipeline(open(os.path.join(HERE, "golden", name + ".es"), "rb").read(), name)


def test_compact_pipeline_on_synth_cases():
    import synth_es
    for name in list(synth_es.CASES) + list(synth_es.B_CASES):
        compact_pipeline(synth_es.make_case(name), name)


def test_compact_pipeline_on_b_fixture():
    es = open(os.path.join(HERE, "fixtures", "b_clip_1280x720.m1v"), "rb").read()
    compact_pipeline(es, "720p I/P/B fixture")


def test_compact_pipeline_on_encoder_clips_clean_and_damaged():
    pytest.importorskip("cv2")
    es = b"".join(p for _, p in helpers.clip_packets(320, 240, 8))
    compact_pipeline(es, "ffmpeg 320x240")
    rng = np.random.default_rng(7)
    for trial in range(4):
        bad = bytearray(es)
        for pos in rng.integers(200, len(es), size=4):
            bad[pos] ^= 1 << int(rng.integers(0, 8))
        compact_pipeline(bytes(bad), f"ffmpeg 320x240 damaged {trial}", damaged=True)


def test_compact_pipeline_on_mini_enc_streams():
    pytest.importorskip("cv2")
    import mini_enc
    es, types, _, _ = mini_enc.make_b_clip(frames=10)
    decoded, _, _ = compact_pipeline(es, "mini_enc 176x144 I/P/B")
    assert decoded == len(types)


def test_quantiser_scale_1_takes_the_dense_form():
    """At quantiser scale 1 most coded blocks carry more than 12 values: the dense records carry the picture."""
    pytest.importorskip("cv2")
    import mini_enc
    es, types, _, _ = mini_enc.make_b_clip(frames=7, qscale=(1, 1, 1))
    decoded, coded, dense = compact_pipeline(es, "mini_enc qscale 1")
    assert decoded == len(types) and dense * 2 > coded, (dense, coded)


def _asan_run():
    lib = compact_lib(asan=True)
    import synth_es
    for name in GOLDEN:
        compact_pipeline(open(os.path.join(HERE, "golden", name + ".es"), "rb").read(), name, lib=lib)
    for name in list(synth_es.B_CASES)[:2]:
        compact_pipeline(synth_es.make_case(name), name, lib=lib)
    print("asan clean")


def test_compact_path_is_memory_safe_under_address_sanitizer():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not asan or not os.path.exists(asan):
        pytest.skip("libasan not available")
    build_compact_lib(asan=True)  # built here, loaded only in the sanitizer's process
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0")
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, capture_output=True, text=True, timeout=1200, cwd=HERE)
    assert r.returncode == 0 and "asan clean" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    _asan_run()
