"""Lane-parallel walk == serial walk, record for record, WITHOUT a GPU.

tests/emu/walk_emu.cpp compiles the device code of jsmpeg_b200/csrc/walk.cuh for the host and runs a
warp as 32 threads.  The serial walk is the one the GPU parity tests pin to the oracle; here every
picture of the golden streams, of the syntax-level generator's cases and of encoder-made clips is
walked both ways and the outputs must be identical: macroblock records, the {bit offset, dc} pair of
every coded block in the dense side array (the walk's hand-over to stage 1b), and the picture info
(end_bit, counts, error).
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers  # noqa: F401  (adds tools/ to sys.path)

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_SRC = os.path.join(HERE, "emu", "walk_emu.cpp")
EMU_LIB = os.path.join(HERE, "emu", "libwalk_emu.so")
CSRC = os.path.join(HERE, "..", "jsmpeg_b200", "csrc")


def emu_lib(define=None):
    """The emulation library; `define` builds a variant with -D<define>."""
    out = EMU_LIB if define is None else EMU_LIB.replace(".so", "_" + define.lower() + ".so")
    deps = [EMU_SRC] + [os.path.join(CSRC, f) for f in ("walk.cuh", "walk_b.cuh", "walk_slices.cuh", "recon.cuh", "common.cuh", "records.h", "vlc_tables.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        tmp = out + ".%d.tmp" % os.getpid()
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wno-attributes", "-Wno-unknown-pragmas",
                               "-I/usr/local/cuda/include"] + (["-D" + define] if define else []) + ["-o", tmp, EMU_SRC])
        os.replace(tmp, out)
    lib = ctypes.CDLL(out)
    lib.emu_walk_picture.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_int, ctypes.c_int,
                                     ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    return lib


def stream_geometry(es):
    i = es.find(b"\x00\x00\x01\xb3")
    assert i >= 0
    w = (es[i + 4] << 4) | (es[i + 5] >> 4)
    h = ((es[i + 5] & 15) << 8) | es[i + 6]
    return (w + 15) >> 4, (h + 15) >> 4


def picture_starts(es):
    out, i = [], 0
    while True:
        i = es.find(b"\x00\x00\x01\x00", i)
        if i < 0:
            return out
        out.append(i + 4)
        i += 4


def walk(lib, buf, n, start, mbw, mbh, lanes):
    mb = mbw * mbh
    hdr = np.zeros(mb * 4, dtype=np.uint32)
    park = np.full(mb * 6 * 2, 0xDEADBEEF, dtype=np.uint32)  # 8 bytes per coded block: {bit offset, intra dc}
    info = np.zeros(12, dtype=np.int32)
    lib.emu_walk_picture(buf.ctypes.data, n, start, mbw, mbh, hdr.ctypes.data, park.ctypes.data, info.ctypes.data, lanes)
    return hdr.reshape(mb, 4), park.reshape(mb * 6, 2), info


def check_stream(lib, es, what, expect_lanes=None, slice_walk_used=None):
    mbw, mbh = stream_geometry(es)
    buf = np.frombuffer(es + b"\0" * 16, dtype=np.uint8).copy()  # 4-byte aligned base, padded like the ES mirror
    used = 0
    starts = picture_starts(es)
    for k, s in enumerate(starts):
        h0, c0, i0 = walk(lib, buf, len(es), s, mbw, mbh, 0)
        # 1: staged relative records + fix-up (the product's path); 2: staging area too small, the lanes fall back to
        # the second, storing pass; 3: no staging area at all; 4: the slice walk (a lane per slice, walk_slices.cuh)
        for mode in (1, 2, 3, 4):
            h1, c1, i1 = walk(lib, buf, len(es), s, mbw, mbh, mode)
            if mode == 4 and slice_walk_used is not None and i1[2] == 1:
                slice_walk_used.append(int(i1[9]) == 2)
            if mode == 1:
                used += int(i1[9])
                # with the product's staging area every slice the lane walk takes is finished by the fix-up, not a second pass
                assert not i1[9] or i1[11] > 0, f"{what}: picture {k}: lane walk without fix-up"
            elif mode == 3:
                assert i1[11] == 0
            coded = np.zeros(len(c0), dtype=bool)  # the pairs of uncoded blocks are never read: only coded ones are compared
            hb = h0.view(np.uint8).reshape(-1, 16)
            for blk in range(6):
                coded[blk::6] = ((hb[:, 4] & 1) != 0) & ((hb[:, 5] & (0x20 >> blk)) != 0)
            assert np.array_equal(i0[:9], i1[:9]), f"{what}: picture {k} mode {mode}: info {i0[:9]} vs {i1[:9]}"
            assert np.array_equal(h0, h1), f"{what}: picture {k} mode {mode}: records differ at mb {np.nonzero((h0 != h1).any(axis=1))[0][:8]}"
            assert np.array_equal(c0[coded], c1[coded]), \
                f"{what}: picture {k} mode {mode}: parked block data differ at slot {np.nonzero(coded & (c0 != c1).any(axis=1))[0][:8]}"
    if expect_lanes is not None:
        assert used >= expect_lanes, f"{what}: lane-parallel walk used for {used} of {len(starts)} pictures"
    return used, len(starts)


GOLDEN = sorted(f[:-3] for f in os.listdir(os.path.join(HERE, "golden")) if f.endswith(".es"))


@pytest.mark.parametrize("name", GOLDEN)
def test_golden_streams(name):
    es = open(os.path.join(HERE, "golden", name + ".es"), "rb").read()
    check_stream(emu_lib(), es, name)


def test_synth_cases():
    import synth_es
    lib = emu_lib()
    for name in synth_es.CASES:
        check_stream(lib, synth_es.make_case(name), name)


@pytest.mark.parametrize("size,frames", [((320, 240), 14), ((1280, 720), 4), ((1920, 1080), 3)])
def test_encoder_clips_use_the_lane_walk(size, frames):
    pytest.importorskip("cv2")
    es = b"".join(p for _, p in helpers.clip_packets(size[0], size[1], frames))
    used, n = check_stream(emu_lib(), es, f"clip {size}")
    assert used == n, f"lane-parallel walk fell back on {n - used} of {n} clean pictures"


def test_slice_walk_takes_clean_multi_slice_pictures():
    """walk_slices.cuh (a lane per slice): on clean streams it finishes every decoded picture itself (info.reserved[0]
    == 2) -- a slice per macroblock row, slices starting mid-row, gaps between slices, one slice per picture, 45 slices
    of a natural 720p clip -- and its records equal the serial walk's (check_stream compares them)."""
    import synth_es
    lib = emu_lib()
    for name in ("rows_ip", "fcodes_fullpel", "random_slices_gaps", "odd_size", "i_only_320x240", "escapes_matrices"):
        took = []
        check_stream(lib, synth_es.make_case(name), name, slice_walk_used=took)
        assert took and all(took), f"{name}: slice walk fell back on {took.count(False)} of {len(took)} clean pictures"
    es = open(os.path.join(HERE, "fixtures", "b_clip_1280x720.m1v"), "rb").read()  # 45 slices per picture; B pictures are ignored here
    took = []
    check_stream(lib, es, "720p fixture", slice_walk_used=took)
    assert len(took) == 5 and all(took)


def test_slice_walk_falls_back_on_overlapping_slices():
    """Two slices claiming the same macroblock row: the reference decodes them one after the other and the second one
    wins; the slice walk must notice (address ranges not strictly increasing) and leave the picture to the serial walk."""
    import synth_es
    es = bytearray(synth_es.make_case("rows_ip"))
    starts = picture_starts(bytes(es))
    # the slices of the first picture: make the third one carry the second one's row number
    p = starts[0]
    codes = []
    i = p
    while len(codes) < 3:
        i = bytes(es).find(b"\x00\x00\x01", i)
        if 1 <= es[i + 3] <= 0xAF:
            codes.append(i)
        i += 3
    es[codes[2] + 3] = es[codes[1] + 3]
    took = []
    check_stream(emu_lib(), bytes(es), "overlapping slices", slice_walk_used=took)
    assert took[0] is False and all(took[1:4])


def test_truncated_and_corrupt_streams_fall_back_identically():
    pytest.importorskip("cv2")
    es = b"".join(p for _, p in helpers.clip_packets(320, 240, 6))
    lib = emu_lib()
    check_stream(lib, es[: len(es) * 2 // 3], "truncated")
    rng = np.random.default_rng(5)
    for trial in range(6):
        bad = bytearray(es)
        for pos in rng.integers(200, len(es), size=4):
            bad[pos] ^= 1 << int(rng.integers(0, 8))
        check_stream(lib, bytes(bad), f"corrupt {trial}")


def test_walks_are_memory_safe_under_address_sanitizer():
    """Both walks -- and the B-picture extension's walk, stage 1b and two-reference stage 2 -- on exact-size heap
    buffers (clean, bit-flipped and truncated streams) with the emulation library built with -fsanitize=address: no read or write outside the ES, the record
    arrays or the picture info.  (compute-sanitizer covers the same on the GPU when there is budget.)"""
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not asan or not os.path.exists(asan):
        pytest.skip("libasan not available")
    lib = os.path.join(HERE, "emu", "libwalk_emu_asan.so")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-shared", "-fPIC", "-fsanitize=address", "-fno-omit-frame-pointer",
                           "-Wno-attributes", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-o", lib, EMU_SRC])
    # three pictures of every stream here; ASAN_CHECK_PICTURES=0 python tests/emu/asan_check.py <lib> runs all (minutes)
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0",
               ASAN_CHECK_PICTURES=os.environ.get("ASAN_CHECK_PICTURES", "60"))
    r = subprocess.run([sys.executable, os.path.join(HERE, "emu", "asan_check.py"), lib], env=env, capture_output=True, text=True,
                       timeout=1200)
    assert r.returncode == 0 and "asan clean over" in r.stdout and " B pictures" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


@pytest.mark.parametrize("name", GOLDEN)
def test_device_walk_code_matches_the_oracle_records(name):
    """The device code of both walks, emulated on the host, against the ORACLE (the CPU restatement
    pinned to the reference): macroblock records, end_bit and the picture counts of every picture the
    oracle decodes.  The same comparison runs on the GPU (tests/test_gpu_parity.py); this one needs none."""
    from jsmpeg_b200 import decoder
    es = open(os.path.join(HERE, "golden", name + ".es"), "rb").read()
    olib = helpers.oracle_lib()
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=olib)
    d.write(0, [es])
    mb = olib.oracle_seq_params(d.decoder).contents.mb_size
    lib = emu_lib()
    mbw, mbh = stream_geometry(es)
    buf = np.frombuffer(es + b"\0" * 16, dtype=np.uint8).copy()
    checked = 0
    while d.decode():
        info = olib.oracle_last_picture_info(d.decoder).contents
        want = np.ctypeslib.as_array(ctypes.cast(olib.oracle_last_mb_records(d.decoder), ctypes.POINTER(ctypes.c_uint32)),
                                     shape=(mb, 4)).copy()
        for lanes in (1, 0):
            got, _, gi = walk(lib, buf, len(es), info.start_byte, mbw, mbh, lanes)
            assert np.array_equal(got, want), f"{name}: picture at byte {info.start_byte}, lanes={lanes}: records differ"
            assert (gi[1], gi[6], gi[7]) == (info.end_bit, info.n_present, info.n_coded_blocks), (name, info.start_byte, lanes)
        checked += 1
    assert checked > 0


@pytest.mark.parametrize("name", GOLDEN)
def test_stage1_device_code_matches_the_oracle_coefficients(name):
    """Stage 1 end to end on the CPU: the emulated walk (lane-parallel and serial) followed by stage
    1b's per-block device code (expand_block) against the ORACLE's dequantised coefficient blocks."""
    from jsmpeg_b200 import decoder
    es = open(os.path.join(HERE, "golden", name + ".es"), "rb").read()
    olib = helpers.oracle_lib()
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=olib)
    d.write(0, [es])
    seq = olib.oracle_seq_params(d.decoder).contents
    mb = seq.mb_size
    lib = emu_lib()
    lib.emu_set_quant(bytes(seq.intra_q), bytes(seq.non_intra_q))
    lib.emu_expand_picture.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    mbw, mbh = stream_geometry(es)
    buf = np.frombuffer(es + b"\0" * 16, dtype=np.uint8).copy()
    checked = 0
    while d.decode():
        info = olib.oracle_last_picture_info(d.decoder).contents
        want_hdr = np.ctypeslib.as_array(ctypes.cast(olib.oracle_last_mb_records(d.decoder), ctypes.POINTER(ctypes.c_uint32)),
                                         shape=(mb, 4)).copy()
        want = np.ctypeslib.as_array(ctypes.cast(olib.oracle_last_coefficients(d.decoder), ctypes.POINTER(ctypes.c_int16)),
                                     shape=(mb * 6, 64)).copy()
        h = want_hdr.view(np.uint8).reshape(mb, 16)
        present = (h[:, 4] & 1).astype(bool)
        for lanes in (1, 0):
            hdr = np.zeros(mb * 4, dtype=np.uint32)
            park = np.zeros(mb * 6 * 2, dtype=np.uint32)
            coef = np.zeros(mb * 6 * 32, dtype=np.uint32)
            pinfo = np.zeros(12, dtype=np.int32)
            lib.emu_walk_picture(buf.ctypes.data, len(es), info.start_byte, mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                                 pinfo.ctypes.data, lanes)
            lib.emu_expand_picture(buf.ctypes.data, len(es), mbw, mbh, hdr.ctypes.data, park.ctypes.data, coef.ctypes.data,
                                   pinfo.ctypes.data)
            got = coef.view(np.int16).reshape(mb * 6, 64)
            for blk in range(6):
                rows = np.nonzero(present & ((h[:, 5] & (0x20 >> blk)) != 0))[0] * 6 + blk
                assert np.array_equal(got[rows], want[rows]), f"{name}: picture at byte {info.start_byte}, lanes={lanes}, block {blk}"
        checked += 1
    assert checked > 0


def _pipeline_against_oracle_planes(es, name, define=None, walk_mode=1):
    from jsmpeg_b200 import decoder
    olib = helpers.oracle_lib()
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=olib)
    d.write(0, [es])
    seq = olib.oracle_seq_params(d.decoder).contents
    mb = seq.mb_size
    lib = emu_lib(define)
    lib.emu_set_quant(bytes(seq.intra_q), bytes(seq.non_intra_q))
    lib.emu_expand_picture.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.emu_reconstruct_picture.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                            ctypes.c_int, ctypes.c_int]
    mbw, mbh = stream_geometry(es)
    buf = np.frombuffer(es + b"\0" * 16, dtype=np.uint8).copy()
    ysize = mb * 256
    # Y | Cr | Cb, ping-pong (mpeg1.js:221-246), with the product's readable slack behind (coded width + 64)
    planes = [np.zeros(ysize * 3 // 2 + mbw * 16 + 64, dtype=np.uint8) for _ in range(2)]
    cur = 0
    checked = 0
    while d.decode():
        info = olib.oracle_last_picture_info(d.decoder).contents
        hdr = np.zeros(mb * 4, dtype=np.uint32)
        park = np.zeros(mb * 6 * 2, dtype=np.uint32)
        coef = np.zeros(mb * 6 * 32, dtype=np.uint32)
        pinfo = np.zeros(12, dtype=np.int32)
        lib.emu_walk_picture(buf.ctypes.data, len(es), info.start_byte, mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                             pinfo.ctypes.data, walk_mode)
        if pinfo[2] != 1:
            continue  # B / D picture or P without f_code: consumed, nothing decoded, no swap (mpeg1.js:181-193)
        lib.emu_expand_picture(buf.ctypes.data, len(es), mbw, mbh, hdr.ctypes.data, park.ctypes.data, coef.ctypes.data,
                               pinfo.ctypes.data)
        lib.emu_reconstruct_picture(hdr.ctypes.data, coef.ctypes.data, planes[cur].ctypes.data, planes[cur ^ 1].ctypes.data, mbw, mbh)
        y, cr, cb = d.planes()
        got = planes[cur]
        assert np.array_equal(got[:ysize], y), f"{name}: picture {checked}: Y differs"
        assert np.array_equal(got[ysize:ysize + ysize // 4], cr), f"{name}: picture {checked}: Cr differs"
        assert np.array_equal(got[ysize + ysize // 4:ysize * 3 // 2], cb), f"{name}: picture {checked}: Cb differs"
        cur ^= 1
        checked += 1
    assert checked > 0
    return checked


@pytest.mark.parametrize("name", GOLDEN)
def test_whole_hot_path_device_code_matches_the_oracle_planes(name):
    """The whole hot path on the CPU: emulated walk (lane-parallel) -> stage 1b -> stage 2
    (jsmpeg_b200/csrc/recon.cuh, a warp = 32 coroutines, the TMA copy and the packed instructions
    replaced by plain C) with the product's ping-pong planes, against the ORACLE's planes of every
    decoded picture.  Bit-exact, like the GPU parity tests -- which remain the check of the real thing."""
    _pipeline_against_oracle_planes(open(os.path.join(HERE, "golden", name + ".es"), "rb").read(), name)


@pytest.mark.parametrize("name", GOLDEN)
def test_whole_hot_path_with_the_slice_walk_matches_the_oracle_planes(name):
    """The same with stage 1a = the slice walk (walk_slices.cuh, a lane per slice; its serial fall-back where a
    picture is outside its clean domain)."""
    _pipeline_against_oracle_planes(open(os.path.join(HERE, "golden", name + ".es"), "rb").read(), name, walk_mode=4)


def test_whole_hot_path_device_code_on_an_encoder_clip():
    """The same on an FFmpeg-made I+P clip (one slice per picture, half-pel vectors everywhere)."""
    pytest.importorskip("cv2")
    es = b"".join(p for _, p in helpers.clip_packets(320, 240, 14))
    assert _pipeline_against_oracle_planes(es, "clip 320x240") == 14
