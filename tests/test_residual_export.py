"""The residual export of decode_residuals WITHOUT a GPU: the block code of the export kernel (idct_block / idct_dc of
jsmpeg_b200/csrc/idct.cuh, coef_record_scatter of coef_records.h) built with g++ against the oracle's transform and
numpy; the vectorised numpy transform of macroblock_model against the oracle and the reference's recorded outputs; a
rigorous bound that keeps every residual inside int16; macroblock_model.residuals pinned to the oracle's own
sequential decode (prediction + residual, or the clamped residual of an intra macroblock, give the decoded samples);
and the export kernel's recorded SASS hash."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import helpers
import macroblock_model
from jsmpeg_b200 import decoder
from test_coefficient_export import numpy_unpack, random_records
from test_macroblock_index import GOLDEN, MINI_ENC, corpus_stream

PM = macroblock_model.PREMULTIPLIER
LO, HI = -2048, 2047  # the clip range of every coefficient


class Planes(ctypes.Structure):  # the oracle's planes_t
    _fields_ = [("y", ctypes.c_void_p), ("cr", ctypes.c_void_p), ("cb", ctypes.c_void_p)]


def planes_struct(buf, n):
    """planes_t over a contiguous Y | Cr | Cb uint8 array of luma size n"""
    base = buf.ctypes.data
    return Planes(base, base + n, base + n + n // 4)


def oracle_idct(blocks):
    """oracle_idct (the oracle's 2-D transform) of premultiplied int blocks [n, 64], one call per block"""
    fn = helpers.oracle_lib().oracle_idct
    out = []
    for b in np.asarray(blocks, np.int64):
        a = (ctypes.c_int * 64)(*[int(x) for x in b])
        fn(a)
        out.append(list(a))
    return np.array(out, np.int64).reshape(-1, 64)


# ---- a rigorous bound: the transform as a linear map plus the error of its rounding steps -----------------------------

class Bound:
    """A value of the transform as the real linear form `form` over the 64 coefficients (premultipliers folded in,
    roundings removed) and a bound `err` on how far the integer computation can be from that form: |int - form . c| <=
    err for every block c.  With |c_j| <= 2048 the value's magnitude is at most |form|_1 * 2048 + err.  Every Bound
    made is seen by `largest`, the magnitude of the biggest intermediate (int32 overflow check)."""
    largest = 0.0

    def __init__(self, form, err):
        self.form, self.err = form, err
        Bound.largest = max(Bound.largest, self.magnitude())

    def magnitude(self):
        return float(np.abs(self.form).sum()) * 2048 + self.err

    def __add__(self, o):
        return Bound(self.form + o.form, self.err + o.err)

    def __sub__(self, o):
        return Bound(self.form - o.form, self.err + o.err)

    def __neg__(self):
        return Bound(-self.form, self.err)

    def __mul__(self, k):
        return Bound(self.form * k, self.err * abs(k))

    def round8(self):
        # (z + 128) >> 8 = floor(z / 256 + 1/2), within 1/2 of z / 256; |z - form . c| <= err carries over as err / 256
        Bound.largest = max(Bound.largest, self.magnitude() + 128)
        return Bound(self.form / 256, self.err / 256 + 0.5)


def transform_bounds():
    """[64] Bound of the outputs of the transform of premultiplied coefficients, through macroblock_model.idct8 -- the
    code the model runs on integers"""
    Bound.largest = 0.0
    v = [Bound(np.eye(64)[j] * PM[j], 0.0) for j in range(64)]
    for c in range(8):  # column passes: elements c, c + 8, ... c + 56
        for k, x in enumerate(macroblock_model.idct8([v[c + 8 * k] for k in range(8)], False)):
            v[c + 8 * k] = x
    for r in range(8):  # row passes
        v[8 * r:8 * r + 8] = macroblock_model.idct8(v[8 * r:8 * r + 8], True)
    return v


def extreme_blocks(bounds):
    """Per output the two coefficient blocks in [-2048, 2047] that drive its linear form furthest up and down"""
    out = []
    for b in bounds:
        out.append(np.where(b.form > 0, HI, LO))
        out.append(np.where(b.form > 0, LO, HI))
    return np.array(out, np.int64)


def test_every_residual_fits_int16():
    """The linear form's L1 norm times 2048 plus the propagated rounding error bounds every output; it is below 32767,
    and every intermediate (including the products before a rounding) stays far below 2^31.  The extreme sign-pattern
    blocks come within a few units of the bound from inside."""
    bounds = transform_bounds()
    limit = max(b.magnitude() for b in bounds)
    assert limit < 14_500 < 32767, limit
    assert Bound.largest < 2 ** 30, Bound.largest
    ext = extreme_blocks(bounds)
    got = macroblock_model.idct(ext * PM)
    assert np.array_equal(got, oracle_idct(ext * PM))
    assert np.abs(got).max() <= limit and np.abs(got).max() > limit - 64, (np.abs(got).max(), limit)


def test_the_numpy_transform_equals_the_reference_and_the_oracle():
    stored = np.load(os.path.join(helpers.REFERENCE_DATA, "idct.npz"))
    for name in ("random", "sparse_extreme"):
        assert np.array_equal(macroblock_model.idct(stored[name + "_in"]), stored[name + "_out"]), name
    rng = np.random.default_rng(5)
    blocks = rng.integers(LO, HI + 1, size=(400, 64)) * PM
    assert np.array_equal(macroblock_model.idct(blocks), oracle_idct(blocks))
    assert macroblock_model.idct(blocks[0]).shape == (64,)


def host_check(tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not available")
    inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(inc, "cuda_runtime.h")):
        pytest.skip("CUDA headers not available")
    exe = tmp_path / "residuals_check"
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", "-Wno-unknown-pragmas", "-I", inc, "-o", str(exe),
                        os.path.join(helpers.ROOT, "tests", "emu", "residuals_check.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def test_the_block_transform_compiled_for_the_host_equals_the_oracle(tmp_path):
    """idct_block of raw coefficients (premultiplied inside, as the kernel does) = oracle_idct of the premultiplied
    block, on random, zero, DC-only and extreme sign-pattern blocks; idct_dc = the full transform of DC-only blocks."""
    exe = host_check(tmp_path)
    rng = np.random.default_rng(9)
    dc = np.zeros((40, 64), np.int64)
    dc[:, 0] = np.concatenate([[LO, HI, -1, 1, 0, 8, -8, 1016, -1024, 255 * 8], rng.integers(LO, HI + 1, 30)])
    sparse = np.zeros((200, 64), np.int64)
    for b in sparse:  # 1 to 12 values, as compact records hold them; a third of the blocks with extreme or tiny ones
        pos = rng.choice(64, rng.integers(1, 13), replace=False)
        b[pos] = rng.choice([LO, HI, -1, 1, 7, -9], len(pos)) if rng.random() < 0.3 else rng.integers(LO, HI + 1, len(pos))
    blocks = np.concatenate([rng.integers(LO, HI + 1, size=(300, 64)), np.zeros((3, 64), np.int64), dc, sparse,
                             np.full((1, 64), LO), np.full((1, 64), HI), extreme_blocks(transform_bounds())])
    path = tmp_path / "blocks.bin"
    path.write_bytes(blocks.astype(np.int16).tobytes())
    out = np.frombuffer(subprocess.run([str(exe), "idct", str(path)], capture_output=True, check=True).stdout,
                        np.int32).reshape(-1, 65)
    want = oracle_idct(blocks * PM)
    assert np.array_equal(out[:, :64], want)
    assert np.array_equal(macroblock_model.idct(blocks * PM), want)
    is_dc = (blocks[:, 1:] == 0).all(axis=1)
    shortcut = (blocks[:, 0] * PM[0] + 128) >> 8
    assert is_dc.sum() >= 43 and np.array_equal(out[is_dc, 64], shortcut[is_dc])
    assert (out[is_dc, :64] == shortcut[is_dc, None]).all()  # the full transform of a DC-only block is the shortcut


def test_the_record_scatter_compiled_for_the_host_equals_numpy_unpacking(tmp_path):
    exe = host_check(tmp_path)
    rec = random_records(np.random.default_rng(4))
    path = tmp_path / "records.bin"
    path.write_bytes(rec.tobytes())
    out = np.frombuffer(subprocess.run([str(exe), "scatter", str(path)], capture_output=True, check=True).stdout, np.int16)
    assert np.array_equal(out.reshape(-1, 64), numpy_unpack(rec))


# ---- the model against the oracle's sequential decode -----------------------------------------------------------------

def sample_mask(per_mb, mb_width, mb_height):
    """[coded_size * 3 // 2] bool in the planes' layout from a [mb_height * mb_width] per-macroblock bool"""
    m = np.asarray(per_mb, bool).reshape(mb_height, mb_width)
    y = np.repeat(np.repeat(m, 16, 0), 16, 1).reshape(-1)
    c = np.repeat(np.repeat(m, 8, 0), 8, 1).reshape(-1)
    return np.concatenate([y, c, c])


def sequential_decode(es):
    """The oracle (B pictures on) fed `es`: per picture its decode() consumes (start code position, picture_info,
    records, coefficient plane, planes afterwards, the prediction of its present non-intra macroblocks).  The
    prediction is the oracle's own reconstruction of the same records with every cbp bit cleared, from the references
    the decode used: for P the newest I/P picture, for B the two newest (older = forward)."""
    lib = helpers.oracle_lib()
    for name, args in (("oracle_reconstruct", [ctypes.POINTER(Planes)] * 2),
                       ("oracle_reconstruct_b", [ctypes.POINTER(Planes)] * 3)):
        getattr(lib, name).restype = None
        getattr(lib, name).argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, *args]
    lib.oracle_set_decode_b(1)
    out = []
    try:
        d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=lib)
        d.write(0.0, [es])
        seq = lib.oracle_seq_params(d.decoder)
        mb, mbw = seq.contents.mb_size, seq.contents.mb_width
        cw, ch = mbw * 16, mb // mbw * 16
        cs = cw * ch
        refs = [np.zeros(cs * 3 // 2, np.uint8)] * 2  # the oracle's planes start zeroed
        while d.decode():
            info = helpers.PictureInfo.from_buffer_copy(lib.oracle_last_picture_info(d.decoder).contents)
            rec = np.ctypeslib.as_array(ctypes.cast(lib.oracle_last_mb_records(d.decoder), ctypes.POINTER(ctypes.c_uint8)),
                                        shape=(mb * 16,)).reshape(mb, 16).copy()
            coef = np.ctypeslib.as_array(ctypes.cast(lib.oracle_last_coefficients(d.decoder), ctypes.POINTER(ctypes.c_int16)),
                                         shape=(mb * 6 * 64,)).copy()
            planes = np.concatenate([np.ctypeslib.as_array(ctypes.cast(p(d.decoder), ctypes.POINTER(ctypes.c_uint8)),
                                                           shape=(n,)).copy()
                                     for p, n in ((lib.mpeg1_decoder_get_y_ptr, cs), (lib.mpeg1_decoder_get_cr_ptr, cs // 4),
                                                  (lib.mpeg1_decoder_get_cb_ptr, cs // 4))])
            pred = np.zeros(cs * 3 // 2, np.uint8)
            if info.status == 1 and info.picture_type in (2, 3):
                hdr = rec.copy()
                hdr[:, 5] = 0  # no block is added: the prediction alone
                fwd = refs[-1] if info.picture_type == 2 else refs[-2]
                f, o = planes_struct(fwd, cs), planes_struct(pred, cs)
                sp = ctypes.cast(seq, ctypes.c_void_p)
                if info.picture_type == 2:
                    lib.oracle_reconstruct(sp, cw, ch, hdr.ctypes.data, coef.ctypes.data, ctypes.byref(f), ctypes.byref(o))
                else:
                    bk = planes_struct(refs[-1], cs)
                    lib.oracle_reconstruct_b(sp, cw, ch, hdr.ctypes.data, coef.ctypes.data, ctypes.byref(f),
                                             ctypes.byref(bk), ctypes.byref(o))
            out.append((info.start_byte - 4, info, rec, coef, planes, pred, mbw, mb // mbw))
            if info.status == 1 and info.picture_type in (1, 2):
                refs = [refs[-1], planes]
        d.destroy()
    finally:
        lib.oracle_set_decode_b(0)
    return out


@pytest.mark.parametrize("name", GOLDEN + ["ffmpeg_320x240", "ffmpeg_1280x720"] + sorted(MINI_ENC))
def test_the_model_gives_what_the_decoder_adds(name):
    """Every listed picture of the oracle's sequential decode: clamp(prediction + residual) is the decoded sample of
    every present non-intra macroblock, clamp(residual) that of every intra macroblock."""
    es = corpus_stream(name)
    listed = {e["byte_pos"] for e in macroblock_model.macroblock_index(es)}
    checked, kinds = 0, set()
    for pos, info, rec, coef, planes, pred, mbw, mbh in sequential_decode(es):
        if info.status != 1 or pos not in listed:
            continue
        res = macroblock_model.residuals(rec, coef, mbw, mbh)
        assert res.dtype == np.int16 and res.shape == planes.shape
        r = np.frombuffer(rec.tobytes(), macroblock_model.RECORD)
        present = (r["flags"] & macroblock_model.MBF_PRESENT) != 0
        intra = present & ((r["flags"] & macroblock_model.MBF_INTRA) != 0)
        pm, im = sample_mask(present & ~intra, mbw, mbh), sample_mask(intra, mbw, mbh)
        got = np.clip(np.where(im, 0, pred.astype(np.int32)) + res, 0, 255)
        assert np.array_equal(got[pm | im], planes[pm | im]), (name, pos, info.picture_type)
        assert not res[~sample_mask(present, mbw, mbh)].any()
        checked += 1
        kinds.add(info.picture_type)
    assert checked == len(listed) > 0 and 1 in kinds, name


def test_the_model_places_blocks_as_the_planes_are_laid_out():
    """One macroblock row of two macroblocks, each block DC-only with its own value: block b of macroblock m covers
    the 8 x 8 samples stage 2 writes (luma quadrants, 4 = Cb = third plane, 5 = Cr = second)"""
    rec = np.zeros((2, 16), np.uint8)
    rec[:, 4], rec[:, 5] = macroblock_model.MBF_PRESENT, 0x3F
    coef = np.zeros((2, 6, 64), np.int16)
    coef[:, :, 0] = (np.arange(12).reshape(2, 6) + 1) * 8 * 4  # every sample of block (m, b) = 4 * (6 m + b + 1)
    res = macroblock_model.residuals(rec, coef.reshape(-1), 2, 1)
    y, cr, cb = res[:512].reshape(16, 32), res[512:640].reshape(8, 16), res[640:].reshape(8, 16)
    val = lambda m, b: 4 * (6 * m + b + 1)
    for m in range(2):
        for b in range(4):
            assert (y[(b >> 1) * 8:(b >> 1) * 8 + 8, m * 16 + (b & 1) * 8:m * 16 + (b & 1) * 8 + 8] == val(m, b)).all()
        assert (cb[:, m * 8:m * 8 + 8] == val(m, 4)).all() and (cr[:, m * 8:m * 8 + 8] == val(m, 5)).all()


def test_the_export_kernel_is_the_measured_one():
    """profiles/sass_hashes_sm90a.txt records the residual export kernel's SASS md5 (tools/sass_hash.py) on the build its
    H100 numbers were taken with; recompiling residuals.cu must give the same machine code."""
    import sys
    if not (shutil.which("nvcc") and shutil.which("cuobjdump")):
        pytest.skip("nvcc / cuobjdump not available")
    sys.path.insert(0, os.path.join(helpers.ROOT, "tools"))
    import sass_hash
    line = next(x for x in open(os.path.join(helpers.ROOT, "profiles", "sass_hashes_sm90a.txt"))
                if "residuals.cu" in x and "export_residuals_kernel" in x)
    recorded = next(p for p in line.split() if len(p) == 32)
    now = {sass_hash.demangle(k): md5 for k, (md5, _) in sass_hash.kernel_hashes("residuals.cu").items()}
    assert now == {"export_residuals_kernel": recorded}
