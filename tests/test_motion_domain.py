"""Stage 2 over the whole motion-vector domain, without a GPU.

tools/synth_es.py's Knobs.vectors draws vectors over the f_code's whole range ("wide"), footprints that wrap from one
row into the next by flat index ("wrap"), taps outside the plane ("outside") and all of them per macroblock ("mixed");
synth_es.VECTOR_CASES are the streams.  Here:
  * the generator: its default draws are unchanged, and each domain really occurs in the oracle's records;
  * the oracle's planes equal tools/recon_model.py, a plain numpy statement of stage 2's rules, picture for picture;
  * the compiled reference decodes the "wide" and "wrap" I/P streams as the oracle does (tests/golden/reference);
  * the device code (walk, stage 1b, stage 2 incl. its per-tap slow path), emulated on the host, equals the oracle.
The GPU twin is tests/test_gpu_motion_domain.py.
"""
import functools
import hashlib
import os
from collections import Counter

import numpy as np
import pytest

import accumulate_model
import chain_model
import helpers
import recon_model
import synth_es
from test_b_pictures import _emulated_b_pipeline
from test_picture_index import fresh_decode
from test_walk_emu import _pipeline_against_oracle_planes

IP_CASES = sorted(n for n, s in synth_es.VECTOR_CASES.items() if not s["knobs"].get("b_frames"))
B_CASES = sorted(n for n, s in synth_es.VECTOR_CASES.items() if s["knobs"].get("b_frames"))
# the cases every tap of which the compiled reference reads inside its planes (the "outside" taps read its heap)
REFERENCE_CASES = [n for n in IP_CASES if synth_es.VECTOR_CASES[n]["knobs"]["vectors"] in ("wide", "wrap")]
# what the cases not committed under tests/golden/ are (SHA-256, first 16 hex digits): the default draws stay put
B_CASE_SHA256 = {"b_rows": "4ee2008d787e342b", "b_one_slice_fcodes": "8dbd0c395b66ba8f",
                 "b_random_slices": "0e3d5bac7141d47a", "b_three": "ff6d0b56e9776653"}


def mode(name):
    return synth_es.VECTOR_CASES[name]["knobs"]["vectors"]


@functools.lru_cache(maxsize=None)
def stream(name):
    return synth_es.make_case(name)


@functools.lru_cache(maxsize=None)
def oracle_run(name, decode_b):
    """[(start byte, picture_info, records, coefficients, Y | Cr | Cb)] of every picture the oracle's decode() consumes"""
    got, mbw, mbh = accumulate_model.oracle_decode(helpers.oracle_lib(), stream(name), decode_b=decode_b)
    return got, mbw, mbh


def model_replay(name, decode_b):
    """The oracle's pictures next to the model's, the model fed the oracle's records and coefficients and the planes the
    model itself made before: (picture type, oracle planes, model planes) per reconstructed picture."""
    got, mbw, mbh = oracle_run(name, decode_b)
    size = mbw * mbh * 384
    refs = [np.zeros(size, np.uint8), np.zeros(size, np.uint8)]  # older, newer I/P picture
    b_sets = [np.zeros(size, np.uint8), np.zeros(size, np.uint8)]  # B pictures are written to two sets in turn
    b_cur = 0
    out = []
    for _, info, rec, coef, planes in got:
        if info.status != 1:
            continue
        if info.picture_type == 3:
            mine = recon_model.reconstruct(rec, coef, refs[0], b_sets[b_cur], mbw, mbh, bwd=refs[1])
            b_sets[b_cur] = mine
            b_cur ^= 1
        else:
            mine = recon_model.reconstruct(rec, coef, refs[1], refs[0], mbw, mbh)
            refs = [refs[1], mine]
        out.append((info.picture_type, planes, mine))
    return out


def domain_counts(name, decode_b):
    got, mbw, mbh = oracle_run(name, decode_b)
    total = Counter()
    for _, info, rec, _, _ in got:
        if info.status == 1 and info.picture_type in (2, 3):
            total += recon_model.categories(rec, mbw, mbh, info.picture_type)
    return total


# ---- the generator ---------------------------------------------------------------------------------------------------

def test_default_knobs_reproduce_the_committed_cases():
    for name in synth_es.CASES:
        with open(os.path.join(helpers.GOLDEN, name + ".es"), "rb") as f:
            assert synth_es.make_case(name) == f.read(), name
    for name, digest in B_CASE_SHA256.items():
        assert hashlib.sha256(synth_es.make_case(name)).hexdigest()[:16] == digest, name


# per domain: the categories (recon_model.categories) its streams (I/P and I/P/B) must contain at least this often,
# counted from the ORACLE's records, and those they must not contain
WANT = {
    "wide": {"large": 1000, "neg_odd": 100, "parity_00": 100, "parity_01": 100, "parity_10": 100, "parity_11": 100},
    "wrap": {"wrap": 1000, "large": 50, "neg_odd": 100, "parity_00": 30, "parity_01": 30, "parity_10": 30, "parity_11": 30},
    "outside": {"one_row_out": 200, "far_out": 100, "partly_out": 100, "chroma_only_out": 3, "neg_odd_edge": 10,
                "parity_00": 30, "parity_01": 30, "parity_10": 30, "parity_11": 30},
    "mixed": {"wrap": 100, "one_row_out": 50, "far_out": 50, "partly_out": 50, "large": 10, "neg_odd_edge": 5,
              "parity_00": 50, "parity_01": 50, "parity_10": 50, "parity_11": 50},
}
NEVER = {"wide": ("wrap", "one_row_out", "far_out", "partly_out", "chroma_only_out"),
         "wrap": ("one_row_out", "far_out", "partly_out", "chroma_only_out")}


@pytest.mark.parametrize("domain", sorted(WANT))
def test_each_domain_occurs_in_the_oracles_records(domain):
    counts = Counter()
    for name in sorted(synth_es.VECTOR_CASES):
        if mode(name) == domain:
            counts += domain_counts(name, name in B_CASES)
    for key, least in WANT[domain].items():
        assert counts[key] >= least, (domain, key, counts)
    for key in NEVER.get(domain, ()):
        assert counts[key] == 0, (domain, key, counts)


def test_the_streams_have_every_macroblock_coded():
    """No slice gaps: every picture's chain codes every macroblock, so decode_pictures / seek_pictures of any listed
    picture give the sequential decode's picture (the GPU tests compare them with it)."""
    for name in sorted(synth_es.VECTOR_CASES):
        decode_b = name in B_CASES
        got, mbw, mbh = oracle_run(name, decode_b)
        assert all(info.n_present == mbw * mbh for _, info, _, _, _ in got if info.status == 1), name
        if mbw * mbh > 2000:
            continue  # (the fresh decodes of the large ones cost more than they add)
        seq = {start - 4: planes for start, info, _, _, planes in got if info.status == 1}
        positions = chain_model.picture_positions(stream(name))
        for entry in chain_model.picture_index(stream(name), decode_b):
            planes, _, _ = fresh_decode(stream(name), entry, decode_b)
            assert np.array_equal(np.concatenate([np.ravel(p) for p in planes]), seq[positions[entry["picture"]]]), \
                (name, entry["picture"])


# ---- the model -------------------------------------------------------------------------------------------------------

def test_model_idct_is_the_references():
    stored = np.load(os.path.join(helpers.REFERENCE_DATA, "idct.npz"))
    for kind in ("random", "sparse_extreme"):
        assert np.array_equal(recon_model.idct(stored[kind + "_in"]), stored[kind + "_out"]), kind


def test_model_rules_on_hand_made_records_with_the_intra_dc_x_256():
    """One macroblock of 2 x 2 on a ramp, each rule in isolation: flat-index wrap, the four roundings, a tap out, chroma
    truncation toward zero, B averaging, absent and intra macroblocks, dc_only."""
    mbw, mbh = 2, 2
    size = mbw * mbh * 384
    ref = (np.arange(size) * 7 % 251).astype(np.uint8)
    zero = np.zeros(mbw * mbh * 6 * 64, np.int16)

    def rec(**kw):
        r = np.zeros(mbw * mbh, recon_model.mm.RECORD)
        r["flags"] = recon_model.MBF_PRESENT
        for k, v in kw.items():
            r[k][1] = v  # macroblock (row 0, col 1)
        return r

    cw = mbw * 16
    # h = 2: one sample right; block 1 of macroblock 1 reads across the row's end into the next row's first samples
    out = recon_model.reconstruct(rec(mv_h=2), zero, ref, np.zeros(size, np.uint8), mbw, mbh)
    y = out[:mbw * mbh * 256].reshape(-1, cw)
    assert y[0, 31] == ref[32] and y[0, 16] == ref[17]
    # h = 3, v = 1: the four-tap rounding, luma and chroma (h / 2 = 1, v / 2 = 0: horizontal half only)
    out = recon_model.reconstruct(rec(mv_h=3, mv_v=1), zero, ref, np.zeros(size, np.uint8), mbw, mbh)
    r32 = ref.astype(int)
    assert out[16] == (r32[17] + r32[18] + r32[17 + cw] + r32[18 + cw] + 2) >> 2
    ysz = mbw * mbh * 256
    assert out[ysz + 8] == (r32[ysz + 8] + r32[ysz + 9] + 1) >> 1
    # v = -2 at the top row: the block's first row is outside the plane, zeroed; the second row is the first one's
    out = recon_model.reconstruct(rec(mv_v=-2), zero, ref, np.zeros(size, np.uint8), mbw, mbh)
    assert (out[16:32] == 0).all() and (out[cw + 16:cw + 32] == ref[16:32]).all()
    # h = -1: chroma -1 / 2 = 0 (truncation), where -1 >> 1 = -1 would read one sample to the left
    out = recon_model.reconstruct(rec(mv_h=-1), zero, ref, np.zeros(size, np.uint8), mbw, mbh)
    assert (out[ysz + 8:ysz + 16] == ref[ysz + 8:ysz + 16]).all()
    # B: forward h = 2, backward v = 2, averaged with rounding up
    bwd = ref[::-1].copy()
    out = recon_model.reconstruct(rec(mv_h=2, bwd_y=2, flags=recon_model.MBF_PRESENT | recon_model.MBF_MOTION_FWD |
                                      recon_model.MBF_MOTION_BWD), zero, ref, np.zeros(size, np.uint8), mbw, mbh, bwd=bwd)
    assert out[16] == (r32[17] + int(bwd[16 + cw]) + 1) >> 1
    # absent keeps, intra saturates its residual, dc_only fills the block with (c0 * 32 + 128) >> 8 added to the prediction
    cur = np.full(size, 9, np.uint8)
    coef = zero.copy()
    coef[(1 * 6 + 0) * 64] = 100
    coef[(1 * 6 + 0) * 64 + 5] = 7  # ignored by the dc_only shortcut
    r = rec(flags=0)
    assert np.array_equal(recon_model.reconstruct(r, coef, ref, cur, mbw, mbh)[16:32], cur[16:32])
    r = rec(cbp=0x20, dc_only=0x20)
    out = recon_model.reconstruct(r, coef, ref, cur, mbw, mbh)
    assert (out[16:24] == np.clip(ref[16:24].astype(int) + ((100 * 32 + 128) >> 8), 0, 255)).all()
    r = rec(cbp=0x20, flags=recon_model.MBF_PRESENT | recon_model.MBF_INTRA)
    out = recon_model.reconstruct(r, coef, ref, cur, mbw, mbh)
    blk = np.zeros(64, np.int64)
    blk[0], blk[5] = 100, 7
    pm = recon_model.mm.PREMULTIPLIER.copy()
    pm[0] = 256  # an intra block's coefficient 0 is its dc itself, x 256 (jsmpeg_b200/csrc/records.h)
    want = np.clip(recon_model.idct(blk * pm), 0, 255).reshape(8, 8)
    assert np.array_equal(out[:ysz].reshape(-1, cw)[:8, 16:24], want)
    assert (out[:ysz].reshape(-1, cw)[:8, 24:32] == 0).all()  # an intra block without coefficients: 0


@pytest.mark.parametrize("name", sorted(synth_es.VECTOR_CASES))
def test_oracle_equals_the_model(name):
    """Picture for picture, I/P and (with the extension on) B: pins the oracle's out-of-plane rule to a plain statement"""
    for decode_b in ((False, True) if name in B_CASES else (False,)):
        pics = model_replay(name, decode_b)
        assert len(pics) >= 3
        for k, (ptype, want, mine) in enumerate(pics):
            if not np.array_equal(want, mine):
                bad = np.nonzero(want != mine)[0]
                raise AssertionError(f"{name} decode_b={decode_b}: picture {k} (type {ptype}): {len(bad)} samples differ, "
                                     f"first at {bad[:6]}: oracle {want[bad[:6]]} model {mine[bad[:6]]}")
        assert (3 in {t for t, _, _ in pics}) == decode_b


@pytest.mark.parametrize("name", REFERENCE_CASES)
def test_oracle_equals_the_compiled_reference(name):
    """The compiled reference (its decodes stored in tests/golden/reference/decodes.json) on the streams whose taps all
    lie inside its planes: row-wrapping vectors are a parity target."""
    packets = [(0.0, stream(name))]
    frames, idx, d = helpers.decode_all(helpers.oracle_lib(), packets)
    helpers.assert_frames_match_reference(frames, idx, packets, f"{name}: oracle vs compiled reference")
    d.destroy()


# ---- the device code, emulated ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("walk_mode", [1, 4])
@pytest.mark.parametrize("name", IP_CASES)
def test_emulated_device_code_equals_the_oracle_ip(name, walk_mode):
    """walk (lane-parallel: 1, slice walk: 4) -> stage 1b -> stage 2, on the host, against the oracle's planes"""
    pictures = synth_es.VECTOR_CASES[name]["knobs"]["pictures"]
    assert _pipeline_against_oracle_planes(stream(name), name, walk_mode=walk_mode) == pictures


@pytest.mark.parametrize("name", B_CASES)
def test_emulated_device_code_equals_the_oracle_b(name):
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(1)
    try:
        checked, n_b = _emulated_b_pipeline(stream(name), name)
    finally:
        lib.oracle_set_decode_b(0)
    assert checked == synth_es.VECTOR_CASES[name]["knobs"]["pictures"] and n_b > 0


# ---- random records: every flag, cbp and coefficient form, vectors from 0 to the int16 extremes ------------------------

def random_picture(seed, mb_width, mb_height):
    """(records, coefficients, forward planes, current planes) of a random picture of mb_width x mb_height macroblocks:
    absent, intra, skipped and predicted macroblocks, any cbp, dc_only only on blocks whose one value is coefficient 0
    (uncoded blocks carry garbage coefficients and dc_only bits, which stage 2 must ignore), blocks of at most 12 values
    (compact records) and of more (dense ones), values over [-2048, 2047] and intra DC over [-32767, 32767], vectors
    small, medium, large, at the int16 extremes and aimed at the plane edges; where the picture is big enough, warps
    built on purpose: 31 lanes on the fast path and 1 on the per-tap one, 1 half-sample lane among full-sample ones."""
    rng = np.random.default_rng(seed)
    n = mb_width * mb_height
    cw, ch = mb_width * 16, mb_height * 16
    rec = np.zeros(n, recon_model.mm.RECORD)
    kind = rng.integers(0, 4, n)  # absent, intra, skipped, predicted
    rec["cbp"] = rng.integers(0, 64, n)
    row, col = np.divmod(np.arange(n), mb_width)

    def component(here, size):
        form = rng.integers(0, 5, n)
        edge = np.where(rng.random(n) < 0.5, -here + rng.integers(-2, 3, n), size - 16 - here + rng.integers(-2, 3, n))
        v = np.select([form == 0, form == 1, form == 2, form == 3],
                      [rng.integers(-8, 9, n), rng.integers(-300, 301, n), rng.integers(-4000, 4001, n),
                       rng.choice([-32768, -32767, 32766, 32767], n)], 2 * edge + rng.integers(0, 2, n))
        return np.clip(v, -32768, 32767)

    rec["mv_h"], rec["mv_v"] = component(col * 16, cw), component(row * 16, ch)
    if mb_width >= 32 and mb_height >= 4:
        # row 0, macroblocks 0-15 (the first warp: their top luma blocks): full-sample vectors inside the plane, but
        # macroblock 3's reaches one sample left of the plane with block 0 and stays inside with block 1
        kind[:16] = 3
        rec["mv_h"][:16], rec["mv_v"][:16] = 4, 4
        rec["mv_h"][3], rec["mv_v"][3] = -2 * 3 * 16 - 2, 0
        # row 2, macroblocks 0-31 (a warp of Cb blocks): chroma vectors (2, -2) but macroblock 7's (1, -2)
        r2 = 2 * mb_width
        kind[r2:r2 + 32] = 3
        rec["mv_h"][r2:r2 + 32], rec["mv_v"][r2:r2 + 32] = 4, -4
        rec["mv_h"][r2 + 7] = 2
    rec["flags"] = np.select([kind == 0, kind == 1, kind == 2], [0, recon_model.MBF_PRESENT | recon_model.MBF_INTRA,
                                                                 recon_model.MBF_PRESENT | 0x04], recon_model.MBF_PRESENT)
    coef = rng.integers(-2048, 2048, (n, 6, 64)).astype(np.int16)  # (the uncoded blocks keep this garbage)
    dc_only = rng.integers(0, 64, n)  # (garbage on uncoded blocks)
    intra = kind == 1
    for mb in range(n):
        for b in range(6):
            bit = 0x20 >> b
            if not (kind[mb] and rec["cbp"][mb] & bit):
                continue
            form = rng.integers(0, 3)
            blk = np.zeros(64, np.int64)
            if form == 0:  # DC only (dc_only set most of the time; the full transform gives the same without it)
                count = 0
                dc_only[mb] = dc_only[mb] | bit if rng.random() < 0.7 else dc_only[mb] & ~bit
            else:
                count = int(rng.integers(1, 13)) if form == 1 else int(rng.integers(13, 65))
                dc_only[mb] &= ~bit
            at = rng.choice(np.arange(1, 64), size=min(count, 63), replace=False)
            blk[at] = rng.choice(np.r_[np.arange(-2048, 0), np.arange(1, 2048)], size=len(at))
            if form == 0 or rng.random() < 0.8:
                blk[0] = rng.integers(-32767, 32768) if intra[mb] else rng.integers(-2048, 2048)
            coef[mb, b] = blk
    rec["dc_only"] = dc_only
    fwd = rng.integers(0, 256, n * 384).astype(np.uint8)
    cur = rng.integers(0, 256, n * 384).astype(np.uint8)
    return rec, coef.reshape(-1), fwd, cur


RECORD_SHAPES = [(1, 1), (2, 3), (45, 30), (80, 68)]  # (mb_width, mb_height)


@pytest.mark.parametrize("mb_width,mb_height", RECORD_SHAPES[:3])
def test_emulated_stage2_on_random_records_equals_the_model(mb_width, mb_height):
    """recon.cuh's plain path on the host (dense records) against the model; the GPU twin runs the real kernel"""
    import ctypes

    from test_walk_emu import emu_lib
    lib = emu_lib()
    vp = ctypes.c_void_p
    lib.emu_reconstruct_picture.argtypes = [vp, vp, vp, vp, ctypes.c_int, ctypes.c_int]
    for seed in range(3):
        rec, coef, fwd, cur = random_picture(seed, mb_width, mb_height)
        pad = np.zeros(mb_width * 16 + 64, np.uint8)
        out = np.concatenate([cur, pad])
        ref = np.concatenate([fwd, pad])
        lib.emu_reconstruct_picture(rec.ctypes.data, coef.ctypes.data, out.ctypes.data, ref.ctypes.data, mb_width, mb_height)
        want = recon_model.reconstruct(rec, coef, fwd, cur, mb_width, mb_height)
        bad = np.nonzero(out[:len(cur)] != want)[0]
        assert not len(bad), (seed, len(bad), bad[:8], out[bad[:8]], want[bad[:8]])
