"""The value domain of intra DC and coefficients WITHOUT a GPU (the GPU side: tests/test_gpu_value_domain.py), on
synth_es.VALUE_CASES: intra DC predictors far outside 0..255 -- past +-4095, where 8 * dc leaves int16, past the
records' clamp INTRA_DC_BOUND and up to about +-300,000 -- next to AC coefficients that make dc + ac(x) cross 0 and 255;
every escape form, quantiser scales 0 and 31, matrix entries 0 and 255.

  * the oracle against the compiled reference's recorded decodes, every picture and every bit index;
  * the device code built for the host (walk: serial, lane-parallel and slice walk; stage 1b; stage 2) against the
    same recorded decodes, and every walk's records against the serial one's;
  * tools/macroblock_model.py and tools/recon_model.py against the oracle, and the decode_residuals rule (the clamped
    residual of an intra block is the decoded block);
  * coverage: the cases reach what their names promise, and saturating the DC at +-4095 changes decoded samples.
"""
import ctypes
import functools
import os
import re

import numpy as np
import pytest

import helpers
import macroblock_model
import recon_model
import synth_es
from test_walk_emu import check_stream, emu_lib, stream_geometry

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = sorted(synth_es.VALUE_CASES)
B_CASES = sorted(synth_es.VALUE_B_CASES)
INTRA_DC_BOUND = int(re.search(r"#define INTRA_DC_BOUND (\d+)",
                               open(os.path.join(HERE, "..", "jsmpeg_b200", "csrc", "records.h")).read()).group(1))


@functools.lru_cache(maxsize=None)
def stream(name):
    return synth_es.make_case(name)


@functools.lru_cache(maxsize=None)
def oracle_pictures(name):
    """[(picture_info fields, records, coefficient plane, Y | Cr | Cb, (least, greatest) intra DC predictor)] of every
    picture the oracle reconstructs (B pictures off)"""
    lib = helpers.oracle_lib()
    lib.oracle_last_dc_range.argtypes = [ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
    from jsmpeg_b200 import decoder
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=lib)
    d.write(0.0, [stream(name)])
    mb = lib.oracle_seq_params(d.decoder).contents.mb_size
    out = []
    while d.decode():
        info = lib.oracle_last_picture_info(d.decoder).contents
        if info.status != 1:
            continue
        lo, hi = ctypes.c_int(), ctypes.c_int()
        lib.oracle_last_dc_range(ctypes.byref(lo), ctypes.byref(hi))
        rec = np.ctypeslib.as_array(ctypes.cast(lib.oracle_last_mb_records(d.decoder), ctypes.POINTER(ctypes.c_uint8)),
                                    shape=(mb * 16,)).copy()
        coef = np.ctypeslib.as_array(ctypes.cast(lib.oracle_last_coefficients(d.decoder), ctypes.POINTER(ctypes.c_int16)),
                                     shape=(mb * 384,)).copy()
        planes = np.concatenate([np.ravel(p).copy() for p in d.planes()])
        out.append((info.picture_type, rec, coef, planes, (lo.value, hi.value)))
    d.destroy()
    return out


@pytest.mark.parametrize("name", CASES + B_CASES)
def test_oracle_matches_the_reference(name):
    packets = [(0.0, stream(name))]
    frames, idx, od = helpers.decode_all(helpers.oracle_lib(), packets)
    helpers.assert_frames_match_reference(frames, idx, packets, f"{name}: oracle")
    assert len(frames) >= 1
    od.destroy()


def _emulated_frames(es, walk_mode):
    """Y | Cr | Cb of every picture the device code built for the host reconstructs (walk of `walk_mode`: 0 serial, 1
    lane-parallel, 4 slice walk; stage 1b; stage 2 with the product's ping-pong planes), and how many pictures the lane
    walk took"""
    olib = helpers.oracle_lib()
    from jsmpeg_b200 import decoder
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=olib)
    d.write(0, [es])
    seq = olib.oracle_seq_params(d.decoder).contents
    mb = seq.mb_size
    lib = emu_lib()
    lib.emu_set_quant(bytes(seq.intra_q), bytes(seq.non_intra_q))
    lib.emu_expand_picture.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.emu_reconstruct_picture.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                            ctypes.c_int, ctypes.c_int]
    mbw, mbh = stream_geometry(es)
    buf = np.frombuffer(es + b"\0" * 16, dtype=np.uint8).copy()
    ysize = mb * 256
    planes = [np.zeros(ysize * 3 // 2 + mbw * 16 + 64, dtype=np.uint8) for _ in range(2)]
    cur, frames, lanes = 0, [], 0
    while d.decode():
        info = olib.oracle_last_picture_info(d.decoder).contents
        hdr = np.zeros(mb * 4, dtype=np.uint32)
        park = np.zeros(mb * 6 * 2, dtype=np.uint32)
        coef = np.zeros(mb * 6 * 32, dtype=np.uint32)
        pinfo = np.zeros(12, dtype=np.int32)
        lib.emu_walk_picture(buf.ctypes.data, len(es), info.start_byte, mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                             pinfo.ctypes.data, walk_mode)
        if pinfo[2] != 1:
            continue
        lanes += int(pinfo[9] == 1)
        lib.emu_expand_picture(buf.ctypes.data, len(es), mbw, mbh, hdr.ctypes.data, park.ctypes.data, coef.ctypes.data,
                               pinfo.ctypes.data)
        lib.emu_reconstruct_picture(hdr.ctypes.data, coef.ctypes.data, planes[cur].ctypes.data, planes[cur ^ 1].ctypes.data,
                                    mbw, mbh)
        got = planes[cur]
        frames.append((got[:ysize].copy(), got[ysize:ysize * 5 // 4].copy(), got[ysize * 5 // 4:ysize * 3 // 2].copy()))
        cur ^= 1
    d.destroy()
    return frames, lanes


@pytest.mark.parametrize("walk_mode", [0, 1, 4], ids=["serial", "lanes", "slice_walk"])
@pytest.mark.parametrize("name", CASES)
def test_emulated_device_code_matches_the_reference(name, walk_mode):
    """Walk, stage 1b and stage 2 as the GPU runs them, compiled for the host, give the reference's pictures"""
    frames, lanes = _emulated_frames(stream(name), walk_mode)
    want = helpers.reference_decode([(0.0, stream(name))])["fnv1a64"]
    got = helpers.frame_hashes(frames)
    assert len(got) == len(want), (name, len(got), len(want))
    bad = [k for k in range(len(got)) if got[k] != want[k]]
    assert not bad, f"{name} walk {walk_mode}: pictures {bad} differ from the reference"
    if walk_mode == 1 and synth_es.VALUE_CASES[name] and synth_es.VALUE_CASES[name]["knobs"]["slices"] == "one":
        assert lanes == len(frames), f"{name}: the lane-parallel walk took {lanes} of {len(frames)} pictures"


@pytest.mark.parametrize("name", CASES + B_CASES)
def test_every_walk_parks_the_same_records(name):
    """The lane walk's relative DC sums (fixed up across lane boundaries), the slice walk and the serial walk agree on
    every record and every parked DC, clamp included"""
    check_stream(emu_lib(), stream(name), name)


@pytest.mark.parametrize("name", CASES)
def test_models_match_the_oracle(name):
    """macroblock_model's coefficient export and residual, recon_model's planes, against the oracle's own decode"""
    w, h = stream_geometry(stream(name))
    prev = None
    for k, (ptype, rec, coef, planes, _) in enumerate(oracle_pictures(name)):
        fwd = prev if prev is not None else np.zeros_like(planes)
        got = recon_model.reconstruct(rec, coef, fwd, np.zeros_like(planes), w, h)
        assert np.array_equal(got, planes), (name, k)
        r = np.frombuffer(rec.tobytes(), macroblock_model.RECORD)
        intra = (r["flags"] & macroblock_model.MBF_INTRA) != 0
        res = macroblock_model.residuals(rec, coef, w, h)
        assert np.abs(res.astype(np.int64)).max() <= 255 + 2 * INTRA_DC_BOUND
        # decode_residuals' rule: an intra macroblock's samples are its residual, clamped
        ysz = w * h * 256
        for _, off, stride, rows, px in recon_model.planes_layout(w, h):
            sl = slice(off, off + stride * rows)
            s_intra = recon_model._per_sample(intra.reshape(h, w), px).reshape(-1)
            assert np.array_equal(np.clip(res[sl], 0, 255)[s_intra], planes[sl][s_intra]), (name, k)
        # decode_coefficients: intra DC as sat16(8 * dc), everything else as the records hold it
        exp = macroblock_model.coefficients(rec, coef).astype(np.int64)
        raw = macroblock_model.records_coefficients(rec, coef).astype(np.int64)
        assert np.array_equal(exp[:, :, 1:], raw[:, :, 1:])
        assert np.array_equal(exp[intra, :, 0], np.clip(8 * raw[intra, :, 0], -32768, 32767))
        assert ysz * 3 // 2 == len(planes)
        prev = planes


def test_the_cases_reach_the_value_domain():
    """The oracle's DC predictors: past +-4095 and past the records' clamp in both directions, about +-300,000 in the
    one-slice 320x240 pictures; and saturating the DC at +-4095 (the old 8 * dc in int16) changes decoded samples of
    most cases, the repro among them"""
    lo = min(p[4][0] for n in CASES for p in oracle_pictures(n))
    hi = max(p[4][1] for n in CASES for p in oracle_pictures(n))
    assert hi >= 290_000 and lo <= -290_000, (lo, hi)
    assert hi < 1 << 23 and lo > -(1 << 23)  # the reference's dc << 8 stays inside int32
    past_clamp = [n for n in CASES if any(max(-p[4][0], p[4][1] - 255) > INTRA_DC_BOUND for p in oracle_pictures(n))]
    assert len(past_clamp) >= 4, past_clamp
    for name in B_CASES:  # (the B pictures' own predictors: tests/test_gpu_value_domain.py)
        assert max(max(-p[4][0], p[4][1]) for p in oracle_pictures(name)) > 4095, name
    changed = []
    for name in CASES:
        w, h = stream_geometry(stream(name))
        prev = None
        n = 0
        for ptype, rec, coef, planes, _ in oracle_pictures(name):
            r = np.frombuffer(rec.tobytes(), macroblock_model.RECORD)
            intra = (r["flags"] & macroblock_model.MBF_INTRA) != 0
            sat = coef.reshape(-1, 6, 64).copy()
            sat[intra, :, 0] = np.clip(sat[intra, :, 0], -4096, 4095)
            fwd = prev if prev is not None else np.zeros_like(planes)
            n += int((recon_model.reconstruct(rec, sat.reshape(-1), fwd, np.zeros_like(planes), w, h) != planes).sum())
            prev = planes
        if n:
            changed.append(name)
    assert "val_repro_96x16" in changed and len(changed) >= 6, changed
