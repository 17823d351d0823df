"""The value domain of intra DC and coefficients on the GPU (the CPU side: tests/test_value_domain.py), on
synth_es.VALUE_CASES and VALUE_B_CASES: intra DC predictors past +-4095, past the records' clamp and up to about
+-300,000, next to AC coefficients that make dc + ac(x) cross 0 and 255; every escape form, quantiser scales 0 and 31.

  * the reference ABI and BatchDecoder.decode() against the compiled reference's recorded decodes (I/P streams) and the
    oracle (B pictures on), with the lane walk, the slice walk and -- in a child process -- the serial walk, in every
    stage-2 variant; the residual and accumulated map against the models;
  * decode_pictures, decode_intra and seek_pictures of every listed picture, decode_frames (planes and RGBA) and its
    decode_frames_into form (with coefficients and accumulated maps), decode_coefficients and decode_residuals against
    the oracle and the models;
  * one batch of the value cases with the bench-like clips, so that compact and dense records meet in one launch.
"""
import os

import numpy as np
import pytest

import helpers
import macroblock_model
import synth_es
from jsmpeg_b200 import capi
from jsmpeg_b200.batch import OUT_ACCUMULATED, OUT_DEVICE, OUT_HOST, OUT_RESIDUALS, OUT_RGBA, BatchDecoder
from test_gpu_motion_domain import _sequential_planes, oracle_maps, oracle_steps
from test_gpu_parity import _canvas2d_rgba

pytestmark = pytest.mark.gpu

IP_CASES = sorted(synth_es.VALUE_CASES)
B_CASES = sorted(synth_es.VALUE_B_CASES)
CASES = IP_CASES + B_CASES


def stream(name):
    return synth_es.make_case(name)


def geometry(name):
    es = stream(name)
    i = es.index(b"\x00\x00\x01\xb3") + 4
    return (es[i] << 4 | es[i + 1] >> 4), ((es[i + 1] & 15) << 8 | es[i + 2])


@pytest.mark.parametrize("name", CASES)
def test_reference_abi_decode_equals_the_reference(name):
    packets = [(0.0, stream(name))]
    got, got_idx, gd = helpers.decode_all(capi.product_library(), packets)
    helpers.assert_frames_match_reference(got, got_idx, packets, f"{name}: CUDA vs compiled reference")
    gd.destroy()


PASSES = [(0, OUT_DEVICE), (1, OUT_HOST | OUT_RGBA), (0, OUT_RESIDUALS | OUT_ACCUMULATED), (1, OUT_RGBA | OUT_RESIDUALS)]


@pytest.mark.parametrize("name", CASES)
def test_batch_decode_equals_the_reference_in_every_stage2_variant(name):
    """decode() with the lane walk and the slice walk, every stage-2 variant: planes and indices against the oracle
    (which test_value_domain pins to the reference on every I/P picture), the first pass's hashes against the reference
    itself, the lane walk's use, RGBA, the residual and the accumulated map against the models"""
    width, height = geometry(name)
    for decode_b in ((0, 1) if name in B_CASES else (0,)):
        want = oracle_steps(name, decode_b)
        maps = oracle_maps(name, decode_b)
        for slice_walk, flags in PASSES:
            what = (name, decode_b, slice_walk, flags)
            bd = BatchDecoder(1, slice_walk=slice_walk, decode_b=decode_b)
            bd.write(0, stream(name))
            res_now, map_now, frames = None, None, []
            for k, (index, status, ptype, planes, res) in enumerate(want):
                assert bd.decode(1, flags) == 1, what + (k,)
                assert bd.get_index(0) == index, what + (k,)
                got = np.concatenate(bd.read_planes(0))
                if not np.array_equal(got, planes):
                    bad = np.nonzero(got != planes)[0]
                    raise AssertionError(f"{what} picture {k} (type {ptype}): {len(bad)} samples differ, first at {bad[:8]}")
                ysz = len(planes) * 2 // 3
                frames.append((got[:ysz], got[ysz:ysz * 5 // 4], got[ysz * 5 // 4:]))
                if status == 1:
                    res_now = res
                    if ptype in (1, 2):
                        map_now = maps[index]
                    if flags & OUT_RGBA:
                        exp = _canvas2d_rgba(planes[:ysz], planes[ysz:ysz * 5 // 4], planes[ysz * 5 // 4:], width, height)
                        assert np.array_equal(bd.read_rgba(0), exp), what + (k, "rgba")
                if flags & OUT_RESIDUALS and res_now is not None:
                    assert np.array_equal(bd.read_residuals(0), res_now), what + (k, "residual")
                if flags & OUT_ACCUMULATED and map_now is not None:
                    assert np.array_equal(bd.read_accumulated(0), map_now), what + (k, "accumulated")
            assert bd.decode(1, flags) == 0
            assert bd.last_error() is None
            if not decode_b:
                helpers.assert_frames_match_reference(frames, [s[0] for s in want], [(0.0, stream(name))], str(what))
            if not slice_walk and synth_es.VALUE_CASES.get(name) and synth_es.VALUE_CASES[name]["knobs"]["slices"] == "one" \
                    and os.environ.get("JSMPEG_B200_WALK") != "serial":
                assert bd.stats()["lane_walk_pictures"] >= sum(s[1] == 1 for s in want), what
            bd.close()


@pytest.mark.parametrize("name", CASES)
def test_decode_pictures_intra_and_seek_equal_the_oracles_decode(name):
    decode_b = name in B_CASES
    want = _sequential_planes(name, decode_b)
    for slice_walk in (0, 1):
        bd = BatchDecoder(1, slice_walk=slice_walk, decode_b=decode_b)
        bd.write(0, stream(name))
        entries = bd.picture_index(0)
        got = bd.decode_pictures([(0, e["picture"]) for e in entries])
        for e, t, i in zip(entries, got, bd.last_pictures_info):
            assert i["status"] == 1, (name, e["picture"], i)
            assert np.array_equal(t.cpu().numpy(), want[e["picture"]]), (name, slice_walk, e["picture"])
        intra = bd.intra_index(0)
        for e, t in zip(intra, bd.decode_intra([(0, e["picture"]) for e in intra])):
            assert np.array_equal(t.cpu().numpy(), want[e["picture"]]), (name, slice_walk, "intra", e["picture"])
        for e in entries[::-1] if slice_walk else entries:
            assert bd.seek_pictures([(0, e["picture"])], OUT_HOST) == 1
            assert np.array_equal(np.concatenate(bd.read_planes(0)), want[e["picture"]]), (name, slice_walk, e["picture"])
        assert bd.last_error() is None
        bd.close()


@pytest.mark.parametrize("name", IP_CASES)
def test_coefficient_and_residual_exports_equal_the_models(name):
    """decode_coefficients: the records' values with an intra DC as sat16(8 * dc); decode_residuals: the transform with
    an intra block's coefficient 0 (its clamped dc) x 256 -- both against the models of the oracle's records"""
    import accumulate_model
    mbw, mbh = [(v + 15) // 16 for v in geometry(name)]
    pics = [p for p in accumulate_model.oracle_decode(helpers.oracle_lib(), stream(name))[0] if p[1].status == 1]
    bd = BatchDecoder(1)
    bd.write(0, stream(name))
    entries = bd.macroblock_index(0)
    assert len(entries) == len(pics)
    reqs = [(0, e["picture"]) for e in entries]
    coefs = bd.decode_coefficients(reqs)
    res = bd.decode_residuals(reqs)
    for k, (_, _, rec, coef, _) in enumerate(pics):
        want = macroblock_model.coefficients(rec, coef).reshape(mbh, mbw, 6, 64)
        got = coefs[k].cpu().numpy().reshape(mbh, mbw, 6, 64)
        assert np.array_equal(got, want), (name, k, "coefficients")
        assert np.array_equal(res[k].cpu().numpy(), macroblock_model.residuals(rec, coef, mbw, mbh)), (name, k, "residuals")
    assert bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("rgba", [False, True])
def test_decode_frames_of_every_case_equal_the_oracle(rgba):
    """decode_frames (planes, fused RGBA) of all the I/P value cases in one batch, one picture per call"""
    want = {n: [s for s in oracle_steps(n, 0) if s[1] == 1] for n in IP_CASES}
    bd = BatchDecoder(len(IP_CASES))
    for s, n in enumerate(IP_CASES):
        bd.write(s, stream(n))
    seen = {n: 0 for n in IP_CASES}
    while True:
        out = bd.decode_frames(1, rgba=rgba)
        if not any(f["n_frames"] for f in out):
            break
        for s, n in enumerate(IP_CASES):
            for j in range(out[s]["n_frames"]):
                planes = want[n][seen[n]][3]
                assert np.array_equal(out[s]["planes"][j].cpu().numpy().reshape(-1), planes), (n, seen[n])
                if rgba:
                    w, h = geometry(n)
                    ysz = len(planes) * 2 // 3
                    exp = _canvas2d_rgba(planes[:ysz], planes[ysz:ysz * 5 // 4], planes[ysz * 5 // 4:], w, h)
                    assert np.array_equal(out[s]["rgba"][j].cpu().numpy().reshape(-1), np.asarray(exp).reshape(-1)), (n, seen[n])
                seen[n] += 1
    assert seen == {n: len(w) for n, w in want.items()}
    assert bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("name", IP_CASES)
def test_decode_frames_into_equals_the_oracle_and_the_models(name):
    """decode_frames with coefficients and accumulated maps (jsmpeg_b200_batch_decode_frames_into), every picture of the
    stream in one call: planes, fused RGBA, residual and map against the oracle and the models, coefficients as
    decode_coefficients reports them"""
    import accumulate_model
    want = [s for s in oracle_steps(name, 0) if s[1] == 1]
    maps = oracle_maps(name, 0)
    pics = [p for p in accumulate_model.oracle_decode(helpers.oracle_lib(), stream(name))[0] if p[1].status == 1]
    w, h = geometry(name)
    mbw, mbh = (w + 15) // 16, (h + 15) // 16
    bd = BatchDecoder(1)
    bd.write(0, stream(name))
    out = bd.decode_frames(len(want), OUT_ACCUMULATED, rgba=True, residuals=True, coefficients=True, accumulated=True)[0]
    assert out["n_frames"] == len(want)
    for k, (index, _, _, planes, res) in enumerate(want):
        ysz = len(planes) * 2 // 3
        assert np.array_equal(out["planes"][k].cpu().numpy().reshape(-1), planes), (name, k)
        exp = _canvas2d_rgba(planes[:ysz], planes[ysz:ysz * 5 // 4], planes[ysz * 5 // 4:], w, h)
        assert np.array_equal(out["rgba"][k].cpu().numpy().reshape(-1), np.asarray(exp).reshape(-1)), (name, k, "rgba")
        assert np.array_equal(out["residuals"][k].cpu().numpy().reshape(-1), res), (name, k, "residual")
        assert np.array_equal(out["accumulated"][k].cpu().numpy().reshape(-1), np.asarray(maps[index]).reshape(-1)), (name, k)
        _, _, rec, coef, _ = pics[k]
        assert np.array_equal(out["coefficients"][k].cpu().numpy().reshape(-1),
                              macroblock_model.coefficients(rec, coef).reshape(-1)), (name, k, "coefficients")
    assert bd.last_error() is None
    bd.close()


def test_one_batch_of_value_cases_and_clips():
    """The value cases (many coded blocks, long escape runs: dense records) in one batch with bench-like clips (compact
    records): every expand and reconstruct launch mixes the two"""
    clips = [b"".join(p for _, p in helpers.clip_packets(320, 240, 8))]
    names = IP_CASES
    bd = BatchDecoder(len(names) + len(clips))
    for s, n in enumerate(names):
        bd.write(s, stream(n))
    for j, es in enumerate(clips):
        bd.write(len(names) + j, es)
    want = [oracle_steps(n, 0) for n in names]
    clip_frames = [helpers.decode_all(helpers.oracle_lib(), [(0.0, es)]) for es in clips]
    want += [[(idx, 1, 0, np.concatenate([np.ravel(p) for p in f]), None) for f, idx in zip(fr, ix)]
             for fr, ix, _ in clip_frames]
    for _, _, od in clip_frames:
        od.destroy()
    done = [0] * len(want)
    while True:
        before = [bd.get_index(s) for s in range(len(want))]
        if not bd.decode(1, OUT_DEVICE):
            break
        for s in range(len(want)):
            if bd.get_index(s) == before[s] or done[s] == len(want[s]):
                continue
            assert bd.get_index(s) == want[s][done[s]][0], (s, done[s])
            assert np.array_equal(np.concatenate(bd.read_planes(s)), want[s][done[s]][3]), (s, done[s])
            done[s] += 1
    assert done == [len(w) for w in want]
    assert bd.last_error() is None
    bd.close()


def test_value_tests_with_the_serial_walk_in_a_child_process():
    """The walk variant is chosen once per process: the decode tests again with JSMPEG_B200_WALK=serial"""
    import subprocess
    import sys
    if os.environ.get("JSMPEG_B200_WALK") == "serial":
        pytest.skip("already running with the serial walk")
    env = dict(os.environ, JSMPEG_B200_WALK="serial")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-x", "-q", "-p",
                        "no:cacheprovider", "-k", "reference and not serial"], env=env, capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
