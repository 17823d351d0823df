"""The picture's geometry and the spread of its bits on the GPU (the CPU side: tests/test_geometry_domain.py), on
synth_es.GEOMETRY_CASES and GEOMETRY_B_CASES: one macroblock and a 1x1 display, 256 one-macroblock rows, a row of 256
macroblocks, 4095x4095, 250 rows behind one slice of code 0xAF, an odd macroblock width with cropped edges,
letterboxed pictures and a fade to black; B-picture twins of the column, the row and the single macroblock.

  * the reference ABI and BatchDecoder.decode() against the oracle (and the compiled reference's recorded decodes where
    it decodes the case), with the slice walk off and on, B pictures off and on, in every stage-2 variant: planes, bit
    indices, RGBA at the display size, the residual and the accumulated map against the models -- at every size, the
    4095x4095 one included (its models take seconds, not minutes);
  * the lane walk's storing pass (pass D) on the device: jsmpeg_b200_debug_parse_picture on the letterboxed I pictures
    keeps the lane walk without a fix-up, with the oracle's records and coefficients; decode() of those streams walks
    every picture with the lane walk and gives the oracle's planes;
  * decode_pictures, decode_intra, seek_pictures of every listed picture; decode_macroblocks, decode_coefficients,
    decode_residuals and decode_accumulated against the models; decode_frames in its into and display forms;
  * one batch of every case at once: launches mixing mb_width 1 with 256, tiny tasks with the 4095x4095 one;
  * the decode tests once more with the serial walk, in a child process.
"""
import ctypes
import os

import numpy as np
import pytest

import accumulate_model
import chain_model
import display_model
import helpers
import macroblock_model
from jsmpeg_b200 import capi, decoder
from jsmpeg_b200.batch import OUT_ACCUMULATED, OUT_DEVICE, OUT_HOST, OUT_RESIDUALS, OUT_RGBA, BatchDecoder
from test_geometry_domain import B_CASES, CASES, IP_CASES, LETTERBOX, REFERENCE_CASES, display_size, oracle_run, packets
from test_gpu_motion_domain import _sequential_planes, oracle_maps, oracle_steps
from test_gpu_parity import _canvas2d_rgba
from test_motion_domain import stream

pytestmark = pytest.mark.gpu

SERIAL = os.environ.get("JSMPEG_B200_WALK") == "serial"


@pytest.mark.parametrize("name", CASES)
def test_reference_abi_decode_equals_the_oracle(name):
    want, want_idx, od = helpers.decode_all(helpers.oracle_lib(), packets(name))
    got, got_idx, gd = helpers.decode_all(capi.product_library(), packets(name))
    assert got_idx == want_idx
    helpers.assert_frames_equal(got, want, f"{name}: CUDA vs oracle")
    if name in REFERENCE_CASES:
        helpers.assert_frames_match_reference(got, got_idx, packets(name), f"{name}: CUDA vs compiled reference")
    od.destroy()
    gd.destroy()


# (slice_walk, flags): the plain, RGBA, residual and RGBA + residual variants of stage 2 (with the accumulate kernel)
PASSES = [(0, OUT_DEVICE), (1, OUT_HOST | OUT_RGBA), (0, OUT_RESIDUALS | OUT_ACCUMULATED), (1, OUT_RGBA | OUT_RESIDUALS)]


@pytest.mark.parametrize("name", CASES)
def test_batch_decode_equals_the_oracle_in_every_stage2_variant(name):
    width, height = display_size(stream(name))
    for decode_b in ((0, 1) if name in B_CASES else (0,)):
        want = oracle_steps(name, decode_b)
        maps = oracle_maps(name, decode_b)
        for slice_walk, flags in PASSES:
            what = (name, decode_b, slice_walk, flags)
            bd = BatchDecoder(1, slice_walk=slice_walk, decode_b=decode_b)
            bd.write(0, stream(name))
            res_now, map_now = None, None
            for k, (index, status, ptype, planes, res) in enumerate(want):
                assert bd.decode(1, flags) == 1, what + (k,)
                assert bd.get_index(0) == index, what + (k,)
                got = np.concatenate(bd.read_planes(0))
                if not np.array_equal(got, planes):
                    bad = np.nonzero(got != planes)[0]
                    raise AssertionError(f"{what} picture {k} (type {ptype}): {len(bad)} samples differ, first at {bad[:8]}")
                if flags & OUT_HOST:
                    assert np.array_equal(np.concatenate([p.copy() for p in bd.host_planes(0)]), planes), what + (k,)
                if status == 1:
                    res_now = res
                    if ptype in (1, 2):
                        map_now = maps[index]
                    if flags & OUT_RGBA:
                        ysz = len(planes) * 2 // 3
                        exp = _canvas2d_rgba(planes[:ysz], planes[ysz:ysz * 5 // 4], planes[ysz * 5 // 4:], width, height)
                        assert np.array_equal(bd.read_rgba(0), exp), what + (k, "rgba")
                if flags & OUT_RESIDUALS and res_now is not None:
                    assert np.array_equal(bd.read_residuals(0), res_now), what + (k, "residual")
                if flags & OUT_ACCUMULATED and map_now is not None:
                    assert np.array_equal(bd.read_accumulated(0), map_now), what + (k, "accumulated")
            assert bd.decode(1, flags) == 0
            assert bd.last_error() is None
            bd.close()


@pytest.mark.parametrize("name", LETTERBOX)
def test_letterboxed_pictures_take_pass_d_on_the_device(name):
    """The lane walk's storing pass on the device: every I picture keeps the lane walk (info.reserved[0] == 1) and no
    slice of it is finished from the staged records (reserved[2] == 0), with the oracle's headers and coefficients;
    then decode() takes every I/P picture with the lane walk and gives the oracle's planes"""
    if SERIAL:
        pytest.skip("the lane walk is off")
    es = stream(name)
    lib = capi.product_library()
    got, mbw, mbh = oracle_run(name)
    mb_size = mbw * mbh
    seq = helpers.oracle_lib()
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=seq)
    d.write(0.0, [es])
    sp = seq.oracle_seq_params(d.decoder).contents
    iq, nq = bytes(sp.intra_q), bytes(sp.non_intra_q)
    d.destroy()
    n_i = 0
    for _, pic, rec, coef, _ in got:
        if pic.picture_type != 1:
            continue
        info = helpers.PictureInfo()
        hdr = np.zeros(mb_size * 16, np.uint8)
        out = np.zeros(mb_size * 384, np.int16)
        assert lib.jsmpeg_b200_debug_parse_picture(es, len(es), pic.start_byte, mbw, mbh, iq, nq, ctypes.addressof(info),
                                                   hdr.ctypes.data, out.ctypes.data) == 0
        assert (info.status, info.picture_type, info.end_bit, info.error) == (1, 1, pic.end_bit, 0)
        assert (info.n_present, info.n_coded_blocks) == (pic.n_present, pic.n_coded_blocks)
        assert (info.reserved[0], info.reserved[2]) == (1, 0), (name, pic.start_byte, list(info.reserved))
        assert np.array_equal(hdr.reshape(mb_size, 16)[:, :8], rec.reshape(mb_size, 16)[:, :8]), (name, pic.start_byte)
        coded = np.zeros((mb_size, 6, 64), bool)
        h = rec.reshape(mb_size, 16)
        for blk in range(6):
            coded[:, blk, :] = ((h[:, 4] & 1) != 0)[:, None] & ((h[:, 5] & (0x20 >> blk)) != 0)[:, None]
        assert np.array_equal(out[coded.reshape(-1)], coef[coded.reshape(-1)]), (name, pic.start_byte)
        n_i += 1
    assert n_i == 2
    bd = BatchDecoder(1)
    bd.write(0, es)
    want = oracle_steps(name, 0)
    for index, status, ptype, planes, _ in want:
        assert bd.decode(1, OUT_DEVICE) == 1
        assert bd.get_index(0) == index
        assert np.array_equal(np.concatenate(bd.read_planes(0)), planes), (name, index)
    assert bd.stats()["lane_walk_pictures"] == sum(s[1] == 1 and s[2] in (1, 2) for s in want)
    assert bd.last_error() is None
    bd.close()


# ---- random access and the exports ------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", CASES)
def test_decode_pictures_intra_and_seek_equal_the_oracles_decode(name):
    decode_b = name in B_CASES
    want = _sequential_planes(name, decode_b)
    for slice_walk in (0, 1):
        bd = BatchDecoder(1, slice_walk=slice_walk, decode_b=decode_b)
        bd.write(0, stream(name))
        entries = bd.picture_index(0)
        assert [e["picture"] for e in entries] == [e["picture"] for e in chain_model.picture_index(stream(name), decode_b)]
        got = bd.decode_pictures([(0, e["picture"]) for e in entries])
        for e, t, i in zip(entries, got, bd.last_pictures_info):
            assert i["status"] == 1, (name, e["picture"], i)
            assert np.array_equal(t.cpu().numpy(), want[e["picture"]]), (name, slice_walk, e["picture"])
        intra = bd.intra_index(0)
        assert intra
        for e, t in zip(intra, bd.decode_intra([(0, e["picture"]) for e in intra])):
            assert np.array_equal(t.cpu().numpy(), want[e["picture"]]), (name, slice_walk, "intra", e["picture"])
        for e in entries[::-1] if slice_walk else entries:
            assert bd.seek_pictures([(0, e["picture"])], OUT_HOST) == 1
            assert bd.last_seek_info[0]["status"] == 1
            assert np.array_equal(np.concatenate(bd.read_planes(0)), want[e["picture"]]), (name, slice_walk, e["picture"])
        assert bd.last_error() is None
        bd.close()


@pytest.mark.parametrize("name", IP_CASES)
def test_picture_exports_equal_the_models(name):
    """decode_macroblocks, decode_coefficients, decode_residuals and decode_accumulated of every listed picture against
    macroblock_model and accumulate_model on the oracle's records"""
    got, mbw, mbh = oracle_run(name)
    pics = [(info, rec, coef) for _, info, rec, coef, _ in got if info.status == 1]
    bd = BatchDecoder(1)
    bd.write(0, stream(name))
    entries = bd.macroblock_index(0)
    assert len(entries) == len(pics)
    reqs = [(0, e["picture"]) for e in entries]
    mbs = bd.decode_macroblocks(reqs)
    coefs = bd.decode_coefficients(reqs)
    res = bd.decode_residuals(reqs)
    for k, (info, rec, coef) in enumerate(pics):
        assert np.array_equal(mbs[k].cpu().numpy().reshape(-1, 16), macroblock_model.export(rec, info.picture_type)), (name, k)
        want = macroblock_model.coefficients(rec, coef).reshape(mbh, mbw, 6, 64)
        assert np.array_equal(coefs[k].cpu().numpy().reshape(mbh, mbw, 6, 64), want), (name, k, "coefficients")
        assert np.array_equal(res[k].cpu().numpy(), macroblock_model.residuals(rec, coef, mbw, mbh)), (name, k, "residuals")
    index = chain_model.picture_index(stream(name))
    maps = bd.decode_accumulated([(0, e["picture"]) for e in index])
    for e, m, i in zip(index, maps, bd.last_accumulated_info):
        status, n_present, error, want = accumulate_model.oracle_chain(helpers.oracle_lib(), stream(name), e)
        assert (i["status"], i["n_present"], i["error"]) == (status, n_present, error) == (1, mbw * mbh, 0), (name, e)
        assert np.array_equal(m.cpu().numpy(), want), (name, e["picture"], "accumulated")
    assert bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("name", IP_CASES)
def test_decode_frames_into_equals_the_oracle_and_the_models(name):
    """decode_frames with every kind (jsmpeg_b200_batch_decode_frames_into), every picture of the stream in one call"""
    want = [s for s in oracle_steps(name, 0) if s[1] == 1]
    maps = oracle_maps(name, 0)
    pics = [p for p in oracle_run(name)[0] if p[1].status == 1]
    w, h = display_size(stream(name))
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


def test_decode_frames_display_of_every_case_in_one_batch():
    """decode_frames in presentation order (jsmpeg_b200_batch_decode_frames_display, B pictures on) of every case in one
    batch, two pictures per call, then flush_frames: each stream's frames are the oracle's pictures in the order
    tools/display_model.py presents them"""
    bd = BatchDecoder(len(CASES), decode_b=True)
    for s, name in enumerate(CASES):
        bd.write(s, stream(name))
    coded = [[(t, p) for _, st, t, p, _ in oracle_steps(name, name in B_CASES) if st == 1] for name in CASES]
    want = [[p for call in display_model.present(c, [2] * len(c), type_of=lambda f: f[0]) for _, p in call] for c in coded]
    got = [[] for _ in CASES]
    for _ in range(max(len(c) for c in coded) // 2 + 2):
        for s, o in enumerate(bd.decode_frames(2, OUT_DEVICE, display_order=True)):
            got[s] += [o["planes"][j].cpu().numpy().reshape(-1) for j in range(o["n_frames"])]
    for s, o in enumerate(bd.flush_frames()):
        got[s] += [o["planes"][j].cpu().numpy().reshape(-1) for j in range(o["n_frames"])]
    for s, name in enumerate(CASES):
        assert len(got[s]) == len(want[s]), (name, len(got[s]), len(want[s]))
        for k, (g, w) in enumerate(zip(got[s], want[s])):
            assert np.array_equal(g, w), (name, k)
    assert bd.last_error() is None
    bd.close()


def test_one_batch_decode_of_every_geometry_case():
    """All the cases in one batch (B pictures on): every walk, expand and reconstruct launch mixes mb_width 1 with 256,
    one-macroblock tasks with the 4095x4095 one, compact with dense records; plain and RGBA + residual variant"""
    for flags in (OUT_DEVICE, OUT_RGBA | OUT_RESIDUALS):
        bd = BatchDecoder(len(CASES), decode_b=True)
        for s, name in enumerate(CASES):
            bd.write(s, stream(name))
        want = [oracle_steps(name, name in B_CASES) for name in CASES]
        done = [0] * len(CASES)
        while True:
            before = [bd.get_index(s) for s in range(len(CASES))]
            if not bd.decode(1, flags):
                break
            for s in range(len(CASES)):
                if bd.get_index(s) == before[s] or done[s] == len(want[s]):
                    continue  # (a stream past its last picture may still move its index onto the end code)
                index, status, _, planes, res = want[s][done[s]]
                assert bd.get_index(s) == index, (CASES[s], done[s])
                assert np.array_equal(np.concatenate(bd.read_planes(s)), planes), (CASES[s], done[s], flags)
                if flags & OUT_RGBA and status == 1:
                    w, h = display_size(stream(CASES[s]))
                    ysz = len(planes) * 2 // 3
                    exp = _canvas2d_rgba(planes[:ysz], planes[ysz:ysz * 5 // 4], planes[ysz * 5 // 4:], w, h)
                    assert np.array_equal(bd.read_rgba(s), exp), (CASES[s], done[s], "rgba")
                    assert np.array_equal(bd.read_residuals(s), res), (CASES[s], done[s], "residual")
                done[s] += 1
        assert done == [len(w) for w in want]
        assert bd.last_error() is None
        bd.close()


def test_decode_tests_with_the_serial_walk_in_a_child_process():
    """The walk variant is chosen once per process: the decode tests again with JSMPEG_B200_WALK=serial"""
    import subprocess
    import sys
    if SERIAL:
        pytest.skip("already running with the serial walk")
    env = dict(os.environ, JSMPEG_B200_WALK="serial")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-x", "-q", "-p",
                        "no:cacheprovider", "-k", "decode and not serial"], env=env, capture_output=True, text=True,
                       timeout=3000)
    assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
