"""Stage 2 on the GPU over the whole motion-vector domain (the CPU side: tests/test_motion_domain.py).

  * the reconstruct kernel on random records (jsmpeg_b200_debug_reconstruct) against tools/recon_model.py: every flag
    and cbp, compact and dense records, vectors up to the int16 extremes, warps mixing the fast path with the per-tap
    one and half-sample lanes with full-sample ones;
  * decode() on synth_es.VECTOR_CASES ("wide" up to 1920x1080 with f_code 5-7, "wrap", "outside", "mixed"; I/P and
    I/P/B) through the reference ABI and BatchDecoder, with the slice walk off and on, B pictures off and on, and the
    stage-2 variants the output flags choose (plain, RGBA, residual, both): planes and bit indices against the oracle,
    RGBA against the canvas2d formula, the residual against the model's transform of the oracle's coefficients, the
    accumulated map against tools/accumulate_model.py; one batch of all of them at once;
  * decode_pictures and seek_pictures of every listed picture against the oracle's decode();
  * the decode tests once more with the serial walk, in a child process.
"""
import ctypes
import functools
import os

import numpy as np
import pytest

import accumulate_model
import chain_model
import helpers
import macroblock_model
import recon_model
import synth_es
from jsmpeg_b200 import capi, decoder
from jsmpeg_b200.batch import OUT_ACCUMULATED, OUT_DEVICE, OUT_HOST, OUT_RESIDUALS, OUT_RGBA, BatchDecoder
from test_gpu_parity import _canvas2d_rgba
from test_motion_domain import B_CASES, RECORD_SHAPES, REFERENCE_CASES, random_picture, stream

pytestmark = pytest.mark.gpu

CASES = sorted(synth_es.VECTOR_CASES)


# ---- stage 2 on random records -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("mb_width,mb_height", RECORD_SHAPES)
def test_reconstruct_kernel_on_random_records_equals_the_model(mb_width, mb_height):
    lib = capi.product_library()
    ysz = mb_width * mb_height * 256
    for seed in range(3):
        rec, coef, fwd, cur = random_picture(100 + seed, mb_width, mb_height)
        want = recon_model.reconstruct(rec, coef, fwd, cur, mb_width, mb_height)
        f = [np.ascontiguousarray(p) for p in (fwd[:ysz], fwd[ysz:ysz * 5 // 4], fwd[ysz * 5 // 4:])]
        c = [np.ascontiguousarray(p) for p in (cur[:ysz], cur[ysz:ysz * 5 // 4], cur[ysz * 5 // 4:])]
        assert lib.jsmpeg_b200_debug_reconstruct(mb_width, mb_height, rec.ctypes.data, coef.ctypes.data,
                                                 *[p.ctypes.data for p in f], *[p.ctypes.data for p in c]) == 0
        got = np.concatenate(c)
        bad = np.nonzero(got != want)[0]
        assert not len(bad), f"{mb_width}x{mb_height} seed {seed}: {len(bad)} samples differ, first at {bad[:8]}: " \
                             f"kernel {got[bad[:8]]} model {want[bad[:8]]}"


# ---- decode() on the generated streams -----------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def oracle_steps(name, decode_b):
    """Per decode() of the oracle: (bit index after, status, picture type, Y | Cr | Cb, model residual or None)"""
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(int(decode_b))
    try:
        d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=lib)
        d.write(0.0, [stream(name)])
        seq = lib.oracle_seq_params(d.decoder).contents
        mb, mbw = seq.mb_size, seq.mb_width
        out = []
        while d.decode():
            info = lib.oracle_last_picture_info(d.decoder).contents
            planes = np.concatenate([np.ravel(p).copy() for p in d.planes()])
            res = None
            if info.status == 1:
                rec = np.ctypeslib.as_array(ctypes.cast(lib.oracle_last_mb_records(d.decoder),
                                                        ctypes.POINTER(ctypes.c_uint8)), shape=(mb * 16,)).copy()
                coef = np.ctypeslib.as_array(ctypes.cast(lib.oracle_last_coefficients(d.decoder),
                                                         ctypes.POINTER(ctypes.c_int16)), shape=(mb * 384,)).copy()
                res = macroblock_model.residuals(rec, coef, mbw, mb // mbw)
            out.append((d.bufferGetIndex(), info.status, info.picture_type, planes, res))
        d.destroy()
    finally:
        lib.oracle_set_decode_b(0)
    return out


@functools.lru_cache(maxsize=None)
def oracle_maps(name, decode_b):
    """{bit index after the decode(): accumulated map} of every I/P picture the oracle reconstructs"""
    maps = accumulate_model.sequential(helpers.oracle_lib(), stream(name), decode_b)
    steps = [s for s in oracle_steps(name, decode_b) if s[1] == 1 and s[2] in (1, 2)]
    assert len(steps) == len(maps)
    return {s[0]: m for s, (_, _, m) in zip(steps, maps)}


@pytest.mark.parametrize("name", CASES)
def test_reference_abi_decode_equals_the_oracle(name):
    packets = [(0.0, stream(name))]
    want, want_idx, od = helpers.decode_all(helpers.oracle_lib(), packets)
    got, got_idx, gd = helpers.decode_all(capi.product_library(), packets)
    assert got_idx == want_idx
    helpers.assert_frames_equal(got, want, f"{name}: CUDA vs oracle")
    if name in REFERENCE_CASES:
        helpers.assert_frames_match_reference(got, got_idx, packets, f"{name}: CUDA vs compiled reference")
    od.destroy()
    gd.destroy()


# (slice_walk, flags): the plain, RGBA, residual and RGBA + residual variants of stage 2 (with the accumulate kernel)
PASSES = [(0, OUT_DEVICE), (1, OUT_HOST | OUT_RGBA), (0, OUT_RESIDUALS | OUT_ACCUMULATED), (1, OUT_RGBA | OUT_RESIDUALS)]


@pytest.mark.parametrize("name", CASES)
def test_batch_decode_equals_the_oracle_in_every_stage2_variant(name):
    info_w = synth_es.VECTOR_CASES[name]["knobs"]
    width, height = info_w["width"], info_w["height"]
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


def test_one_batch_decode_of_every_domain_and_size():
    """All the streams in one batch (B pictures on): every reconstruct launch mixes pictures of every domain and size,
    tasks on the fast path and tasks on the per-tap one, plain and RGBA variant"""
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
                index, _, _, planes, _ = want[s][done[s]]
                assert bd.get_index(s) == index, (CASES[s], done[s])
                assert np.array_equal(np.concatenate(bd.read_planes(s)), planes), (CASES[s], done[s], flags)
                done[s] += 1
        assert done == [len(w) for w in want]
        assert bd.last_error() is None
        bd.close()


# ---- random access --------------------------------------------------------------------------------------------------------

def _sequential_planes(name, decode_b):
    """{picture number: Y | Cr | Cb after the oracle's decode() consumed it}"""
    positions = chain_model.picture_positions(stream(name))
    out = {}
    starts = [0] + [idx for idx, *_ in oracle_steps(name, decode_b)]
    for k, (index, _, _, planes, _) in enumerate(oracle_steps(name, decode_b)):
        at = (starts[k] + 7) >> 3
        out[next(i for i, p in enumerate(positions) if p >= at)] = planes
    return out


@pytest.mark.parametrize("name", CASES)
def test_decode_pictures_and_seek_pictures_equal_the_oracles_decode(name):
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
        for e in entries[::-1] if slice_walk else entries:
            assert bd.seek_pictures([(0, e["picture"])], OUT_HOST) == 1
            assert bd.last_seek_info[0]["status"] == 1
            assert np.array_equal(np.concatenate(bd.read_planes(0)), want[e["picture"]]), (name, slice_walk, e["picture"])
        assert bd.last_error() is None
        bd.close()


def test_decode_tests_with_the_serial_walk_in_a_child_process():
    """The walk variant is chosen once per process: the decode tests again with JSMPEG_B200_WALK=serial"""
    import subprocess
    import sys
    if os.environ.get("JSMPEG_B200_WALK") == "serial":
        pytest.skip("already running with the serial walk")
    env = dict(os.environ, JSMPEG_B200_WALK="serial")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-x", "-q", "-p",
                        "no:cacheprovider", "-k", "decode and not serial"], env=env, capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
