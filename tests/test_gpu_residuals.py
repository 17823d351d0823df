"""Residuals on the device (jsmpeg_b200_batch_decode_residuals) against the serial model (macroblock_model.residuals)
applied to the oracle's fresh decode, bit for bit: every listed picture of the key-picture corpus and of I/P/B streams,
with the slice walk and decode_b on and off and the macroblock entries alongside, and against the transform of the
device's own decode_coefficients; a round trip to decode_pictures' planes through the oracle's prediction; an .mpg;
mixed sizes with duplicates, slot pressure, damaged streams, the decode() state the call must leave alone, invalid
requests, launch counts, and the bench's shape."""
import ctypes
import functools
import json
import os
import random
import re
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

import helpers
import macroblock_model
import synth_es
from jsmpeg_b200.batch import OUT_HOST, BatchDecoder
from test_coefficient_export import oracle_fresh_coefficients
from test_gpu_coefficients import _oracle_from, expected as expected_coefficients, records_from_entries
from test_gpu_intra import CORPUS, _assert_same_state, _damage, _state, ffmpeg_es, host
from test_gpu_macroblocks import B_CORPUS, MIXED, geometry, index_tuples, stream
from test_residual_export import planes_struct, sample_mask

pytestmark = pytest.mark.gpu


def es_geometry(es):
    """(mb_width, mb_height) of the first sequence header of `es`"""
    i = es.find(b"\x00\x00\x01\xb3")
    w = (es[i + 4] << 4) | (es[i + 5] >> 4)
    h = ((es[i + 5] & 15) << 8) | es[i + 6]
    return (w + 15) >> 4, (h + 15) >> 4


@functools.lru_cache(maxsize=None)
def expected(name, picture):
    """(n_present, error, int16 [coded_size * 3 // 2]) of listed picture `picture` of corpus stream `name`: the model
    applied to the oracle fed the picture's fresh bytes."""
    n_present, error, coef = expected_coefficients(name, picture)
    return n_present, error, macroblock_model.residual_planes(coef, *es_geometry(stream(name)))


@pytest.mark.parametrize("name", CORPUS + B_CORPUS)
def test_every_listed_picture_equals_the_oracle_with_every_option(name):
    """All listed pictures in one call, with the slice walk and decode_b each off and on: the model's residual of the
    oracle's fresh decode, and the transform of what decode_coefficients gives for the same requests; with the
    macroblock entries asked for, those of decode_macroblocks, and the infos are decode_macroblocks' infos."""
    import torch
    es = stream(name)
    entries = macroblock_model.macroblock_index(es)
    assert entries
    mbw, mbh = es_geometry(es)
    reqs = [(0, e["picture"]) for e in entries]
    for slice_walk, decode_b in ((0, 0), (1, 0), (0, 1), (1, 1)):
        bd = BatchDecoder(1, slice_walk=slice_walk, decode_b=decode_b)
        bd.write(0, es)
        with_mb = slice_walk == decode_b
        got = bd.decode_residuals(reqs, macroblocks=with_mb)
        info = bd.last_residuals_info
        mbs = bd.decode_macroblocks(reqs)
        assert info == bd.last_macroblocks_info
        coefs = bd.decode_coefficients(reqs)
        for k, (e, i) in enumerate(zip(entries, info)):
            r = got[k][0] if with_mb else got[k]
            n_present, error, want = expected(name, e["picture"])
            assert tuple(r.shape) == (mbw * mbh * 384,) and r.dtype == torch.int16 and r.is_cuda
            assert (i["n_present"], i["error"]) == (n_present, error), (name, e["picture"], slice_walk, decode_b)
            assert np.array_equal(host(r), want), (name, e["picture"], slice_walk, decode_b)
            assert np.array_equal(host(r), macroblock_model.residual_planes(host(coefs[k]), mbw, mbh))
            if with_mb:
                assert np.array_equal(host(got[k][1]), host(mbs[k])), (name, e["picture"], slice_walk, decode_b)
        assert bd.last_error() is None
        bd.close()


def test_program_stream_through_write_ps():
    import gen_streams
    data = gen_streams.make_clip_ps(320, 240, 24, form="mpg")
    m1v = gen_streams.make_clip_m1v(320, 240, 24)
    bd = BatchDecoder(1)
    bd.write_ps(0, data)
    model = macroblock_model.macroblock_index(m1v)
    assert index_tuples(bd.macroblock_index(0)) == index_tuples(model) and len(model) >= 20
    got = bd.decode_residuals([(0, e["picture"]) for e in model])
    for e, t in zip(model, got):
        want = macroblock_model.residual_planes(oracle_fresh_coefficients(m1v, e)[2], 20, 15)
        assert np.array_equal(host(t), want), e["picture"]
    bd.close()


def records_with_motion(entries):
    """mb_record_t [n, 16] of public entries, as records_from_entries, with the B picture's motion bits and backward
    vector too"""
    e = np.frombuffer(np.ascontiguousarray(entries).tobytes(), macroblock_model.ENTRY)
    r = np.frombuffer(records_from_entries(entries).tobytes(), macroblock_model.RECORD).copy()
    r["flags"] |= (np.where(e["flags"] & macroblock_model.MB_FORWARD, macroblock_model.MBF_MOTION_FWD, 0) |
                   np.where(e["flags"] & macroblock_model.MB_BACKWARD, macroblock_model.MBF_MOTION_BWD, 0)).astype(np.uint8)
    r["bwd_x"], r["bwd_y"] = e["bwd_x"], e["bwd_y"]
    return r.view(np.uint8).reshape(len(e), 16)


@pytest.mark.parametrize("name", ["ffmpeg_320x240", "mini_enc_fcodes_2_4_fullpel_bwd"])
def test_prediction_and_residual_give_the_pictures(name):
    """Every I, P and B picture listed by both indexes: the oracle's prediction from the references decode_pictures
    returns (the newest I/P picture before it for P, the two newest for B), made from the exported entries with every
    cbp bit cleared, plus the exported residual and clamped, gives decode_pictures' samples of every present non-intra
    macroblock; the clamped residual gives those of every intra macroblock."""
    es = stream(name)
    lib = helpers.oracle_lib()
    from test_residual_export import Planes
    for fn, args in (("oracle_reconstruct", [ctypes.POINTER(Planes)] * 2),
                     ("oracle_reconstruct_b", [ctypes.POINTER(Planes)] * 3)):
        getattr(lib, fn).restype = None
        getattr(lib, fn).argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, *args]
    from jsmpeg_b200 import decoder
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=lib)
    d.write(0.0, [es])
    seq = ctypes.cast(lib.oracle_seq_params(d.decoder), ctypes.c_void_p)
    bd = BatchDecoder(1, decode_b=True)
    bd.write(0, es)
    mbh, mbw = geometry(bd, 0)
    cw, ch = mbw * 16, mbh * 16
    cs = cw * ch
    in_picture_index = {e["picture"] for e in bd.picture_index(0)}
    listed = [e for e in bd.macroblock_index(0) if e["picture"] in in_picture_index]
    reqs = [(0, e["picture"]) for e in listed]
    exported = bd.decode_residuals(reqs, macroblocks=True)
    pictures = [host(t)[:cs * 3 // 2] for t in bd.decode_pictures(reqs)]
    refs = []  # the I/P pictures so far, in coded order
    kinds = Counter()
    for e, (res, entries), want in zip(listed, exported, pictures):
        ent = host(entries).reshape(-1, 16)
        res = host(res).astype(np.int32)
        flags = np.frombuffer(ent.tobytes(), macroblock_model.ENTRY)["flags"]
        present = (flags & macroblock_model.MB_PRESENT) != 0
        intra = present & ((flags & macroblock_model.MB_INTRA) != 0)
        pred = np.zeros(cs * 3 // 2, np.uint8)
        if e["type"] == 2 or (e["type"] == 3 and len(refs) >= 2):
            hdr = records_with_motion(ent)
            hdr[:, 5] = 0  # no block is added: the prediction alone
            zero = np.zeros(mbw * mbh * 384, np.int16)
            fwd = refs[-1] if e["type"] == 2 else refs[-2]
            f, o = planes_struct(fwd, cs), planes_struct(pred, cs)
            if e["type"] == 2:
                lib.oracle_reconstruct(seq, cw, ch, hdr.ctypes.data, zero.ctypes.data, ctypes.byref(f), ctypes.byref(o))
            else:
                bk = planes_struct(refs[-1], cs)
                lib.oracle_reconstruct_b(seq, cw, ch, hdr.ctypes.data, zero.ctypes.data, ctypes.byref(f), ctypes.byref(bk),
                                         ctypes.byref(o))
        elif e["type"] != 1:
            continue
        pm, im = sample_mask(present & ~intra, mbw, mbh), sample_mask(intra, mbw, mbh)
        if e["type"] == 1:
            assert im.all()
        got = np.clip(np.where(im, 0, pred.astype(np.int32)) + res, 0, 255)
        assert np.array_equal(got[pm | im], want[pm | im]), (name, e["picture"], e["type"])
        kinds[e["type"]] += 1
        if e["type"] in (1, 2):
            refs.append(want.copy())
    assert kinds[1] >= 1 and kinds[2] >= 3 and (kinds[3] >= 3 or name.startswith("ffmpeg")), kinds
    d.destroy()
    bd.close()


def test_mixed_sizes_shuffled_with_duplicates():
    bd = BatchDecoder(len(MIXED))
    for s, name in enumerate(MIXED):
        bd.write(s, stream(name))
    rng = random.Random(7)
    reqs = []
    for s in range(len(MIXED)):
        pics = [e["picture"] for e in bd.macroblock_index(s)]
        reqs += [(s, k) for k in rng.sample(pics, min(len(pics), 6))]
    reqs += [reqs[2], reqs[9], reqs[9]]  # the same picture two and three times
    rng.shuffle(reqs)
    got = bd.decode_residuals(reqs)
    for (s, k), t, i in zip(reqs, got, bd.last_residuals_info):
        n_present, error, want = expected(MIXED[s], k)
        mbh, mbw = geometry(bd, s)
        assert tuple(t.shape) == (mbh * mbw * 384,)
        assert (i["n_present"], i["error"]) == (n_present, error) and np.array_equal(host(t), want), (MIXED[s], k)
    bd.close()


def test_slot_pressure_gives_the_same_bytes():
    """Three record slots for tens of requests (with duplicates): many waves, the look-ahead flushed."""
    names = ["ffmpeg_320x240", "rows_ip", "b_rows", "mini_enc_open_gop"]
    outs = []
    for max_slots in (0, 3):
        bd = BatchDecoder(len(names), max_slots=max_slots)
        for s, name in enumerate(names):
            bd.write(s, stream(name))
        reqs = [(s, e["picture"]) for s in range(len(names)) for e in bd.macroblock_index(s)]
        reqs += reqs[::5]
        bd.decode(2)  # the look-ahead holds slots too
        got = bd.decode_residuals(reqs, macroblocks=True)
        outs.append(([(host(r), host(m)) for r, m in got], bd.last_residuals_info))
        bd.close()
    assert len(outs[0][0]) == len(outs[1][0]) >= 50
    assert outs[0][1] == outs[1][1]
    for (a, ma), (b, mb) in zip(outs[0][0], outs[1][0]):
        assert np.array_equal(a, b) and np.array_equal(ma, mb)


def test_damaged_streams_follow_the_stated_rule():
    """Bit flips in every third picture of an I/P stream and in the pictures of a B stream, three seeds: the device
    equals the model of the oracle fed everything from the picture on (decode_coefficients' rule: the block with the
    bad code, and those after it, are 0), error presence and entries included."""
    clean = ffmpeg_es(320, 240, 24) + synth_es.make_case("i_only_320x240")[-4:]  # end code: the last picture closes
    b_clean = synth_es.make_case("b_one_slice_fcodes")
    streams = []
    for seed in (1, 2, 3):
        streams += [_damage(clean, macroblock_model.macroblock_index(clean)[::3], seed),
                    _damage(b_clean, macroblock_model.macroblock_index(b_clean)[1::2], seed, flips=3)]
    bd = BatchDecoder(len(streams))
    errors = 0
    for s, es in enumerate(streams):
        bd.write(s, es)
        entries = macroblock_model.macroblock_index(es)
        got = bd.decode_residuals([(s, e["picture"]) for e in entries], macroblocks=True)
        for e, (r, m), i in zip(entries, got, bd.last_residuals_info):
            info, rec, raw = _oracle_from(es, e)
            want = macroblock_model.residuals(rec, raw, *es_geometry(es))
            assert bool(i["error"]) == bool(info.error), (s, e["picture"])
            assert np.array_equal(host(r), want), (s, e["picture"])
            assert np.array_equal(host(m).reshape(-1, 16), macroblock_model.export(rec, e["type"])), (s, e["picture"])
            errors += bool(i["error"])
    assert errors and bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("name,decode_b", [("ffmpeg_320x240", False), ("b_rows", True)])
def test_decode_state_is_untouched(name, decode_b):
    """decode_residuals in the middle of a decode() run: the state is as before the call, and every picture of the
    run equals that of a twin batch that never called it."""
    es = stream(name)
    runs = []
    for interleave in (False, True):
        bd = BatchDecoder(2, decode_b=decode_b)
        bd.write(0, es)
        bd.write(1, synth_es.make_case("rows_ip"))
        frames = []
        while bd.decode(1, OUT_HOST):
            frames.append(np.concatenate(bd.read_planes(0)))
            if interleave and len(frames) == 5:
                before = _state(bd, 0)
                bd.decode_residuals([(s, e["picture"]) for s in (0, 1) for e in bd.macroblock_index(s)], macroblocks=True)
                _assert_same_state(before, _state(bd, 0))
        runs.append(frames)
        bd.close()
    assert len(runs[0]) == len(runs[1])
    for a, b in zip(*runs):
        assert np.array_equal(a, b)


def test_invalid_requests_are_refused_and_change_nothing():
    import intra_model
    es = synth_es.make_case("b_rows")  # I B B P B B I B B P B B I
    model = macroblock_model.macroblock_index(es)
    cut = es[:model[-1]["close"] + 2]  # the last I picture is not closed yet
    ignored = synth_es.make_case("ignored_pictures_userdata")  # picture 2: P with forward_f_code 0; 6: D
    bd = BatchDecoder(3)
    bd.write(0, cut)
    bd.write(1, es[intra_model.first_sequence_header(es)[0] + 4:])  # no sequence header
    bd.write(2, ignored)
    assert bd.decode(1, OUT_HOST)
    before = _state(bd, 0)
    first, entries = bd.decode_residuals([(0, 1)], macroblocks=True)[0]  # a B picture, decode_b off
    mark, mark_mb = first.clone().fill_(7), entries.clone().fill_(7)

    def call(reqs, dsts, mb_dsts=None):
        n = len(reqs)
        return bd.lib.jsmpeg_b200_batch_decode_residuals(
            bd.handle, n, (ctypes.c_int * n)(*[s for s, _ in reqs]), (ctypes.c_uint32 * n)(*[p for _, p in reqs]),
            (ctypes.c_void_p * n)(*dsts), None if mb_dsts is None else (ctypes.c_void_p * n)(*mb_dsts), None, None)

    # with a valid request in front: the unclosed tail, no sequence header, no stream, no picture, f_code 0, D
    for stream_, pic in ((0, model[-1]["picture"]), (1, 0), (3, 0), (-1, 0), (0, 99), (2, 2), (2, 6)):
        assert call([(0, 4), (stream_, pic)], [mark.data_ptr(), first.data_ptr()]) == -2, (stream_, pic)
        with pytest.raises(ValueError):
            bd.decode_residuals([(0, 4), (stream_, pic)])
    assert call([(0, 4)], [None]) == -2                                  # NULL destination
    assert call([(0, 4)], [mark.data_ptr() + 8]) == -2                   # misaligned destination
    assert call([(0, 4)], [mark.data_ptr()], [mark_mb.data_ptr() + 4]) == -2  # misaligned macroblock destination
    assert call([(0, 4)], [mark.data_ptr()], [None]) == -2               # NULL macroblock destination in a given array
    assert bool((mark == 7).all()) and bool((mark_mb == 7).all())
    _assert_same_state(before, _state(bd, 0))
    assert bd.last_error() is None
    # mb_dst = NULL: the residual alone, and the same bytes
    assert call([(0, 1)], [mark.data_ptr()]) == 1
    assert np.array_equal(host(mark), host(first)) and np.array_equal(host(first), expected("b_rows", 1)[2])
    assert np.array_equal(host(entries), host(bd.decode_macroblocks([(0, 1)])[0]))
    assert call([], []) == 0
    bd.close()


def launch_counts():
    """({kernel: launches} of decode_residuals without and with the entries, the decoder's launch counters) on
    test_gpu_launch_counts' workload, counted by torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from test_gpu_launch_counts import FIXTURE_720P, N_720P, N_SMALL
    small = b"".join(p for _, p in helpers.clip_packets(320, 240, 12))
    big = open(FIXTURE_720P, "rb").read()
    bd = BatchDecoder(N_SMALL + N_720P, max_slots=1200, decode_b=1, slice_walk=1)
    for s in range(N_SMALL):
        bd.write(s, small)
    for s in range(N_720P):
        bd.write(N_SMALL + s, big)
    reqs = [(s, e["picture"]) for s in range(N_SMALL + N_720P) for e in bd.macroblock_index(s)]
    assert len(reqs) < 1200
    bd.reset_stats()
    seen = []
    for macroblocks in (False, True):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            bd.decode_residuals(reqs, macroblocks=macroblocks)
            torch.cuda.synchronize()
        kernels = Counter()
        for ev in prof.events():
            m = re.search(r"(\w+_kernel)\(", ev.name)
            if ev.device_type == torch.autograd.DeviceType.CUDA and m:
                kernels[m.group(1)] += 1
        seen.append(dict(kernels))
    st = bd.stats()
    bd.close()
    return seen, [st["kernel_launches"], st["recon_launches"]]


def test_launch_counts():
    """On test_gpu_launch_counts' workload (one wave): the three walks, expand in the lane walk's 8 size groups and
    beside the other two walks, one export_residuals_kernel, and export_macroblocks_kernel only when the entries are
    asked for; no coefficient export.  The decoder's launch counters are decode()'s and stay as they were.  (Counted in
    a process of its own.)"""
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "launch-counts"], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    seen, counters = json.loads(r.stdout.strip().splitlines()[-1])
    walks = {"walk_pictures_lanes_kernel": 8, "walk_pictures_slices_kernel": 1, "walk_pictures_b_kernel": 1,
             "expand_blocks_kernel": 10, "export_residuals_kernel": 1}
    assert seen == [walks, {**walks, "export_macroblocks_kernel": 1}]
    assert counters == [0, 0]


def test_the_bench_shape():
    """16 pictures from each of the bench's 64 distinct 1080p clips in one call; one picture of every fourth clip
    equals the model of the oracle, and every residual equals the transform of decode_coefficients' output."""
    sys.path.insert(0, helpers.ROOT)
    import bench
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips))
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    rng = random.Random(13)
    reqs = [(s, k) for s in range(len(clips)) for k in sorted(rng.sample([e["picture"] for e in bd.macroblock_index(s)], 16))]
    got = bd.decode_residuals(reqs)
    assert bd.last_error() is None and len(got) == 1024
    for j in range(0, len(reqs), 64):  # the first picture of every fourth clip
        s, k = reqs[j]
        index = {e["picture"]: e for e in macroblock_model.macroblock_index(clips[s])}
        assert tuple(got[j].shape) == (68 * 120 * 384,)
        want = macroblock_model.residual_planes(oracle_fresh_coefficients(clips[s], index[k])[2], 120, 68)
        assert np.array_equal(host(got[j]), want), (s, k)
    for j in range(0, len(reqs), 97):
        coef = bd.decode_coefficients([reqs[j]])[0]
        assert np.array_equal(host(got[j]), macroblock_model.residual_planes(host(coef), 120, 68)), reqs[j]
    bd.close()


if __name__ == "__main__" and sys.argv[1:] == ["launch-counts"]:
    print(json.dumps(launch_counts()))
