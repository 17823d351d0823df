"""Coefficients on the device (jsmpeg_b200_batch_decode_coefficients) against the serial model
(macroblock_model.coefficients) applied to the oracle's fresh decode, bit for bit: every listed picture of the
key-picture corpus, of I/P/B streams and of an .mpg, with the slice walk and decode_b on and off and the macroblock
entries alongside; a round trip through the oracle's reconstruction; mixed sizes with duplicates, slot pressure,
damaged streams, the decode() state the call must leave alone, invalid requests, launch counts, and the bench's shape."""
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
import intra_model
import macroblock_model
import synth_es
from jsmpeg_b200.batch import OUT_HOST, BatchDecoder
from test_coefficient_export import oracle_coefficients, oracle_fresh_coefficients
from test_gpu_intra import CORPUS, _assert_same_state, _damage, _state, ffmpeg_es, host
from test_gpu_macroblocks import B_CORPUS, MIXED, geometry, index_tuples, stream

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def expected(name, picture):
    """(n_present, error, int16 [mb_size, 6, 64]) of listed picture `picture` of corpus stream `name`: the model applied
    to the oracle fed the picture's fresh bytes."""
    es = stream(name)
    entry = next(e for e in macroblock_model.macroblock_index(es) if e["picture"] == picture)
    info, _, coef = oracle_fresh_coefficients(es, entry)
    return info.n_present, info.error, coef


def flat(t):
    return host(t).reshape(-1, 6, 64)


@pytest.mark.parametrize("name", CORPUS + B_CORPUS)
def test_every_listed_picture_equals_the_oracle_with_every_option(name):
    """All listed pictures in one call, with the slice walk and decode_b each off and on: the model's coefficients of
    the oracle's fresh decode; with the macroblock entries asked for, those of decode_macroblocks."""
    import torch
    es = stream(name)
    entries = macroblock_model.macroblock_index(es)
    assert entries
    reqs = [(0, e["picture"]) for e in entries]
    for slice_walk, decode_b in ((0, 0), (1, 0), (0, 1), (1, 1)):
        bd = BatchDecoder(1, slice_walk=slice_walk, decode_b=decode_b)
        bd.write(0, es)
        with_mb = slice_walk == decode_b
        got = bd.decode_coefficients(reqs, macroblocks=with_mb)
        info = bd.last_coefficients_info
        mbs = bd.decode_macroblocks(reqs) if with_mb else None
        assert info == bd.last_macroblocks_info or not with_mb
        for k, (e, i) in enumerate(zip(entries, info)):
            c = got[k][0] if with_mb else got[k]
            n_present, error, want = expected(name, e["picture"])
            assert tuple(c.shape) == (*geometry(bd, 0), 6, 8, 8) and c.dtype == torch.int16 and c.is_cuda
            assert (i["n_present"], i["error"]) == (n_present, error), (name, e["picture"], slice_walk, decode_b)
            assert np.array_equal(flat(c), want), (name, e["picture"], slice_walk, decode_b)
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
    got = bd.decode_coefficients([(0, e["picture"]) for e in model])
    for e, t in zip(model, got):
        assert np.array_equal(flat(t), oracle_fresh_coefficients(m1v, e)[2]), e["picture"]
    bd.close()


def records_from_entries(entries):
    """mb_record_t [n, 16] of public entries (uint8 [n, 16]) of an I or P picture: flags, the forward vector, cbp and
    qscale, dc_only = 0 (the full transform of a DC-only block equals the shortcut)"""
    e = np.frombuffer(np.ascontiguousarray(entries).tobytes(), macroblock_model.ENTRY)
    r = np.zeros(len(e), macroblock_model.RECORD)
    flags = e["flags"]
    r["flags"] = (np.where(flags & macroblock_model.MB_PRESENT, macroblock_model.MBF_PRESENT, 0) |
                  np.where(flags & macroblock_model.MB_INTRA, macroblock_model.MBF_INTRA, 0) |
                  np.where(flags & macroblock_model.MB_SKIPPED, macroblock_model.MBF_SKIPPED, 0))
    r["mv_h"], r["mv_v"] = e["fwd_x"], e["fwd_y"]
    r["cbp"], r["qscale"] = e["cbp"], e["qscale"]
    return r.view(np.uint8).reshape(len(e), 16)


class Planes(ctypes.Structure):  # the oracle's planes_t
    _fields_ = [("y", ctypes.c_void_p), ("cr", ctypes.c_void_p), ("cb", ctypes.c_void_p)]


def planes_struct(buf, n):
    """planes_t over a contiguous Y | Cr | Cb uint8 array of luma size n"""
    base = buf.ctypes.data
    return Planes(base, base + n, base + n + n // 4)


@pytest.mark.parametrize("name", ["ffmpeg_320x240", "mini_enc_fcodes_2_4_fullpel_bwd"])
def test_the_exports_together_with_the_intra_dc_over_8_reconstruct_the_pictures(name):
    """Every listed I and P picture: records built from the exported entries, with the exported coefficients, through
    the oracle's reconstruction (forward picture: zero for I, the previous reference's decode_pictures planes for P)
    give the decode_pictures planes of the picture.  The two exports hold everything the samples are made from: an intra
    DC is exported as 8 * dc (exact in these conforming streams) and goes back into the records as dc."""
    es = stream(name)
    lib = helpers.oracle_lib()
    lib.oracle_reconstruct.restype = None
    lib.oracle_reconstruct.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                       ctypes.POINTER(Planes), ctypes.POINTER(Planes)]
    from jsmpeg_b200 import decoder
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=lib)
    d.write(0.0, [es])
    seq = lib.oracle_seq_params(d.decoder)
    bd = BatchDecoder(1)
    bd.write(0, es)
    info = bd.stream_info(0)
    cw, ch = (info["width"] + 15) // 16 * 16, (info["height"] + 15) // 16 * 16
    listed = [e for e in bd.macroblock_index(0) if e["type"] in (1, 2)]
    in_picture_index = {e["picture"] for e in bd.picture_index(0)}
    assert all(e["picture"] in in_picture_index for e in listed)
    reqs = [(0, e["picture"]) for e in listed]
    exported = bd.decode_coefficients(reqs, macroblocks=True)
    pictures = [host(t) for t in bd.decode_pictures(reqs)]
    fwd = np.zeros(cw * ch * 3 // 2, np.uint8)
    checked = 0
    for e, (coef, entries), want in zip(listed, exported, pictures):
        if e["type"] == 1:
            fwd[:] = 0
        hdr = records_from_entries(host(entries).reshape(-1, 16))
        c = host(coef).reshape(-1, 6, 64).astype(np.int16)
        # the export reports an intra DC as 8 * dc, the records hold dc itself (jsmpeg_b200/csrc/records.h); these
        # conforming streams keep |dc| <= 4095, where 8 * dc is exact
        intra = (hdr.view(np.uint8).reshape(-1, 16)[:, 4] & 0x02) != 0
        assert (c[intra, :, 0] % 8 == 0).all()
        c[intra, :, 0] //= 8
        c = np.ascontiguousarray(c.reshape(-1))
        cur = np.zeros_like(fwd)
        f, o = planes_struct(fwd, cw * ch), planes_struct(cur, cw * ch)
        lib.oracle_reconstruct(ctypes.cast(seq, ctypes.c_void_p), cw, ch, hdr.ctypes.data, c.ctypes.data,
                               ctypes.byref(f), ctypes.byref(o))
        assert np.array_equal(cur, want[:cw * ch * 3 // 2]), (name, e["picture"])
        fwd = want[:cw * ch * 3 // 2].copy()  # the next P picture predicts from this reference
        checked += 1
    assert checked == len(listed) >= 4 and any(e["type"] == 2 for e in listed)
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
    got = bd.decode_coefficients(reqs)
    for (s, k), t, i in zip(reqs, got, bd.last_coefficients_info):
        n_present, error, want = expected(MIXED[s], k)
        assert tuple(t.shape) == (*geometry(bd, s), 6, 8, 8)
        assert (i["n_present"], i["error"]) == (n_present, error) and np.array_equal(flat(t), want), (MIXED[s], k)
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
        got = bd.decode_coefficients(reqs, macroblocks=True)
        outs.append(([(host(c), host(m)) for c, m in got], bd.last_coefficients_info))
        bd.close()
    assert len(outs[0][0]) == len(outs[1][0]) >= 50
    assert outs[0][1] == outs[1][1]
    for (a, ma), (b, mb) in zip(outs[0][0], outs[1][0]):
        assert np.array_equal(a, b) and np.array_equal(ma, mb)


def _oracle_from(es, entry):
    """The oracle fed the first sequence header + es[byte_pos:]: the walk reads the same bits past the closing code
    as the device's does.  (picture_info, records, raw coefficient plane)."""
    h = intra_model.first_sequence_header(es)[0]
    nxt = es.find(intra_model.START, h + 4)
    header = es[h:nxt]
    got = oracle_coefficients(header + es[entry["byte_pos"]:], stop=len(header))
    assert got[0][0] == len(header)
    return got[0][1:]


def test_damaged_streams_follow_the_stated_rule():
    """Bit flips in every third picture of an I/P stream and in the pictures of a B stream, three seeds.  The walk reads
    past the closing code like the oracle fed everything from the picture on; a macroblock it stops in while reading a
    block keeps the cbp bits of the blocks it finished, and the block it could not read (which the oracle half-wrote)
    and those after it are 0.  So the device equals the model of that oracle, error presence and entries included --
    and such half-written blocks occur."""
    clean = ffmpeg_es(320, 240, 24) + synth_es.make_case("i_only_320x240")[-4:]  # end code: the last picture closes
    b_clean = synth_es.make_case("b_one_slice_fcodes")
    streams = []
    for seed in (1, 2, 3):
        streams += [_damage(clean, macroblock_model.macroblock_index(clean)[::3], seed),
                    _damage(b_clean, macroblock_model.macroblock_index(b_clean)[1::2], seed, flips=3)]
    bd = BatchDecoder(len(streams))
    errors = half_written = 0
    for s, es in enumerate(streams):
        bd.write(s, es)
        entries = macroblock_model.macroblock_index(es)
        got = bd.decode_coefficients([(s, e["picture"]) for e in entries], macroblocks=True)
        for e, (c, m), i in zip(entries, got, bd.last_coefficients_info):
            info, rec, raw = _oracle_from(es, e)
            want = macroblock_model.coefficients(rec, raw)
            assert bool(i["error"]) == bool(info.error), (s, e["picture"])
            assert np.array_equal(flat(c), want), (s, e["picture"])
            assert np.array_equal(host(m).reshape(-1, 16), macroblock_model.export(rec, e["type"])), (s, e["picture"])
            errors += bool(i["error"])
            # blocks of present macroblocks with a clear cbp bit that the oracle wrote into: the stopped blocks
            r = np.frombuffer(rec.tobytes(), macroblock_model.RECORD)
            present = (r["flags"] & macroblock_model.MBF_PRESENT) != 0
            uncoded = present[:, None] & (((r["cbp"][:, None] >> (5 - np.arange(6))) & 1) == 0)
            half_written += int((raw.reshape(-1, 6, 64)[uncoded] != 0).any(axis=1).sum())
    assert errors and half_written and bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("name,decode_b", [("ffmpeg_320x240", False), ("b_rows", True)])
def test_decode_state_is_untouched(name, decode_b):
    """decode_coefficients in the middle of a decode() run: the state is as before the call, and every picture of the
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
                bd.decode_coefficients([(s, e["picture"]) for s in (0, 1) for e in bd.macroblock_index(s)], macroblocks=True)
                _assert_same_state(before, _state(bd, 0))
        runs.append(frames)
        bd.close()
    assert len(runs[0]) == len(runs[1])
    for a, b in zip(*runs):
        assert np.array_equal(a, b)


def test_invalid_requests_are_refused_and_change_nothing():
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
    first, entries = bd.decode_coefficients([(0, 1)], macroblocks=True)[0]  # a B picture, decode_b off
    mark, mark_mb = first.clone().fill_(7), entries.clone().fill_(7)

    def call(reqs, dsts, mb_dsts=None):
        n = len(reqs)
        return bd.lib.jsmpeg_b200_batch_decode_coefficients(
            bd.handle, n, (ctypes.c_int * n)(*[s for s, _ in reqs]), (ctypes.c_uint32 * n)(*[p for _, p in reqs]),
            (ctypes.c_void_p * n)(*dsts), None if mb_dsts is None else (ctypes.c_void_p * n)(*mb_dsts), None, None)

    # with a valid request in front: the unclosed tail, no sequence header, no stream, no picture, f_code 0, D
    for stream_, pic in ((0, model[-1]["picture"]), (1, 0), (3, 0), (-1, 0), (0, 99), (2, 2), (2, 6)):
        assert call([(0, 4), (stream_, pic)], [mark.data_ptr(), first.data_ptr()]) == -2, (stream_, pic)
        with pytest.raises(ValueError):
            bd.decode_coefficients([(0, 4), (stream_, pic)])
    assert call([(0, 4)], [None]) == -2                                  # NULL destination
    assert call([(0, 4)], [mark.data_ptr() + 8]) == -2                   # misaligned destination
    assert call([(0, 4)], [mark.data_ptr()], [mark_mb.data_ptr() + 4]) == -2  # misaligned macroblock destination
    assert call([(0, 4)], [mark.data_ptr()], [None]) == -2               # NULL macroblock destination in a given array
    assert bool((mark == 7).all()) and bool((mark_mb == 7).all())
    _assert_same_state(before, _state(bd, 0))
    assert bd.last_error() is None
    # mb_dst = NULL: the coefficients alone, and the same bytes
    assert call([(0, 1)], [mark.data_ptr()]) == 1
    assert np.array_equal(host(mark), host(first)) and np.array_equal(flat(first), expected("b_rows", 1)[2])
    assert np.array_equal(host(entries), host(bd.decode_macroblocks([(0, 1)])[0]))
    bd.close()


def launch_counts():
    """({kernel: launches} of decode_coefficients without and with the entries, the decoder's launch counters) on
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
            bd.decode_coefficients(reqs, macroblocks=macroblocks)
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
    """On test_gpu_launch_counts' workload (lane-walk, slice-walk and B-walk pictures in one wave of more than 64 x 8
    lane-walk pictures): the three walks, expand in the lane walk's 8 size groups and beside the other two walks, one
    export_coefficients_kernel, and export_macroblocks_kernel only when the entries are asked for.  The decoder's launch
    counters are decode()'s and stay as they were.  (Counted in a process of its own: the profiler sessions of this
    count then share nothing with those of other tests.)"""
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "launch-counts"], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    seen, counters = json.loads(r.stdout.strip().splitlines()[-1])
    walks = {"walk_pictures_lanes_kernel": 8, "walk_pictures_slices_kernel": 1, "walk_pictures_b_kernel": 1,
             "expand_blocks_kernel": 10, "export_coefficients_kernel": 1}
    assert seen == [walks, {**walks, "export_macroblocks_kernel": 1}]
    assert counters == [0, 0]


def test_the_bench_shape():
    """8 pictures from each of the bench's 64 distinct 1080p clips in one call equal the model of the oracle."""
    sys.path.insert(0, helpers.ROOT)
    import bench
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips))
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    rng = random.Random(11)
    reqs = [(s, k) for s in range(len(clips)) for k in sorted(rng.sample([e["picture"] for e in bd.macroblock_index(s)], 8))]
    got = bd.decode_coefficients(reqs)
    assert bd.last_error() is None
    by_stream = {}
    for (s, k), t in zip(reqs, got):
        by_stream.setdefault(s, []).append((k, t))
    for s, items in by_stream.items():
        index = {e["picture"]: e for e in macroblock_model.macroblock_index(clips[s])}
        for k, t in items:
            assert tuple(t.shape) == (68, 120, 6, 8, 8)
            assert np.array_equal(flat(t), oracle_fresh_coefficients(clips[s], index[k])[2]), (s, k)
    bd.close()


if __name__ == "__main__" and sys.argv[1:] == ["launch-counts"]:
    print(json.dumps(launch_counts()))
