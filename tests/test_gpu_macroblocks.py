"""Macroblock data on the device (jsmpeg_b200_batch_macroblock_index / _decode_macroblocks) against the serial model
(tools/macroblock_model.py) applied to the oracle's records: the index in any chunking, every listed picture of the
key-picture corpus, of I/P/B streams and of an .mpg, with the slice walk and decode_b on and off, mixed sizes with
duplicates, slot pressure, damaged streams, the decode() state the call must leave alone, and invalid requests."""
import ctypes
import functools
import os
import random

import numpy as np
import pytest

import helpers
import intra_model
import macroblock_model
import synth_es
from jsmpeg_b200.batch import MB_BACKWARD, MB_FORWARD, MB_INTRA, MB_PRESENT, MB_SKIPPED, OUT_HOST, BatchDecoder, macroblocks_view
from test_gpu_intra import CORPUS, _assert_same_state, _damage, _state, ffmpeg_es, host, random_cuts
from test_gpu_intra import stream as intra_stream
from test_macroblock_index import MINI_ENC, corpus_stream, oracle_fresh, oracle_records

pytestmark = pytest.mark.gpu

FIXTURE_720P = os.path.join(helpers.ROOT, "tests", "fixtures", "b_clip_1280x720.m1v")
B_CORPUS = sorted(synth_es.B_CASES) + sorted(MINI_ENC) + ["b_clip_1280x720"]


@functools.lru_cache(maxsize=None)
def stream(name):
    if name == "b_clip_1280x720":
        return open(FIXTURE_720P, "rb").read()
    if name in MINI_ENC:
        return corpus_stream(name)
    return synth_es.make_case(name) if name in synth_es.B_CASES else intra_stream(name)


def index_tuples(entries):
    return [(e["picture"], e["byte_pos"], e["type"], e["temporal_reference"]) for e in entries]


@functools.lru_cache(maxsize=None)
def expected(name, picture):
    """(n_present, error, uint8 [mb_size, 16]) of listed picture `picture` of corpus stream `name`: the model's
    conversion of the records of the oracle fed the picture's fresh bytes."""
    es = stream(name)
    entry = next(e for e in macroblock_model.macroblock_index(es) if e["picture"] == picture)
    info, rec = oracle_fresh(es, entry)
    return info.n_present, info.error, macroblock_model.export(rec, entry["type"])


def geometry(bd, s):
    info = bd.stream_info(s)
    return (info["height"] + 15) // 16, (info["width"] + 15) // 16


@pytest.mark.parametrize("name", ["rows_ip", "ignored_pictures_userdata", "random_slices_gaps", "random_2", "b_rows",
                                  "b_three", "ffmpeg_320x240"])
def test_index_matches_the_model_whole_and_in_random_chunkings(name):
    es = stream(name)
    h_end = (intra_model.first_sequence_header(es)[1] + 7) >> 3
    chunkings = [[]] + [[c for c in random_cuts(len(es), seed, mean) if c > h_end] for seed, mean in ((1, 300), (2, 4000))]
    bd = BatchDecoder(len(chunkings))
    for s, cuts in enumerate(chunkings):
        prev = 0
        for c in cuts + [len(es)]:
            bd.write(s, es[prev:c])
            prev = c
            assert index_tuples(bd.macroblock_index(s)) == index_tuples(macroblock_model.macroblock_index(es[:c])), (name, s, c)
    for decode_b in (1, 0):  # B pictures are listed whatever decode_b says
        bd.set_option("decode_b", decode_b)
        assert index_tuples(bd.macroblock_index(0)) == index_tuples(macroblock_model.macroblock_index(es))
    assert bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("name", CORPUS + B_CORPUS)
def test_every_listed_picture_equals_the_oracle_with_every_option(name):
    """All listed pictures in one call, with the slice walk and decode_b each off and on: the same entries, the model's
    conversion of the oracle's records."""
    es = stream(name)
    entries = macroblock_model.macroblock_index(es)
    assert entries
    for slice_walk, decode_b in ((0, 0), (1, 0), (0, 1), (1, 1)):
        bd = BatchDecoder(1, slice_walk=slice_walk, decode_b=decode_b)
        bd.write(0, es)
        assert index_tuples(bd.macroblock_index(0)) == index_tuples(entries)
        got = bd.decode_macroblocks([(0, e["picture"]) for e in entries])
        for e, t, i in zip(entries, got, bd.last_macroblocks_info):
            n_present, error, want = expected(name, e["picture"])
            assert tuple(t.shape) == (*geometry(bd, 0), 16) and t.is_cuda
            assert (i["n_present"], i["error"]) == (n_present, error), (name, e["picture"], slice_walk, decode_b)
            assert np.array_equal(host(t).reshape(-1, 16), want), (name, e["picture"], slice_walk, decode_b)
        assert bd.last_error() is None
        bd.close()


def test_motion_is_there():
    """The I/P/B corpus carries every kind of entry: intra, forward, backward and bidirectional macroblocks, non-zero
    vectors in both directions, and skipped macroblocks."""
    import torch
    es = stream("b_clip_1280x720")
    bd = BatchDecoder(1)
    bd.write(0, es)
    entries = bd.macroblock_index(0)
    assert [e["type"] for e in entries].count(3) == 8
    views = [macroblocks_view(t) for t in bd.decode_macroblocks([(0, e["picture"]) for e in entries])]
    flags = np.concatenate([host(v["flags"]).reshape(-1) for v in views])
    assert (flags & MB_PRESENT).all() and (flags & MB_SKIPPED).any()
    for kind in (MB_INTRA, MB_FORWARD, MB_BACKWARD, MB_FORWARD | MB_BACKWARD):
        assert ((flags & (MB_INTRA | MB_FORWARD | MB_BACKWARD)) == kind).any(), kind
    assert any(host(v["forward"]).any() for v in views) and any(host(v["backward"]).any() for v in views)
    v = views[0]
    assert v["forward"].dtype == v["backward"].dtype == torch.int16 and tuple(v["backward"].shape) == (45, 80, 2)
    assert tuple(v["flags"].shape) == tuple(v["cbp"].shape) == tuple(v["qscale"].shape) == (45, 80)
    assert (host(v["qscale"]) > 0).all()
    bd.close()


def test_program_stream_through_write_ps():
    import gen_streams
    data = gen_streams.make_clip_ps(320, 240, 24, form="mpg")
    m1v = gen_streams.make_clip_m1v(320, 240, 24)
    bd = BatchDecoder(1)
    _, pes = bd.write_ps(0, data)
    entries = bd.macroblock_index(0)
    model = macroblock_model.macroblock_index(m1v)
    assert index_tuples(entries) == index_tuples(model) and len(entries) >= 20
    assert entries[-1]["pts"] is not None and entries[-1]["pts"] > entries[0]["pts"]
    got = bd.decode_macroblocks([(0, e["picture"]) for e in entries])
    for e, t in zip(model, got):
        info, rec = oracle_fresh(m1v, e)
        assert np.array_equal(host(t).reshape(-1, 16), macroblock_model.export(rec, e["type"])), e["picture"]
    bd.close()


MIXED = ["ffmpeg_320x240", "ffmpeg_1280x720", "ffmpeg_1920x1080", "odd_size", "rows_ip", "b_rows", "mini_enc_open_gop"]


def test_mixed_sizes_shuffled_with_duplicates():
    bd = BatchDecoder(len(MIXED))
    for s, name in enumerate(MIXED):
        bd.write(s, stream(name))
    rng = random.Random(5)
    reqs = []
    for s in range(len(MIXED)):
        pics = [e["picture"] for e in bd.macroblock_index(s)]
        reqs += [(s, k) for k in rng.sample(pics, min(len(pics), 6))]
    reqs += [reqs[2], reqs[9], reqs[9]]  # the same picture two and three times
    rng.shuffle(reqs)
    got = bd.decode_macroblocks(reqs)
    for (s, k), t, i in zip(reqs, got, bd.last_macroblocks_info):
        n_present, error, want = expected(MIXED[s], k)
        assert tuple(t.shape) == (*geometry(bd, s), 16)
        assert (i["n_present"], i["error"]) == (n_present, error) and np.array_equal(host(t).reshape(-1, 16), want), (MIXED[s], k)
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
        outs.append(([host(t) for t in bd.decode_macroblocks(reqs)], bd.last_macroblocks_info))
        bd.close()
    assert len(outs[0][0]) == len(outs[1][0]) >= 50
    assert outs[0][1] == outs[1][1]
    for a, b in zip(outs[0][0], outs[1][0]):
        assert np.array_equal(a, b)


def _oracle_from(es, entry):
    """The oracle fed the first sequence header + es[byte_pos:]: the walk reads the same bits past the closing code
    as the device's does.  (picture_info, entries)."""
    h = intra_model.first_sequence_header(es)[0]
    nxt = es.find(intra_model.START, h + 4)
    header = es[h:nxt]
    got = oracle_records(header + es[entry["byte_pos"]:], stop=len(header))
    assert got[0][0] == len(header)
    return got[0][1], macroblock_model.export(got[0][2], entry["type"])


@pytest.mark.parametrize("seed", [1, 2])
def test_damaged_streams_equal_the_oracle(seed):
    """Bit flips in every third picture of an I/P stream and in the pictures of a B stream: the records and the
    presence of an error equal the oracle's (n_present is a statistic the walks count differently on damage)."""
    clean = ffmpeg_es(320, 240, 24) + synth_es.make_case("i_only_320x240")[-4:]  # end code: the last picture closes
    b_clean = synth_es.make_case("b_one_slice_fcodes")
    streams = [_damage(clean, macroblock_model.macroblock_index(clean)[::3], seed),
               _damage(b_clean, macroblock_model.macroblock_index(b_clean)[1::2], seed, flips=3)]
    bd = BatchDecoder(len(streams))
    errors = 0
    for s, es in enumerate(streams):
        bd.write(s, es)
        entries = macroblock_model.macroblock_index(es)
        assert index_tuples(bd.macroblock_index(s)) == index_tuples(entries)
        got = bd.decode_macroblocks([(s, e["picture"]) for e in entries])
        for e, t, i in zip(entries, got, bd.last_macroblocks_info):
            info, want = _oracle_from(es, e)
            assert bool(i["error"]) == bool(info.error) and np.array_equal(host(t).reshape(-1, 16), want), (seed, s, e["picture"])
            errors += bool(i["error"])
    assert errors and bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("name,decode_b", [("ffmpeg_320x240", False), ("b_rows", False), ("b_rows", True),
                                           ("mini_enc_open_gop", True)])
def test_decode_state_is_untouched(name, decode_b):
    """decode_macroblocks in the middle of a decode() run: the state is as before the call, and every picture of the
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
                reqs = [(s, e["picture"]) for s in (0, 1) for e in bd.macroblock_index(s)]
                bd.decode_macroblocks(reqs)
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
    assert [e["picture"] for e in bd.macroblock_index(0)] == [e["picture"] for e in model[:-1]]
    first = bd.decode_macroblocks([(0, 1)])[0]  # a B picture without a chain start, decode_b off
    mark = first.clone().fill_(7)

    def call(reqs, dsts):
        n = len(reqs)
        return bd.lib.jsmpeg_b200_batch_decode_macroblocks(
            bd.handle, n, (ctypes.c_int * n)(*[s for s, _ in reqs]), (ctypes.c_uint32 * n)(*[p for _, p in reqs]),
            (ctypes.c_void_p * n)(*dsts), None, None)

    # with a valid request in front: the unclosed tail, no sequence header, no stream, no picture, f_code 0, D
    for stream_, pic in ((0, model[-1]["picture"]), (1, 0), (3, 0), (-1, 0), (0, 99), (2, 2), (2, 6)):
        assert call([(0, 4), (stream_, pic)], [mark.data_ptr(), first.data_ptr()]) == -2, (stream_, pic)
        with pytest.raises(ValueError):
            bd.decode_macroblocks([(0, 4), (stream_, pic)])
    assert call([(0, 4)], [None]) == -2                     # NULL destination
    assert call([(0, 4)], [mark.data_ptr() + 8]) == -2      # misaligned destination
    assert bool((mark == 7).all())
    _assert_same_state(before, _state(bd, 0))
    assert bd.last_error() is None
    n_present, error, want = expected("b_rows", 1)
    assert np.array_equal(host(first).reshape(-1, 16), want)
    assert bd.lib.jsmpeg_b200_batch_macroblock_index(bd.handle, 3, None, None, None, None, 0) == -2
    bd.close()
