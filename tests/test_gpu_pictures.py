"""Random access on the device (jsmpeg_b200_batch_picture_index / _decode_pictures) against the serial model
(tools/chain_model.py), the oracle fed the fresh-decoder byte string, and the batch's own decode(): the index in any
chunking, every listed picture of the key-picture corpus and of I/P/B streams, whole streams picture for picture,
mixed sizes, slot pressure, damaged pictures, and the decode() state the call must leave alone."""
import ctypes
import functools
import random

import numpy as np
import pytest

import chain_model
import helpers
import intra_model
import synth_es
from jsmpeg_b200.batch import OUT_HOST, OUT_RGBA, BatchDecoder, planes_view
from test_gpu_intra import CORPUS, _assert_same_state, _state, ffmpeg_es, host, random_cuts
from test_gpu_intra import stream as intra_stream
from test_picture_index import fresh_decode, open_gop_clip

pytestmark = pytest.mark.gpu

B_CORPUS = sorted(synth_es.B_CASES) + ["open_gop"]


def stream(name):
    if name == "open_gop":
        return open_gop_clip()
    return synth_es.make_case(name) if name in synth_es.B_CASES else intra_stream(name)


@functools.lru_cache(maxsize=None)
def oracle_planes(name, picture, decode_b):
    """Y | Cr | Cb of the oracle fed the fresh bytes of picture `picture` of corpus stream `name`."""
    es = stream(name)
    entry = next(e for e in chain_model.picture_index(es, decode_b) if e["picture"] == picture)
    planes, _, _ = fresh_decode(es, entry, decode_b)
    return np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in planes])


def gpu_fresh(es, entry, decode_b=False, rgba=False, whole_tail=False):
    """The device's own decode() of chain_model.fresh_bytes(es, entry) in a new batch, until it consumes picture k:
    (status, Y | Cr | Cb, RGBA or None).  Status 0, zero planes and white RGBA when it never consumes picture k.
    whole_tail: fed the rest of the buffer after the closing code too (a damaged walk may run across that code)."""
    if whole_tail:
        entry = dict(entry, close=len(es) - 4)
    fresh = chain_model.fresh_bytes(es, entry)
    target = chain_model.target_start_byte(es, entry) - 4
    starts = [p for p in intra_model.prefixes(fresh) if p + 3 < len(fresh) and fresh[p + 3] == 0]
    bd = BatchDecoder(1, decode_b=decode_b)
    bd.write(0, fresh)
    info = bd.stream_info(0)
    try:
        while True:
            at = (bd.get_index(0) + 7) >> 3
            nxt = next((p for p in starts if p >= at), None)
            if nxt is None or nxt > target:
                image = np.full((info["height"], info["width"], 4), 255, np.uint8) if rgba else None
                return 0, np.zeros(info["coded_size"] * 3 // 2, np.uint8), image
            assert bd.decode(1, OUT_RGBA if rgba else 0) == 1
            if nxt == target:
                return 1, np.concatenate(bd.read_planes(0)), (bd.read_rgba(0) if rgba else None)
    finally:
        bd.close()


def index_tuples(entries):
    return [(e["picture"], e["byte_pos"], e["type"], e["temporal_reference"], e["chain_start"]) for e in entries]


@pytest.mark.parametrize("decode_b", [False, True])
@pytest.mark.parametrize("name", ["rows_ip", "ignored_pictures_userdata", "random_slices_gaps", "random_2", "b_rows",
                                  "b_three", "ffmpeg_320x240"])
def test_index_matches_the_model_whole_and_in_random_chunkings(name, decode_b):
    es = stream(name)
    h_end = (intra_model.first_sequence_header(es)[1] + 7) >> 3
    chunkings = [[]] + [[c for c in random_cuts(len(es), seed, mean) if c > h_end] for seed, mean in ((1, 300), (2, 4000))]
    bd = BatchDecoder(len(chunkings), decode_b=decode_b)
    for s, cuts in enumerate(chunkings):
        prev = 0
        for c in cuts + [len(es)]:
            bd.write(s, es[prev:c])
            prev = c
            assert index_tuples(bd.picture_index(s)) == index_tuples(chain_model.picture_index(es[:c], decode_b)), (name, s, c)
    bd.set_option("decode_b", not decode_b)  # the index follows the option's current value
    assert index_tuples(bd.picture_index(0)) == index_tuples(chain_model.picture_index(es, not decode_b))
    assert bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("slice_walk", [0, 1])
@pytest.mark.parametrize("name", CORPUS + B_CORPUS)
def test_every_listed_picture_equals_the_fresh_oracle(name, slice_walk):
    es = stream(name)
    decode_b = name in B_CORPUS
    bd = BatchDecoder(1, slice_walk=slice_walk, decode_b=decode_b)
    bd.write(0, es)
    entries = bd.picture_index(0)
    assert index_tuples(entries) == index_tuples(chain_model.picture_index(es, decode_b))
    got = bd.decode_pictures([(0, e["picture"]) for e in entries])
    for e, t, i in zip(entries, got, bd.last_pictures_info):
        assert i["status"] == 1 and i["error"] == 0, (name, e["picture"], i)
        assert np.array_equal(host(t), oracle_planes(name, e["picture"], decode_b)), (name, e["picture"])
    assert bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("name", ["odd_size", "random_slices_gaps", "ffmpeg_320x240", "b_one_slice_fcodes", "open_gop"])
def test_rgba_equals_the_devices_own_fresh_decode(name):
    es = stream(name)
    decode_b = name in B_CORPUS
    bd = BatchDecoder(1, decode_b=decode_b)
    bd.write(0, es)
    entries = bd.picture_index(0)
    got = bd.decode_pictures([(0, e["picture"]) for e in entries], rgba=True)
    info = bd.stream_info(0)
    for e, (planes, image) in zip(chain_model.picture_index(es, decode_b), got):
        status, want_planes, want_image = gpu_fresh(es, e, decode_b, rgba=True)
        assert status == 1 and tuple(image.shape) == (info["height"], info["width"], 4)
        assert np.array_equal(host(planes), want_planes) and np.array_equal(host(image), want_image), (name, e["picture"])
    bd.close()


@pytest.mark.parametrize("name,decode_b", [("ffmpeg_320x240", False), ("open_gop", True)])
def test_every_picture_is_the_batchs_own_decode_sequence(name, decode_b):
    """All listed pictures of a clean stream in one call give exactly what decode() gives, picture for picture."""
    es = stream(name)
    bd = BatchDecoder(2, decode_b=decode_b)
    bd.write(0, es)
    bd.write(1, es)
    entries = bd.picture_index(0)
    got = bd.decode_pictures([(0, e["picture"]) for e in entries])
    sequence = []
    while bd.decode(1, OUT_HOST):
        sequence.append(np.concatenate(bd.read_planes(1)))
    assert len(entries) >= len(sequence) - 1  # (every picture but the unclosed tail is listed)
    for e, t in zip(entries, got):
        assert np.array_equal(host(t), sequence[e["picture"]]), (name, e["picture"])
    bd.close()


def test_program_stream_through_write_ps():
    import gen_streams
    data = gen_streams.make_clip_ps(320, 240, 24, form="mpg")
    m1v = gen_streams.make_clip_m1v(320, 240, 24)
    bd = BatchDecoder(1)
    _, pes = bd.write_ps(0, data)
    entries = bd.picture_index(0)
    assert index_tuples(entries) == index_tuples(chain_model.picture_index(m1v)) and len(entries) >= 20
    offsets = [o for o, _ in pes]
    for e in entries:  # the PTS of the last PES packet that starts at or before the picture (decoder.js:36-47)
        j = max(i for i, o in enumerate(offsets) if o <= e["byte_pos"]) if offsets[0] <= e["byte_pos"] else None
        assert e["pts"] == (pes[j][1] if j is not None else None)
    assert entries[-1]["pts"] is not None and entries[-1]["pts"] > entries[0]["pts"]
    got = bd.decode_pictures([(0, e["picture"]) for e in entries])
    for e, t in zip(chain_model.picture_index(m1v), got):
        planes, _, _ = fresh_decode(m1v, e)
        assert np.array_equal(host(t), np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in planes]))
    bd.close()


MIXED = ["ffmpeg_320x240", "ffmpeg_1280x720", "ffmpeg_1920x1080", "odd_size", "rows_ip", "b_rows", "open_gop"]


def test_mixed_sizes_shuffled_with_duplicates():
    bd = BatchDecoder(len(MIXED), decode_b=True)
    for s, name in enumerate(MIXED):
        bd.write(s, stream(name))
    rng = random.Random(5)
    reqs = []
    for s in range(len(MIXED)):
        pics = [e["picture"] for e in bd.picture_index(s)]
        reqs += [(s, k) for k in rng.sample(pics, min(len(pics), 6))]
    reqs += [reqs[2], reqs[9], reqs[9]]  # the same picture two and three times
    rng.shuffle(reqs)
    got = bd.decode_pictures(reqs, rgba=True)
    assert all(i["status"] == 1 for i in bd.last_pictures_info)
    for (s, k), (t, image) in zip(reqs, got):
        assert t.numel() == bd.stream_info(s)["coded_size"] * 3 // 2
        assert np.array_equal(host(t), oracle_planes(MIXED[s], k, True)), (MIXED[s], k)
    for (s, k), (t, image) in zip(reqs, got):  # duplicates: the same picture and the same RGBA
        first = reqs.index((s, k))
        assert np.array_equal(host(image), host(got[first][1])), (MIXED[s], k)
    y, cr, cb = planes_view(got[0][0], bd.stream_info(reqs[0][0]))
    assert y.data_ptr() == got[0][0].data_ptr() and cr.shape == cb.shape
    bd.close()


def test_slot_pressure_gives_the_same_bytes():
    """Three record slots for chains of up to 12 pictures: several waves per chain group, several chain groups."""
    names = ["ffmpeg_320x240", "rows_ip", "b_rows", "open_gop"]
    outs = []
    for max_slots in (0, 3):
        bd = BatchDecoder(len(names), max_slots=max_slots, decode_b=True)
        for s, name in enumerate(names):
            bd.write(s, stream(name))
        reqs = [(s, e["picture"]) for s in range(len(names)) for e in bd.picture_index(s)]
        bd.decode(2)  # the look-ahead holds slots too
        outs.append([host(t) for t in bd.decode_pictures(reqs)])
        bd.close()
    assert len(outs[0]) == len(outs[1]) >= 40
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def _skipping_cut(es, pics):
    """A copy of `es` with a byte dropped at the end of some picture i such that the oracle's decode() of the copy
    never consumes picture i + 1 (the walk of i runs across its start code): (copy, i)."""
    from jsmpeg_b200 import decoder
    lib = helpers.oracle_lib()
    for i in range(3, len(pics) - 2):
        for drop in range(1, 8):
            buf = es[:pics[i + 1] - drop] + es[pics[i + 1]:]
            d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=lib)
            d.write(0, [buf])
            starts = []
            while d.decode():
                starts.append(lib.oracle_last_picture_info(d.decoder).contents.start_byte - 4)
            d.destroy()
            if pics[i + 1] - drop not in starts:
                return buf, i
    raise AssertionError("no cut makes decode() skip a picture")


@pytest.mark.parametrize("seed", [1, 2])
def test_damaged_pictures_equal_the_devices_own_fresh_decode(seed):
    """Bit flips in every third picture, and a cut that makes one picture's walk run across the next start code (the
    next picture is then never consumed: status 0).  Such a walk reads on past a closing code, so the reference here
    is the device's fresh decoder fed the chain start and everything behind it."""
    from test_gpu_intra import _damage
    clean = ffmpeg_es(320, 240, 24) + synth_es.make_case("i_only_320x240")[-4:]  # end code: the last picture closes
    damaged = _damage(clean, chain_model.picture_index(clean)[::3], seed)
    pics = [p for p in intra_model.prefixes(damaged) if damaged[p + 3] == 0]
    cut, skipped = _skipping_cut(damaged, pics)
    for es in (damaged, cut):
        entries = chain_model.picture_index(es)
        bd = BatchDecoder(1)
        bd.write(0, es)
        assert index_tuples(bd.picture_index(0)) == index_tuples(entries)
        got = bd.decode_pictures([(0, e["picture"]) for e in entries])
        info = bd.last_pictures_info
        for e, t, i in zip(entries, got, info):
            status, planes, _ = gpu_fresh(es, e, whole_tail=True)
            assert i["status"] == status and np.array_equal(host(t), planes), (seed, e["picture"], i)
        if es is cut:
            assert info[[e["picture"] for e in entries].index(skipped + 1)]["status"] == 0
            assert not bool(got[[e["picture"] for e in entries].index(skipped + 1)].any())
        else:
            assert any(i["error"] for i in info)
        assert bd.last_error() is None
        bd.close()


@pytest.mark.parametrize("name,decode_b", [("ffmpeg_320x240", False), ("b_rows", True), ("open_gop", True)])
def test_decode_state_is_untouched(name, decode_b):
    """decode_pictures in the middle of a decode() run: the state is as before the call, and every picture of the run
    equals that of a twin batch that never called it."""
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
                reqs = [(s, e["picture"]) for s in (0, 1) for e in bd.picture_index(s)]
                bd.decode_pictures(reqs, rgba=True)
                _assert_same_state(before, _state(bd, 0))
        runs.append(frames)
        bd.close()
    assert len(runs[0]) == len(runs[1])
    for a, b in zip(*runs):
        assert np.array_equal(a, b)


def test_invalid_requests_are_refused_and_change_nothing():
    es = synth_es.make_case("b_rows")  # I B B P B B I B B P B B I
    model = chain_model.picture_index(es, True)
    cut = es[:model[-1]["close"] + 2]  # the last I picture is not closed yet
    bd = BatchDecoder(2, decode_b=True)
    bd.write(0, cut)
    bd.write(1, es[intra_model.first_sequence_header(es)[0] + 4:])  # no sequence header
    assert bd.decode(1, OUT_HOST)
    before = _state(bd, 0)
    listed = [e["picture"] for e in bd.picture_index(0)]
    assert listed == [e["picture"] for e in model[:-1]]
    first = bd.decode_pictures([(0, 4)])[0]
    mark = first.clone().fill_(7)

    def call(reqs, dsts, flags=0, rgba=None):
        n = len(reqs)
        return bd.lib.jsmpeg_b200_batch_decode_pictures(
            bd.handle, n, (ctypes.c_int * n)(*[s for s, _ in reqs]), (ctypes.c_uint32 * n)(*[p for _, p in reqs]),
            (ctypes.c_void_p * n)(*dsts), rgba, flags, None, None, None)

    # with a valid request in front: a B picture without a chain start, the unclosed tail, no sequence header, no stream
    for stream_, pic in ((0, 1), (0, model[-1]["picture"]), (1, 0), (2, 0), (0, 99)):
        assert call([(0, 4), (stream_, pic)], [mark.data_ptr(), first.data_ptr()]) == -2, (stream_, pic)
        with pytest.raises(ValueError):
            bd.decode_pictures([(0, 4), (stream_, pic)])
    assert call([(0, 4)], [None]) == -2                                  # NULL destination
    assert call([(0, 4)], [mark.data_ptr() + 1]) == -2                   # misaligned destination
    assert call([(0, 4)], [mark.data_ptr()], flags=OUT_RGBA) == -2       # RGBA without RGBA destinations
    bd.set_option("decode_b", 0)
    assert call([(0, 4)], [mark.data_ptr()]) == -2                       # a B picture while decode_b is off
    bd.set_option("decode_b", 1)
    assert bool((mark == 7).all())
    _assert_same_state(before, _state(bd, 0))
    assert bd.last_error() is None
    assert np.array_equal(host(first), oracle_planes("b_rows", 4, True))
    bd.close()
