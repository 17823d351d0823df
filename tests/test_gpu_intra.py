"""Key pictures on the device (jsmpeg_b200_batch_intra_index / _decode_intra) against the serial model
(tools/intra_model.py) and the oracle fed the fresh-decoder byte string: the index in any chunking, the decoded planes
and RGBA pictures byte for byte, mixed sizes in one call, slot pressure, damaged pictures, and the decode() state the
call must leave alone."""
import ctypes
import functools
import random

import numpy as np
import pytest

import helpers
import intra_model
import synth_es
from jsmpeg_b200 import decoder
from jsmpeg_b200.batch import OUT_HOST, OUT_RGBA, BatchDecoder, planes_view

pytestmark = pytest.mark.gpu


def oracle_fresh(es, entry):
    """Y | Cr | Cb of the oracle fed fresh_bytes(es, entry), one decode()."""
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=helpers.oracle_lib())
    rec = decoder.PlaneRecorder()
    d.connect(rec)
    d.write(0.0, [intra_model.fresh_bytes(es, entry)])
    assert d.decode()
    d.destroy()
    return np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in rec.frames[0]])


def gpu_fresh(es, entry, rgba=False):
    """The device's own decode() of fresh_bytes(es, entry) in a new batch: (Y | Cr | Cb, RGBA or None, parse errors)."""
    bd = BatchDecoder(1)
    bd.write(0, intra_model.fresh_bytes(es, entry))
    assert bd.decode(1, OUT_RGBA if rgba else 0) == 1
    planes = np.concatenate(bd.read_planes(0))
    image = bd.read_rgba(0) if rgba else None
    errors = bd.stats()["parse_errors"]
    bd.close()
    return planes, image, errors


def random_stream(seed):
    k = synth_es.Knobs(width=int(16 * (2 + seed)), height=int(16 * (1 + seed % 3)) + 2 * seed, pictures=7, gop=3,
                       slices=["one", "rows", "random"][seed % 3], slice_gap_prob=0.2, stuffing_prob=0.2,
                       skip_prob=0.3, f_codes=(1, 2, 3, 4), full_pel_prob=0.3, escape_prob=0.3,
                       custom_matrices=bool(seed & 1), extension_user_data=True, ignored_pictures=bool(seed & 2))
    return synth_es.SynthStream(k, 1000 + seed).generate()


def ffmpeg_es(w, h, n, seed=1234):
    return b"".join(p for _, p in helpers.clip_packets(w, h, n, seed=seed))


FFMPEG = {"ffmpeg_320x240": (320, 240, 24), "ffmpeg_1280x720": (1280, 720, 6), "ffmpeg_1920x1080": (1920, 1080, 13)}
CORPUS = sorted(synth_es.CASES) + [f"random_{seed}" for seed in range(6)] + list(FFMPEG)


@functools.lru_cache(maxsize=None)
def stream(name):
    """A stream of the corpus by name (made when a test asks for it, not at collection)."""
    if name in FFMPEG:
        return ffmpeg_es(*FFMPEG[name])
    if name.startswith("random_") and name[7:].isdigit():
        return random_stream(int(name[7:]))
    return synth_es.make_case(name)


def index_tuples(entries):
    return [(e["picture"], e["byte_pos"], e["temporal_reference"]) for e in entries]


def host(t):
    return t.cpu().numpy()


def random_cuts(n, seed, mean):
    rng = random.Random(seed)
    cuts, at = [], 0
    while True:
        at += rng.randint(1, 2 * mean)
        if at >= n:
            return cuts
        cuts.append(at)


@pytest.mark.parametrize("name", CORPUS)
def test_index_matches_the_model_whole_and_in_random_chunkings(name):
    es = stream(name)
    want = index_tuples(intra_model.intra_index(es))
    assert want
    h_end = (intra_model.first_sequence_header(es)[1] + 7) >> 3
    chunkings = [[]] + [[c for c in random_cuts(len(es), seed, mean) if c > h_end] for seed, mean in ((1, 300), (2, 4000))]
    bd = BatchDecoder(len(chunkings))
    for s, cuts in enumerate(chunkings):
        prev = 0
        for c in cuts + [len(es)]:
            bd.write(s, es[prev:c])
            prev = c
            # after every write the device's index is the model's of the bytes so far
            assert index_tuples(bd.intra_index(s)) == index_tuples(intra_model.intra_index(es[:c])), (name, s, c)
        assert index_tuples(bd.intra_index(s)) == want
    assert bd.last_error() is None
    bd.close()


def test_a_tail_picture_appears_once_its_closing_code_arrives():
    es = synth_es.make_case("i_only_320x240")
    last = intra_model.intra_index(es)[-1]
    bd = BatchDecoder(1)
    bd.write(0, es[:last["close"] + 3])
    assert last["picture"] not in [e["picture"] for e in bd.intra_index(0)]
    with pytest.raises(ValueError):  # not listed: refused
        bd.decode_intra([(0, last["picture"])])
    bd.write(0, es[last["close"] + 3:last["close"] + 4])
    assert bd.intra_index(0)[-1]["picture"] == last["picture"]
    got = bd.decode_intra([(0, last["picture"])])[0]
    assert np.array_equal(host(got), oracle_fresh(es, last))
    bd.close()


def _decode_all_listed(es, what, **kw):
    bd = BatchDecoder(1, **kw)
    bd.write(0, es)
    entries = bd.intra_index(0)
    got = bd.decode_intra([(0, e["picture"]) for e in entries])
    model = intra_model.intra_index(es)
    assert index_tuples(entries) == index_tuples(model)
    for e, t in zip(model, got):
        assert np.array_equal(host(t), oracle_fresh(es, e)), (what, e["picture"])
    assert all(i["error"] == 0 for i in bd.last_intra_info), what
    assert bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("slice_walk", [0, 1])
@pytest.mark.parametrize("name", CORPUS)
def test_every_listed_picture_equals_the_fresh_oracle(name, slice_walk):
    _decode_all_listed(stream(name), name, slice_walk=slice_walk)


def test_program_stream_through_write_ps():
    import gen_streams
    data = gen_streams.make_clip_ps(320, 240, 24, form="mpg")
    m1v = gen_streams.make_clip_m1v(320, 240, 24)
    bd = BatchDecoder(1)
    _, pes = bd.write_ps(0, data)
    entries = bd.intra_index(0)
    assert index_tuples(entries) == index_tuples(intra_model.intra_index(m1v)) and len(entries) == 2
    offsets = [o for o, _ in pes]
    for e in entries:  # the PTS of the last PES packet that starts at or before the picture (decoder.js:36-47)
        j = max(i for i, o in enumerate(offsets) if o <= e["byte_pos"]) if offsets[0] <= e["byte_pos"] else None
        assert e["pts"] == (pes[j][1] if j is not None else None)
    assert entries[1]["pts"] is not None and entries[1]["pts"] > entries[0]["pts"]
    got = bd.decode_intra([(0, e["picture"]) for e in entries])
    for e, t in zip(intra_model.intra_index(m1v), got):
        assert np.array_equal(host(t), oracle_fresh(m1v, e))
    bd.reset()  # forgets the PES table with the bytes
    bd.write(0, m1v)
    assert [e["pts"] for e in bd.intra_index(0)] == [None, None]
    bd.close()


def test_mixed_sizes_shuffled_over_many_streams_in_one_call():
    clips = [ffmpeg_es(320, 240, 24, seed) for seed in (1, 2, 3)] + [ffmpeg_es(1280, 720, 24, seed) for seed in (4, 5, 6)]
    clips += [ffmpeg_es(1920, 1080, 24, seed) for seed in (7, 8)] + [synth_es.make_case("odd_size")]
    bd = BatchDecoder(len(clips))
    for s, es in enumerate(clips):
        bd.write(s, es)
    reqs = [(s, e["picture"]) for s in range(len(clips)) for e in bd.intra_index(s)]
    reqs.append(reqs[3])  # the same picture twice
    random.Random(7).shuffle(reqs)
    got = bd.decode_intra(reqs)
    model = [{e["picture"]: e for e in intra_model.intra_index(es)} for es in clips]
    for (s, k), t in zip(reqs, got):
        assert t.numel() == bd.stream_info(s)["coded_size"] * 3 // 2
        assert np.array_equal(host(t), oracle_fresh(clips[s], model[s][k])), (s, k)
    y, cr, cb = planes_view(got[0], bd.stream_info(reqs[0][0]))
    info = bd.stream_info(reqs[0][0])
    assert y.shape == ((info["height"] + 15) // 16 * 16, (info["width"] + 15) // 16 * 16) and cr.shape == cb.shape
    assert y.data_ptr() == got[0].data_ptr()
    bd.close()


def test_slot_pressure_gives_the_same_bytes():
    clips = [synth_es.make_case("i_only_320x240"), synth_es.make_case("rows_ip"), ffmpeg_es(320, 240, 24)]
    bd = BatchDecoder(len(clips), max_slots=2)
    for s, es in enumerate(clips):
        bd.write(s, es)
    reqs = [(s, e["picture"]) for s in range(len(clips)) for e in bd.intra_index(s)]
    reqs = reqs + reqs[::2]
    assert len(reqs) >= 20
    bd.decode(2)  # the look-ahead holds slots too
    got = bd.decode_intra(reqs)
    model = [{e["picture"]: e for e in intra_model.intra_index(es)} for es in clips]
    for (s, k), t in zip(reqs, got):
        assert np.array_equal(host(t), oracle_fresh(clips[s], model[s][k])), (s, k)
    bd.close()


def _damage(es, entries, seed, flips=6):
    """Bit flips inside the listed pictures' slice data that neither make nor break a start code."""
    rng = random.Random(seed)
    buf = bytearray(es)
    for e in entries:
        for _ in range(flips):
            at = rng.randrange(e["byte_pos"] + 12, e["close"] - 2)  # (behind the picture header and the slice code)
            window = bytes(buf[at - 3:at + 4])
            buf[at] ^= 1 << rng.randrange(8)
            if intra_model.prefixes(bytes(buf[at - 3:at + 4])) != intra_model.prefixes(window):
                buf[at] ^= window[3] ^ buf[at]  # it would make or break a start code: undone
    return bytes(buf)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_damaged_pictures_equal_the_devices_own_fresh_decode(seed):
    clean = ffmpeg_es(320, 240, 24) + synth_es.make_case("i_only_320x240")[-4:]  # end code: the last I picture closes
    damaged = _damage(clean, intra_model.intra_index(clean), seed)
    entries = intra_model.intra_index(damaged)
    assert index_tuples(entries) == index_tuples(intra_model.intra_index(clean))
    bd = BatchDecoder(1)
    bd.write(0, damaged)
    got = bd.decode_intra([(0, e["picture"]) for e in entries])
    info = bd.last_intra_info
    for e, t, i in zip(entries, got, info):
        planes, _, parse_errors = gpu_fresh(damaged, e)
        assert np.array_equal(host(t), planes), (seed, e["picture"])
        assert (i["error"] == 1) == (parse_errors == 1), (seed, e["picture"], i)
    assert any(i["error"] for i in info)
    assert bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("name", ["odd_size", "random_slices_gaps", "ffmpeg_320x240", "ffmpeg_1280x720"])
def test_rgba_equals_a_fresh_single_picture_decode(name):
    es = stream(name)
    bd = BatchDecoder(1)
    bd.write(0, es)
    entries = bd.intra_index(0)
    got = bd.decode_intra([(0, e["picture"]) for e in entries], rgba=True)
    info = bd.stream_info(0)
    for e, (planes, image) in zip(intra_model.intra_index(es), got):
        want_planes, want_image, _ = gpu_fresh(es, e, rgba=True)
        assert tuple(image.shape) == (info["height"], info["width"], 4)
        assert np.array_equal(host(planes), want_planes) and np.array_equal(host(image), want_image), (name, e["picture"])
    bd.close()


def _state(bd, s):
    return (bd.get_index(s), bd.last_picture(s), [p.copy() for p in bd.host_planes(s)], bd.read_planes(s), bd.stats())


def _assert_same_state(a, b):
    assert a[0] == b[0] and a[1] == b[1] and a[4] == b[4]
    for x, y in zip(a[2] + list(a[3]), b[2] + list(b[3])):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("decode_b", [False, True])
def test_decode_state_is_untouched(decode_b):
    """Decode part of a clip, take all its I pictures, decode the rest: the sequential pictures are the reference's."""
    packets = helpers.clip_packets(320, 240, 24)
    es = b"".join(p for _, p in packets)
    bd = BatchDecoder(2, decode_b=decode_b)
    bd.write(0, es)
    bd.write(1, synth_es.make_case("rows_ip"))
    frames = []
    for _ in range(7):
        assert bd.decode(1, OUT_HOST)
        frames.append(tuple(p.copy() for p in bd.read_planes(0)))
    before = _state(bd, 0)
    reqs = [(s, e["picture"]) for s in (0, 1) for e in bd.intra_index(s)]
    got = bd.decode_intra(reqs)
    _assert_same_state(before, _state(bd, 0))
    assert np.array_equal(host(got[0]), oracle_fresh(es, intra_model.intra_index(es)[0]))
    while bd.decode(1, OUT_HOST):
        if len(frames) < 24:
            frames.append(tuple(p.copy() for p in bd.read_planes(0)))
    want = helpers.reference_decode(packets, "whole")["fnv1a64"]
    assert helpers.frame_hashes(frames) == want
    bd.close()


def test_b_picture_stream_state_is_untouched_with_decode_b():
    es = synth_es.make_case("b_rows")
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(1)
    try:
        exp, _, od = helpers.decode_all(lib, [(0, es)])
        od.destroy()
    finally:
        lib.oracle_set_decode_b(0)
    bd = BatchDecoder(1, decode_b=True)
    bd.write(0, es)
    got = []
    for k in range(len(exp)):
        assert bd.decode(1, OUT_HOST)
        got.append(tuple(p.copy() for p in bd.read_planes(0)))
        if k == 4:
            before = _state(bd, 0)
            bd.decode_intra([(0, e["picture"]) for e in bd.intra_index(0)])
            _assert_same_state(before, _state(bd, 0))
    helpers.assert_frames_equal(got, exp, "b_rows with decode_intra in between")
    bd.close()


def test_invalid_requests_are_refused_and_change_nothing():
    es = synth_es.make_case("rows_ip")  # I P P P I ...
    model = intra_model.intra_index(es)
    cut = es[:model[-1]["close"] + 2]  # the last I picture is not closed yet
    bd = BatchDecoder(2)
    bd.write(0, cut)
    bd.write(1, es[intra_model.first_sequence_header(es)[0] + 4:])  # no sequence header
    assert bd.decode(1, OUT_HOST)
    before = _state(bd, 0)
    listed = [e["picture"] for e in bd.intra_index(0)]
    assert listed == [e["picture"] for e in model[:-1]]
    first = bd.decode_intra([(0, listed[0])])[0]
    mark = first.clone().fill_(7)

    def call(reqs, dsts, flags=0, rgba=None):
        n = len(reqs)
        return bd.lib.jsmpeg_b200_batch_decode_intra(
            bd.handle, n, (ctypes.c_int * n)(*[s for s, _ in reqs]), (ctypes.c_uint32 * n)(*[p for _, p in reqs]),
            (ctypes.c_void_p * n)(*dsts), rgba, flags, None, None)

    # with a valid request in front: a P picture, the unclosed tail picture, a stream without a sequence header, no stream
    for stream, pic in ((0, 1), (0, model[-1]["picture"]), (1, 0), (2, 0)):
        assert call([(0, listed[0]), (stream, pic)], [mark.data_ptr(), first.data_ptr()]) == -2, (stream, pic)
        with pytest.raises(ValueError):
            bd.decode_intra([(0, listed[0]), (stream, pic)])
    assert call([(0, listed[0])], [None]) == -2                                  # NULL destination
    assert call([(0, listed[0])], [mark.data_ptr() + 1]) == -2                   # misaligned destination
    assert call([(0, listed[0])], [mark.data_ptr()], flags=OUT_RGBA) == -2       # RGBA without RGBA destinations
    assert bool((mark == 7).all())
    _assert_same_state(before, _state(bd, 0))
    assert bd.last_error() is None
    assert np.array_equal(host(first), oracle_fresh(es, model[0]))
    while bd.decode(1, OUT_HOST):
        pass
    bd.close()
