"""MPEG program stream demux on the device (jsmpeg_b200_batch_write_ps) against the serial model
(tools/mini_ps.py): the ES bytes resident in HBM, the returned totals and the PES tables, on clean, hand-written
and damaged streams in any chunking; then decoded pictures against the oracle."""
import ctypes

import pytest

import helpers
import mini_ps
import ps_cases
from helpers import assert_frames_equal, decode_all
from jsmpeg_b200.batch import OUT_DEVICE, BatchDecoder

pytestmark = pytest.mark.gpu


def _feed(bd, stream, data, cuts):
    """write_ps `data` cut at `cuts`; returns (sum of the returned totals, PES table in 90 kHz ticks)."""
    total, pes, prev = 0, [], 0
    for c in list(cuts) + [len(data)]:
        n, p = bd.write_ps(stream, data[prev:c])
        total += n
        pes += [(o, round(t * 90000.0)) for o, t in p]
        prev = c
    return total, pes


def _check(data, chunkings, what):
    want_es, want_pes = mini_ps.demux_chunked(data, [])
    bd = BatchDecoder(len(chunkings))
    try:
        for s, cuts in enumerate(chunkings):
            total, pes = _feed(bd, s, data, cuts)
            got = bd.read_es(s)
            assert got == want_es, f"{what}, chunking {s}: ES differs ({len(got)} vs {len(want_es)} bytes)"
            assert total == len(want_es), (what, s)
            assert pes == want_pes, (what, s)
        assert bd.last_error() is None
    finally:
        bd.close()


def _corpus():
    out = [(f"tiny_{k}", v[0]) for k, v in sorted(ps_cases.TINY.items())]
    for name in sorted(ps_cases.WRITER):
        data, _ = ps_cases.writer_case(name)
        out.append((name, data))
        for kind in ("flips", "lengths", "garbage"):
            for seed in (11, 12):
                out.append((f"{name}_{kind}_{seed}", ps_cases.damaged(data, kind, seed)))
    return out


@pytest.mark.parametrize("name,data", _corpus(), ids=[n for n, _ in _corpus()])
def test_device_matches_model_whole_and_in_random_chunkings(name, data):
    chunkings = [[]] + [ps_cases.random_cuts(len(data), seed, mean=m) for seed, m in ((1, 300), (2, 2000), (3, 64))]
    _check(data, chunkings, name)


@pytest.mark.parametrize("name", sorted(ps_cases.TINY))
def test_hand_written_streams_in_one_byte_writes_and_cut_at_every_offset(name):
    """Every cut covers every offset inside each pack header and PES header."""
    data, want_es, want_pes = ps_cases.TINY[name]
    assert mini_ps.demux(data)[:2] == (want_es, want_pes)
    _check(data, [range(1, len(data))] + [[c] for c in range(1, len(data))], name)


def _decode_steps(bd, streams, exp_frames, what):
    n = 0
    while bd.decode(1, OUT_DEVICE):
        for s in streams:
            assert_frames_equal([bd.read_planes(s)], [exp_frames[n]], f"{what}: stream {s} picture {n}")
        n += 1
    assert n == len(exp_frames), what


@pytest.mark.parametrize("size,form", [((320, 240, 24), "mpg"), ((320, 240, 24), "vob"), ((1280, 720, 30), "vob"),
                                       ((1920, 1080, 60), "mpg")])
def test_ffmpeg_program_streams_decode_bit_exact(size, form):
    """FFmpeg's .mpg / .vob muxers: stream 0 written in one call, stream 1 in 64 KB chunks; the ES equals the raw
    .m1v of the same encode, the pictures and the bit index equal the oracle's."""
    import gen_streams
    w, h, n = size
    data = gen_streams.make_clip_ps(w, h, n, form=form)
    m1v = gen_streams.make_clip_m1v(w, h, n)
    exp_frames, exp_idx, od = decode_all(helpers.oracle_lib(), [(0, m1v)])
    bd = BatchDecoder(2)
    _feed(bd, 0, data, [])
    _feed(bd, 1, data, range(65536, len(data), 65536))
    assert bd.read_es(0) == m1v == bd.read_es(1)
    _decode_steps(bd, (0, 1), exp_frames, f"{form} {w}x{h}")
    assert bd.get_index(0) == exp_idx[-1] == bd.get_index(1)
    od.destroy()
    bd.close()


def test_ipb_clip_with_hostile_audio_decodes_b_pictures_bit_exact():
    """A tools/mini_enc.py I/P/B clip, muxed with audio packets whose payloads hold 00 00 01 BA / E0 / BB, decoded
    with the B-picture extension: the pictures equal the oracle's, the bit index that of the same ES written plainly."""
    import mini_enc
    es = mini_enc.make_b_clip(176, 144, 13)[0]
    data, _ = mini_ps.mux(es, form="mpg", packet=900, audio=600, padding=True, seed=9)
    assert mini_ps.demux(data)[0] == es
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(1)
    try:
        exp_frames, _, od = decode_all(lib, [(0, es)])
    finally:
        lib.oracle_set_decode_b(0)
    bd = BatchDecoder(2, decode_b=True)  # stream 1: the same ES written the ordinary way
    _feed(bd, 0, data, ps_cases.random_cuts(len(data), 4, mean=1000))
    bd.write(1, es)
    assert bd.read_es(0) == es
    _decode_steps(bd, (0, 1), exp_frames, "I/P/B in PS")
    assert bd.get_index(0) == bd.get_index(1)
    od.destroy()
    bd.close()


def test_write_ps_write_ts_and_write_give_the_same_pictures():
    import gen_streams
    from jsmpeg_b200 import ts
    w, h, n = 640, 480, 13
    m1v = gen_streams.make_clip_m1v(w, h, n)
    bd = BatchDecoder(3)
    bd.write_ps(0, gen_streams.make_clip_ps(w, h, n, form="vob"))
    bd.write_ts(1, gen_streams.make_clip_ts(w, h, n))
    bd.write(2, m1v)
    assert bd.read_es(0) == m1v == bd.read_es(1)
    assert b"".join(p for _, p in ts.demux_video_es(gen_streams.make_clip_ts(w, h, n))) == m1v
    steps = 0
    while bd.decode(1, OUT_DEVICE):
        planes = [bd.read_planes(s) for s in range(3)]
        assert_frames_equal(planes[:1], planes[2:], f"write_ps vs write, picture {steps}")
        assert_frames_equal(planes[1:2], planes[2:], f"write_ts vs write, picture {steps}")
        steps += 1
    assert steps == n
    bd.close()


def test_stream_id_outside_the_video_range_is_refused_and_the_batch_lives_on():
    data, want_es, _ = ps_cases.TINY["false_pack_in_audio"]
    bd = BatchDecoder(1)
    with pytest.raises(ValueError):
        bd.write_ps(0, data, stream_id=0x20)
    lib = bd.lib
    n = ctypes.c_int(5)
    assert lib.jsmpeg_b200_batch_write_ps(bd.handle, 0, data, len(data), 0xC0, None, None, 0, ctypes.byref(n)) == -2
    assert n.value == 0 and bd.last_error() is None and bd.read_es(0) == b""
    assert bd.write_ps(0, data)[0] == len(want_es)
    assert bd.read_es(0) == want_es
    bd.close()
