"""decode() takes a wave's picture infos to the host behind the walks alone and consumes them, and queues every reconstruct
step, while the wave's expand (stage 1b) is still running (jsmpeg_b200/csrc/engine.cu: parse_wave with early_infos).
What the synchronous stage 1 gave for free is now an ordering between streams: no step may start before the expand
has ended, a record slot released during consumption must not be walked again before the expand of the wave that held
it, and the next wave's task list must not overwrite one a queued expand still reads.

Ordinary calls only, planes against the oracle: ragged streams of three picture sizes in waves of more than 64 x 8
lane-walk pictures (which stage 1 forks into 8 size groups), slot pools so small that a call takes several rounds, a
look-ahead beyond what a call consumes, every output kind, the three walk kernels in one wave, and other calls between
two decode() calls on the same batch.
"""
import numpy as np
import pytest

import helpers
from helpers import assert_frames_equal, clip_packets, decode_all
from jsmpeg_b200.batch import OUT_DEVICE, OUT_HOST, OUT_RGBA, BatchDecoder
from test_b_pictures import natural_clip
from test_gpu_parity import _canvas2d_rgba

pytestmark = pytest.mark.gpu

# (width, height, pictures, copies): 480 + 400 + 24 = 904 pictures, ragged in size and in length
SHAPES = [(320, 240, 12, 40), (176, 144, 20, 20), (640, 480, 6, 4)]


def es_of(width, height, pictures):
    return b"".join(p for _, p in clip_packets(width, height, pictures))


_expected = {}


def oracle_frames(es, decode_b=False):
    """The oracle's pictures of `es` in decode() order (each distinct stream decoded once)"""
    key = (es, decode_b)
    if key not in _expected:
        lib = helpers.oracle_lib()
        lib.oracle_set_decode_b(1 if decode_b else 0)
        try:
            frames, _, d = decode_all(lib, [(0, es)])
            d.destroy()
        finally:
            lib.oracle_set_decode_b(0)
        _expected[key] = frames
    return _expected[key]


def ragged_batch(**kw):
    data = []
    for w, h, n, copies in SHAPES:
        data += [es_of(w, h, n)] * copies
    # (interleaved, so that a wave's size order, stream order and step order all differ)
    data = data[::3] + data[1::3] + data[2::3]
    bd = BatchDecoder(len(data), **kw)
    for i, es in enumerate(data):
        bd.write(i, es)
    return bd, data


def check_latest(bd, data, done, flags, what, decode_b=False):
    """Every stream's latest picture is the oracle's picture done[i] - 1, in the output `flags` asks for"""
    for i, es in enumerate(data):
        frames = oracle_frames(es, decode_b)
        if not 0 < done[i] <= len(frames):
            continue
        exp = frames[done[i] - 1]
        got = bd.host_planes(i) if flags & OUT_HOST else bd.read_planes(i)
        assert_frames_equal([got], [exp], f"{what}: stream {i} picture {done[i] - 1}")
        if flags & OUT_RGBA:
            info = bd.stream_info(i)
            assert np.array_equal(bd.read_rgba(i), _canvas2d_rgba(*exp, info["width"], info["height"])), (what, i)


def run_calls(bd, data, calls, flags, what, decode_b=False):
    """decode(n) for every n of `calls`, then to the end; after each call every stream's latest picture is checked"""
    lengths = [len(oracle_frames(es, decode_b)) for es in data]
    done = [0] * len(data)
    for n in list(calls) + [max(lengths)]:
        got = bd.decode(n, flags)
        new = [min(d + n, m) for d, m in zip(done, lengths)]
        assert got == sum(new) - sum(done), (what, n, got)
        done = new
        check_latest(bd, data, done, flags, f"{what} after decode({n})", decode_b)
    assert done == lengths and bd.decode(1, flags) == 0
    st = bd.stats()
    assert st["parse_errors"] == 0 and bd.last_error() is None
    return st


@pytest.mark.parametrize("flags", [OUT_DEVICE, OUT_HOST, OUT_RGBA])
@pytest.mark.parametrize("max_slots,lookahead", [(0, 1), (600, 1), (0, 16), (700, 16)])
def test_ragged_streams_in_forked_waves(max_slots, lookahead, flags):
    """Calls of 1, 2, 3 and 7 pictures, then the rest.  max_slots 0: one forked wave per call as far as the look-ahead
    does not already hold the pictures; 600 or 700 slots for 64 streams: several rounds per call, every one a forked wave
    into slots the round before released, with lookahead 16 also into slots of look-ahead pictures no step took."""
    bd, data = ragged_batch(max_slots=max_slots)
    bd.set_option("lookahead", lookahead)
    st = run_calls(bd, data, [1, 2, 3, 7], flags, f"max_slots={max_slots} lookahead={lookahead} flags={flags}")
    assert st["pictures"] == sum(n * c for _, _, n, c in SHAPES)
    assert st["lane_walk_pictures"] >= st["pictures"]
    bd.close()


def test_picture_by_picture_out_of_a_long_look_ahead():
    """decode(1) throughout with a look-ahead of 20: the first call walks and expands 904 pictures and reconstructs 64;
    every later step takes pictures an earlier call's wave expanded."""
    bd, data = ragged_batch()
    bd.set_option("lookahead", 20)
    run_calls(bd, data, [1] * 20, OUT_DEVICE, "picture by picture")
    bd.close()


@pytest.mark.parametrize("slice_walk", [0, 1])
def test_three_walk_kernels_in_one_wave(slice_walk):
    """One-slice I/P clips (lane-parallel walk, a forked wave) beside row-sliced clips with B pictures: the B pictures go
    to the B walk and, with slice_walk, the row-sliced I/P pictures to the slice walk, each with an expand of its own on
    a side stream that the steps wait for as well."""
    b_es = natural_clip()[0]
    data = [es_of(320, 240, 12)] * 48 + [b_es] * 6 + [es_of(176, 144, 20)] * 4
    bd = BatchDecoder(len(data), decode_b=1, slice_walk=slice_walk)
    for i, es in enumerate(data):
        bd.write(i, es)
    run_calls(bd, data, [1, 4, 2], OUT_RGBA, f"slice_walk={slice_walk}", decode_b=True)
    bd.close()


def test_other_calls_between_two_decode_calls():
    """decode(5), then decode_pictures (a wave of its own, complete when its infos arrive, into the slots decode() released and
    beside the ones its look-ahead holds), then a rewind and the whole decode again: the same pictures as the oracle's."""
    bd, data = ragged_batch(max_slots=1000)
    bd.set_option("lookahead", 8)
    lengths = [len(oracle_frames(es)) for es in data]
    assert bd.decode(5, OUT_DEVICE) == 5 * len(data)
    check_latest(bd, data, [5] * len(data), OUT_DEVICE, "decode(5)")
    reqs = [(s, e["picture"]) for s in range(0, len(data), 7) for e in bd.picture_index(s)]
    for (s, pic), t in zip(reqs, bd.decode_pictures(reqs)):
        exp = oracle_frames(data[s])[pic]
        assert np.array_equal(t.cpu().numpy(), np.concatenate(exp)), ("decode_pictures", s, pic)
    assert bd.decode(1, OUT_DEVICE) == len(data)  # decode() goes on where it was
    check_latest(bd, data, [6] * len(data), OUT_DEVICE, "decode(1) after decode_pictures")
    bd.rewind()
    assert bd.decode(3, OUT_HOST) == 3 * len(data)
    check_latest(bd, data, [3] * len(data), OUT_HOST, "decode(3) after rewind")
    assert bd.decode(100, OUT_DEVICE) == sum(lengths) - 3 * len(data)
    check_latest(bd, data, lengths, OUT_DEVICE, "the rest after rewind")
    assert bd.last_error() is None
    bd.close()
