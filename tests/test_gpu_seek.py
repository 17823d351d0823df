"""Seeking decode() (jsmpeg_b200_batch_seek_pictures) against the batch's own sequential decode() on clean streams, and
against the device's own fresh decoder fed the seek bytes (tools/chain_model.py seek_bytes) and continued on gappy
and damaged ones: the state right after the seek and after every later decode(), many streams in one call with some
left alone, the output flags, slot pressure, interplay with writes and the other random-access calls, invalid
requests, and the reconstruct launches of a 64-stream seek."""
import ctypes
import functools
import random
import re
from collections import Counter

import numpy as np
import pytest

import chain_model
import intra_model
import synth_es
from jsmpeg_b200.batch import OUT_HOST, OUT_RGBA, BatchDecoder
from test_gpu_intra import CORPUS, _assert_same_state, _damage, _state, ffmpeg_es
from test_gpu_pictures import B_CORPUS, MIXED, _skipping_cut, stream
from test_seek_model import seek_run

pytestmark = pytest.mark.gpu


def snapshot(bd, s, flags=0, delta=0):
    """What decode() observes of stream s: (bit index + 8 * delta, last_picture, Y | Cr | Cb, RGBA under OUT_RGBA)."""
    return (bd.get_index(s) + 8 * delta, bd.last_picture(s), np.concatenate(bd.read_planes(s)),
            bd.read_rgba(s) if flags & OUT_RGBA else None)


def assert_same(a, b, what):
    assert a[0] == b[0] and a[1] == b[1], (what, a[:2], b[:2])
    assert np.array_equal(a[2], b[2]), what
    assert (a[3] is None) == (b[3] is None) and (a[3] is None or np.array_equal(a[3], b[3])), what


def device_sequential(es, decode_b=False, flags=0):
    """The device's decode() of `es` from the start: [(start code position of the consumed picture, snapshot)]."""
    bd = BatchDecoder(1, decode_b=decode_b)
    bd.write(0, es)
    pics = chain_model.picture_positions(es)
    steps = []
    while True:
        at = (bd.get_index(0) + 7) >> 3
        if bd.decode(1, flags) != 1:
            break
        steps.append((next(p for p in pics if p >= at), snapshot(bd, 0, flags)))
    bd.close()
    return steps


@functools.lru_cache(maxsize=None)
def sequential(name, decode_b):
    return device_sequential(stream(name), decode_b)


def gpu_fresh_run(es, entry, decode_b=False, flags=0):
    """The device's own decode() of chain_model.seek_bytes(es, entry) in a new batch: (status, [snapshot right after
    the decode() that consumes picture k -- or, when it never does, after the last one before -- and after every
    later decode()]), translated to the positions of `es`."""
    data = chain_model.seek_bytes(es, entry, decode_b)
    delta = len(es) - len(data)
    target = entry["byte_pos"] - delta
    starts = chain_model.picture_positions(data)
    bd = BatchDecoder(1, decode_b=decode_b)
    bd.write(0, data)
    status = 0
    while True:
        at = (bd.get_index(0) + 7) >> 3
        nxt = next((p for p in starts if p >= at), None)
        if nxt is None or nxt > target:
            break
        assert bd.decode(1, flags) == 1
        if nxt == target:
            status = 1
            break
    run = [snapshot(bd, 0, flags, delta)]
    while bd.decode(1, flags) == 1:
        run.append(snapshot(bd, 0, flags, delta))
    bd.close()
    return status, run


def assert_goes_on_as(bd, s, run, flags, what):
    """Stream s of `bd` (alone in its batch) shows run[0] now and run[1:] after each later decode()."""
    assert_same(snapshot(bd, s, flags), run[0], what)
    for i, want in enumerate(run[1:]):
        assert bd.decode(1, flags) == 1, (what, i)
        assert_same(snapshot(bd, s, flags), want, (what, i))
    assert bd.decode(1, flags) == 0, what


@functools.lru_cache(maxsize=None)
def clean_entries(name, decode_b):
    """The listed pictures of a corpus stream after which a seek must go on exactly as sequential decode(): the
    stream starts with an I picture and every picture from the seek chain start on codes every macroblock (by the
    oracle)."""
    es = stream(name)
    if chain_model.picture_type(es, chain_model.picture_positions(es)[0]) != 1:
        return frozenset()
    return frozenset(e["picture"] for e in chain_model.picture_index(es, decode_b) if seek_run(es, e, decode_b)[1])


@pytest.mark.parametrize("slice_walk", [0, 1])
@pytest.mark.parametrize("decode_b", [False, True])
@pytest.mark.parametrize("name", CORPUS + B_CORPUS)
def test_seek_goes_on_as_the_sequential_decode(name, decode_b, slice_walk):
    es = stream(name)
    seq = sequential(name, decode_b)
    step_of = {pos: i for i, (pos, _) in enumerate(seq)}
    clean = clean_entries(name, decode_b)
    bd = BatchDecoder(1, decode_b=decode_b, slice_walk=slice_walk)
    bd.write(0, es)
    entries = bd.picture_index(0)
    assert [e["picture"] for e in entries] == [e["picture"] for e in chain_model.picture_index(es, decode_b)]
    if len(entries) > 12:
        entries = random.Random(len(es)).sample(entries, 12)
    checked = 0
    for n, e in enumerate(entries):
        bd.decode(n % 4)  # an arbitrary state before the seek
        assert bd.seek_pictures([(0, e["picture"])]) == 1
        assert bd.last_seek_info[0]["status"] == 1, (name, e["picture"])
        if e["picture"] not in clean:
            continue
        at = step_of[e["byte_pos"]]
        assert bd.last_seek_info[0]["n_present"] == seq[at][1][2].size * 2 // 3 // 256
        assert_goes_on_as(bd, 0, [snap for _, snap in seq[at:]], 0, (name, e["picture"]))
        checked += 1
    if name in ("rows_ip", "ffmpeg_320x240", "ffmpeg_1920x1080", "b_rows", "open_gop"):
        assert checked == len(entries) > 0, name
    assert bd.last_error() is None
    bd.close()


def damaged_streams():
    clean = ffmpeg_es(320, 240, 24) + synth_es.make_case("i_only_320x240")[-4:]  # end code: the last picture closes
    damaged = _damage(clean, chain_model.picture_index(clean)[::3], 1)
    cut, skipped = _skipping_cut(damaged, chain_model.picture_positions(damaged))
    return [("random_slices_gaps", synth_es.make_case("random_slices_gaps"), None), ("damaged", damaged, None),
            ("cut", cut, skipped + 1)]


@pytest.mark.parametrize("flags", [0, OUT_RGBA])
def test_gappy_and_damaged_streams_equal_the_devices_own_fresh_decoder(flags):
    zero_status = 0
    for name, es, never in damaged_streams():
        bd = BatchDecoder(1)
        bd.write(0, es)
        for e in chain_model.picture_index(es):
            bd.decode(2)
            assert bd.seek_pictures([(0, e["picture"])], flags) == 1
            status, run = gpu_fresh_run(es, e, False, flags)
            assert bd.last_seek_info[0]["status"] == status, (name, e["picture"])
            assert status == 0 or e["picture"] != never, (name, e["picture"])
            zero_status += status == 0
            assert_goes_on_as(bd, 0, run, flags, (name, e["picture"]))
        assert bd.last_error() is None
        bd.close()
    assert zero_status >= 1


def test_many_streams_in_one_call_leave_the_others_alone():
    streams = [stream(name) for name in MIXED] * 2
    bd, twin = BatchDecoder(len(streams), decode_b=True), BatchDecoder(len(streams), decode_b=True)
    for s, es in enumerate(streams):
        bd.write(s, es)
        twin.write(s, es)
    bd.decode(2)
    twin.decode(2)
    rng = random.Random(3)
    named = sorted(rng.sample(range(len(streams)), len(streams) // 2 + 1))
    reqs = {s: rng.choice(bd.picture_index(s))["picture"] for s in named}
    before = {s: _state(bd, s) for s in range(len(streams)) if s not in reqs}
    order = list(reqs.items())
    rng.shuffle(order)
    assert bd.seek_pictures(order) == len(order)
    assert all(i["status"] == 1 for i in bd.last_seek_info)
    runs = {}
    for s, k in reqs.items():
        e = next(e for e in chain_model.picture_index(streams[s], True) if e["picture"] == k)
        runs[s] = gpu_fresh_run(streams[s], e, True)[1]
        assert_same(snapshot(bd, s), runs[s][0], (s, k))
    for s, st in before.items():
        _assert_same_state(st, _state(bd, s))
    # every stream on: the named ones as their fresh decoders, the others as the twin that never sought
    step = {s: 0 for s in reqs}
    while bd.decode(1) | twin.decode(1):
        for s in range(len(streams)):
            if s in reqs:
                if step[s] + 1 < len(runs[s]) and bd.get_index(s) != runs[s][step[s]][0]:
                    step[s] += 1
                    assert_same(snapshot(bd, s), runs[s][step[s]], (s, step[s]))
            else:
                assert_same(snapshot(bd, s), snapshot(twin, s), s)
    assert all(step[s] == len(runs[s]) - 1 for s in reqs)
    bd.close()
    twin.close()


@pytest.mark.parametrize("name,decode_b", [("ffmpeg_320x240", False), ("b_rows", True), ("open_gop", True)])
def test_flags_host_ring_and_rgba(name, decode_b):
    es = stream(name)
    bd = BatchDecoder(1, decode_b=decode_b)
    bd.write(0, es)
    for e in bd.picture_index(0):
        k = e["picture"]
        bd.decode(3, OUT_HOST)  # the seek follows a decode() whose host copies were just queued
        assert bd.seek_pictures([(0, k)], OUT_HOST | OUT_RGBA) == 1
        planes, image = bd.decode_pictures([(0, k)], rgba=True)[0]
        device = np.concatenate(bd.read_planes(0))
        assert np.array_equal(device, planes.cpu().numpy()), (name, k)
        assert np.array_equal(np.concatenate([p.copy() for p in bd.host_planes(0)]), device), (name, k)
        assert np.array_equal(bd.read_rgba(0), image.cpu().numpy()), (name, k)
    bd.close()


def test_slot_pressure_and_chain_groups_give_the_same_bytes():
    """Three record slots for four chains of up to 12 pictures: several waves per chain, several chain groups."""
    names = ["ffmpeg_320x240", "rows_ip", "b_rows", "open_gop"]
    outs = []
    for max_slots in (0, 3):
        bd = BatchDecoder(len(names), max_slots=max_slots, decode_b=True)
        for s, name in enumerate(names):
            bd.write(s, stream(name))
        bd.decode(2)  # the look-ahead holds slots too
        got = []
        for rnd in range(3):
            reqs = [(s, bd.picture_index(s)[-1 - rnd]["picture"]) for s in range(len(names))]
            assert bd.seek_pictures(reqs, OUT_RGBA) == len(names)
            got.append([snapshot(bd, s, OUT_RGBA) for s in range(len(names))])
            bd.decode(1, OUT_RGBA)
            got.append([snapshot(bd, s, OUT_RGBA) for s in range(len(names))])
        outs.append(got)
        bd.close()
    for a, b in zip(*outs):
        for x, y in zip(a, b):
            assert_same(x, y, "slot pressure")


def test_seek_then_write_more_then_decode():
    es = stream("ffmpeg_320x240")
    seq = sequential("ffmpeg_320x240", False)
    entries = chain_model.picture_index(es)
    half = entries[len(entries) // 2]["close"] + 4
    bd = BatchDecoder(1)
    bd.write(0, es[:half])
    listed = bd.picture_index(0)
    k = next(e for e in reversed(listed) if e["type"] == 2)
    assert bd.seek_pictures([(0, k["picture"])]) == 1
    bd.write(0, es[half:])
    at = [pos for pos, _ in seq].index(k["byte_pos"])
    assert_goes_on_as(bd, 0, [snap for _, snap in seq[at:]], 0, "write after seek")
    bd.close()


@pytest.mark.parametrize("name,decode_b", [("ffmpeg_320x240", False), ("open_gop", True)])
def test_other_random_access_calls_leave_the_sought_state_alone(name, decode_b):
    es = stream(name)
    seq = sequential(name, decode_b)
    bd = BatchDecoder(1, decode_b=decode_b)
    bd.write(0, es)
    entries = bd.picture_index(0)
    k = entries[len(entries) // 2]
    assert bd.seek_pictures([(0, k["picture"])], OUT_HOST) == 1
    before = _state(bd, 0)
    bd.decode_pictures([(0, e["picture"]) for e in entries])
    bd.decode_accumulated([(0, e["picture"]) for e in entries if e["type"] != 3])
    _assert_same_state(before, _state(bd, 0))
    at = [pos for pos, _ in seq].index(k["byte_pos"])
    assert_goes_on_as(bd, 0, [snap for _, snap in seq[at:]], 0, name)
    bd.close()


def test_program_stream_through_write_ps():
    import gen_streams
    data = gen_streams.make_clip_ps(320, 240, 24, form="mpg")
    m1v = gen_streams.make_clip_m1v(320, 240, 24)
    seq = device_sequential(m1v)
    bd = BatchDecoder(1)
    bd.write_ps(0, data)
    entries = bd.picture_index(0)
    assert [e["byte_pos"] for e in entries] == [e["byte_pos"] for e in chain_model.picture_index(m1v)]
    for e in entries[1::5]:
        assert bd.seek_pictures([(0, e["picture"])]) == 1
        at = [pos for pos, _ in seq].index(e["byte_pos"])
        assert_goes_on_as(bd, 0, [snap for _, snap in seq[at:]], 0, e["picture"])
    bd.close()


def test_invalid_requests_are_refused_and_change_nothing():
    es = synth_es.make_case("b_rows")  # I B B P B B I B B P B B I
    model = chain_model.picture_index(es, True)
    cut = es[:model[-1]["close"] + 2]  # the last I picture is not closed yet
    bd = BatchDecoder(2, decode_b=True)
    bd.write(0, cut)
    bd.write(1, es[intra_model.first_sequence_header(es)[0] + 4:])  # no sequence header
    assert bd.decode(2, OUT_HOST)
    before = _state(bd, 0)

    def call(reqs):
        n = len(reqs)
        return bd.lib.jsmpeg_b200_batch_seek_pictures(bd.handle, n, (ctypes.c_int * n)(*[s for s, _ in reqs]),
                                                      (ctypes.c_uint32 * n)(*[p for _, p in reqs]), 0, None, None, None)

    # with a valid request in front: the same stream twice, a B picture without a chain start, the unclosed tail, no
    # sequence header, no stream, no picture
    for stream_, pic in ((0, 3), (0, 1), (0, model[-1]["picture"]), (1, 0), (2, 0), (-1, 0), (0, 99)):
        assert call([(0, 4), (stream_, pic)]) == -2, (stream_, pic)
        with pytest.raises(ValueError):
            bd.seek_pictures([(0, 4), (stream_, pic)])
    assert bd.lib.jsmpeg_b200_batch_seek_pictures(bd.handle, 1, None, None, 0, None, None, None) == -2
    assert bd.lib.jsmpeg_b200_batch_seek_pictures(bd.handle, -1, None, None, 0, None, None, None) == -2
    assert call([]) == 0
    _assert_same_state(before, _state(bd, 0))
    assert bd.last_error() is None
    bd.close()


def test_a_64_stream_seek_issues_one_reconstruct_launch_per_depth():
    import torch
    from torch.profiler import ProfilerActivity, profile
    es = ffmpeg_es(320, 240, 24)
    entries = [e for e in chain_model.picture_index(es) if e["type"] == 2]
    bd = BatchDecoder(64)
    for s in range(64):
        bd.write(s, es)
    rng = random.Random(11)
    reqs = [(s, rng.choice(entries)) for s in range(64)]
    depth = max(e["picture"] - e["chain_start"] for _, e in reqs)  # (every picture of these chains is decoded)
    bd.seek_pictures([(0, entries[0]["picture"])])  # warm-up
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        assert bd.seek_pictures([(s, e["picture"]) for s, e in reqs]) == 64
        torch.cuda.synchronize()
    kernels = Counter()
    for ev in prof.events():
        m = re.search(r"(reconstruct\w*_kernel)\(", ev.name)
        if ev.device_type == torch.autograd.DeviceType.CUDA and m:
            kernels[m.group(1)] += 1
    assert dict(kernels) == {"reconstruct_kernel": depth + 1}
    assert all(i["status"] == 1 for i in bd.last_seek_info)
    bd.close()
