"""The residual of the playback path (decode() and seek_pictures with OUT_RESIDUALS, include/jsmpeg_b200.h) against
decode_residuals of the picture decode() reconstructed: every stream of the key-picture and B corpora with the slice walk
and decode_b on and off, an .mpg, damaged streams, decode(n) on streams that end in different steps, seeks, the other
output flags, launch counts and the bench's shape; and the flag moves nothing else."""
from collections import Counter

import numpy as np
import pytest

import chain_model
import synth_es
from jsmpeg_b200.batch import (OUT_ACCUMULATED, OUT_DEVICE, OUT_HOST, OUT_MACROBLOCKS, OUT_RESIDUALS, OUT_RGBA, BatchDecoder,
                               planes_view)
from test_gpu_intra import CORPUS, _damage, ffmpeg_es, host
from test_gpu_macroblocks import B_CORPUS, MIXED, stream

pytestmark = pytest.mark.gpu
ALL = OUT_HOST | OUT_RGBA | OUT_MACROBLOCKS | OUT_ACCUMULATED


def listed_residuals(bd, s):
    """{picture: host residual} of every picture decode_residuals lists for stream s, and {picture: error}"""
    pics = [e["picture"] for e in bd.macroblock_index(s)]
    got = bd.decode_residuals([(s, k) for k in pics])
    return ({k: host(t) for k, t in zip(pics, got)}, {k: i["error"] for k, i in zip(pics, bd.last_residuals_info)})


def step_through(bd, es, flags=OUT_RESIDUALS):
    """decode(1, flags) through stream 0 of `bd` (holding `es`): per picture decode() reconstructs, (bit index after
    it, picture number, residual read back, Y | Cr | Cb)."""
    starts = chain_model.picture_positions(es)
    out = []
    while True:
        at = (bd.get_index(0) + 7) >> 3
        before = bd.stats()["pictures_decoded"]
        if bd.decode(1, flags) != 1:
            return out
        if bd.stats()["pictures_decoded"] > before:
            k = next(i for i, p in enumerate(starts) if p >= at)
            out.append((bd.get_index(0), k, bd.read_residuals(0), np.concatenate(bd.read_planes(0))))


@pytest.mark.parametrize("name", CORPUS + B_CORPUS + ["mpg"])
def test_every_reconstructed_picture_equals_decode_residuals(name):
    import gen_streams
    es = gen_streams.make_clip_m1v(320, 240, 24) if name == "mpg" else stream(name)
    for slice_walk in (0, 1):
        for decode_b in (0, 1):
            bd = BatchDecoder(1, slice_walk=slice_walk, decode_b=decode_b)
            if name == "mpg":
                bd.write_ps(0, gen_streams.make_clip_ps(320, 240, 24, form="mpg"))
            else:
                bd.write(0, es)
            want, _ = listed_residuals(bd, 0)
            flags = OUT_RESIDUALS | (OUT_RGBA if slice_walk else 0)  # (the RGBA variants too)
            steps = step_through(bd, es, flags)
            compared = 0
            for _, k, got, _ in steps:
                if k in want:  # (an unclosed tail picture is not listed)
                    assert np.array_equal(got, want[k]), (name, k, slice_walk, decode_b)
                    compared += 1
            assert compared >= len(steps) - 1 and compared > 0, (name, slice_walk, decode_b)
            view = bd.device_residuals(0)
            assert view.is_cuda and tuple(view.shape) == steps[-1][2].shape
            assert np.array_equal(host(view), steps[-1][2])
            assert sum(p.numel() for p in planes_view(view, bd.stream_info(0))) == view.numel()
            assert bd.last_error() is None
            bd.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_damaged_streams(seed):
    """The walk that starts at k's start code on both paths: the same residual, pictures with errors among them."""
    import macroblock_model
    clean = ffmpeg_es(320, 240, 24) + synth_es.make_case("i_only_320x240")[-4:]  # end code: the last picture closes
    b_clean = synth_es.make_case("b_one_slice_fcodes")
    streams = [(_damage(clean, macroblock_model.macroblock_index(clean)[::3], seed), 0),
               (_damage(b_clean, macroblock_model.macroblock_index(b_clean)[1::2], seed, flips=3), 1)]
    errors = 0
    for es, decode_b in streams:
        bd = BatchDecoder(1, decode_b=decode_b)
        bd.write(0, es)
        want, error = listed_residuals(bd, 0)
        steps = step_through(bd, es)
        compared = 0
        for _, k, got, _ in steps:
            if k in want:
                assert np.array_equal(got, want[k]), (seed, decode_b, k)
                compared += 1
                errors += error[k] != 0
        assert compared >= max(5, len(steps) - 1), (seed, decode_b)
        assert bd.last_error() is None
        bd.close()
    assert errors > 0


def _sequence(name, decode_b):
    """step_through of `name` alone: [(bit index after, residual)] per reconstruction"""
    es = stream(name)
    bd = BatchDecoder(1, decode_b=decode_b)
    bd.write(0, es)
    out = [(at, res) for at, _, res, _ in step_through(bd, es)]
    bd.close()
    return out


def test_decode_n_stores_the_last_picture_of_each_stream():
    """decode(n, flag), n = 2 ... 6, on a batch whose streams end in different steps: each stream's residual is that of
    the last picture it reconstructed (named by the bit index), 0 before its first one."""
    seqs = [_sequence(name, 1) for name in MIXED]
    assert len({len(s) for s in seqs}) > 1  # (the streams end in different steps)
    bd = BatchDecoder(len(MIXED), decode_b=True)
    for s, name in enumerate(MIXED):
        bd.write(s, stream(name))
    calls = 0
    for n in [2, 3, 4, 5, 6] * 20:
        if not bd.decode(n, OUT_RESIDUALS):
            break
        calls += 1
        for s in range(len(MIXED)):
            at = bd.get_index(s)
            done = [res for idx, res in seqs[s] if idx <= at]
            got = bd.read_residuals(s)
            if done:
                assert np.array_equal(got, done[-1]), (MIXED[s], n, calls)
            else:
                assert not got.any()
    assert calls >= 5
    assert bd.last_error() is None
    bd.close()


def _observed(bd, n_streams):
    return [(bd.get_index(s), bd.last_picture(s), np.concatenate(bd.read_planes(s)),
             np.concatenate([p.copy() for p in bd.host_planes(s)]), bd.read_rgba(s), bd.read_macroblocks(s),
             bd.host_macroblocks(s).copy(), bd.read_accumulated(s)) for s in range(n_streams)]


def test_nothing_else_moves():
    """Planes, RGBA, host ring, entries, maps, bit index and last_picture after every call, and every stats field, are
    those of a twin batch without the flag (all other flags set, decode(n) for n > 1; a batch this small stays within
    every kernel's capacity, so kernel_launches agrees too)."""
    runs, stats = [], []
    for extra in (0, OUT_RESIDUALS):
        bd = BatchDecoder(len(MIXED), decode_b=True)
        for s, name in enumerate(MIXED):
            bd.write(s, stream(name))
        seen = []
        for n in [1, 3, 2, 5, 1, 4] * 6:
            got = bd.decode(n, ALL | extra)
            seen.append((got, _observed(bd, len(MIXED))))
            if not got:
                break
        runs.append(seen)
        stats.append(bd.stats())
        bd.close()
    assert len(runs[0]) == len(runs[1]) and runs[0][-1][0] == 0
    for (ga, a), (gb, b) in zip(*runs):
        assert ga == gb
        for x, y in zip(a, b):
            assert x[:2] == y[:2]
            for u, v in zip(x[2:], y[2:]):
                assert np.array_equal(u, v)
    off, on = stats
    for key in off:
        if not key.endswith("_ms"):
            assert on[key] == off[key], key


def test_all_flags_together_equal_decode_residuals():
    es = stream("b_clip_1280x720")
    bd = BatchDecoder(1, decode_b=1)
    bd.write(0, es)
    want, _ = listed_residuals(bd, 0)
    steps = step_through(bd, es, ALL | OUT_RESIDUALS)
    kinds = Counter()
    for _, k, got, _ in steps:
        if k in want:
            assert np.array_equal(got, want[k]), k
            kinds[k] += 1
    assert len(kinds) >= len(steps) - 1 > 5
    bd.close()


def test_residual_is_zero_before_the_flag_and_after_reset_and_calls_without_it_write_none():
    es = stream("ffmpeg_320x240")
    bd = BatchDecoder(2)
    bd.write(0, es)
    assert bd.decode(2) == 2
    assert not bd.read_residuals(0).any()
    assert bd.decode(1, OUT_RESIDUALS) == 1
    first = bd.read_residuals(0)
    assert first.any()
    assert bd.decode(2, OUT_DEVICE) == 2  # no flag: the residual stays that of picture 2
    assert np.array_equal(bd.read_residuals(0), first)
    bd.rewind()
    assert np.array_equal(bd.read_residuals(0), first)
    bd.reset()
    assert not bd.read_residuals(0).any() and not host(bd.device_residuals(0)).any()
    for s, call in ((1, bd.read_residuals), (1, bd.device_residuals), (2, bd.read_residuals), (-1, bd.device_residuals)):
        with pytest.raises(ValueError):
            call(s)
    for s in (1, 2, -1):
        assert bd.lib.jsmpeg_b200_batch_get_residuals(bd.handle, s, None) != 0
        assert bd.lib.jsmpeg_b200_batch_read_residuals(bd.handle, s, None) != 0
    assert bd.last_error() is None
    bd.close()


def _fresh_residuals(es, entry, decode_b):
    """The device's own decode() with OUT_RESIDUALS of chain_model.seek_bytes(es, entry) in a new batch: status and the
    residual right after the decode() that consumes picture k (or the last one before, when none does), then after
    every later decode()."""
    data = chain_model.seek_bytes(es, entry, decode_b)
    target = entry["byte_pos"] - (len(es) - len(data))
    starts = chain_model.picture_positions(data)
    bd = BatchDecoder(1, decode_b=decode_b)
    bd.write(0, data)
    status = 0
    while True:
        nxt = next((p for p in starts if p >= (bd.get_index(0) + 7) >> 3), None)
        if nxt is None or nxt > target:
            break
        assert bd.decode(1, OUT_RESIDUALS) == 1
        if nxt == target:
            status = 1
            break
    run = [bd.read_residuals(0)]
    while bd.decode(1, OUT_RESIDUALS) == 1:
        run.append(bd.read_residuals(0))
    bd.close()
    return status, run


def test_seek_with_the_flag():
    """Status 1 (clean streams, decode_b on and off) and status 0 (damaged and cut streams): the residual of the picture
    the state ends on, as the fresh decoder has it, and that of every decode() after it."""
    import test_gpu_seek
    cases = [(name, es, 0) for name, es, _ in test_gpu_seek.damaged_streams()]
    cases += [("b_clip_1280x720", stream("b_clip_1280x720"), 1), ("rows_ip", stream("rows_ip"), 0)]
    statuses = Counter()
    for name, es, decode_b in cases:
        bd = BatchDecoder(1, decode_b=decode_b)
        bd.write(0, es)
        want, _ = listed_residuals(bd, 0)
        for n, e in enumerate(chain_model.picture_index(es, decode_b)):
            bd.decode(n % 3, OUT_RESIDUALS if n % 2 else OUT_DEVICE)  # an arbitrary state before the seek
            assert bd.seek_pictures([(0, e["picture"])], OUT_RESIDUALS) == 1
            status, run = _fresh_residuals(es, e, decode_b)
            assert bd.last_seek_info[0]["status"] == status, (name, e["picture"])
            statuses[status] += 1
            if status and e["picture"] in want:
                assert np.array_equal(run[0], want[e["picture"]]), (name, e["picture"])
            assert np.array_equal(bd.read_residuals(0), run[0]), (name, e["picture"])
            for i, after in enumerate(run[1:3]):
                assert bd.decode(1, OUT_RESIDUALS) == 1
                assert np.array_equal(bd.read_residuals(0), after), (name, e["picture"], i)
        assert bd.last_error() is None
        bd.close()
    assert statuses[0] >= 1 and statuses[1] >= 10


def test_launch_counts():
    """76 equal-length streams (four tasks more than the plain RES kernel carries per launch, fewer than the plain
    kernel's 80): decode(6) with the flag puts its last step on reconstruct_res_kernel, two launches instead of one, and
    every other step is unchanged.  Streams of unequal length (the mixed batch, each stream's last step on a RES
    kernel, within every capacity): no launch is added."""
    import helpers
    small = b"".join(p for _, p in helpers.clip_packets(320, 240, 12))
    counts = []
    for flags in (OUT_DEVICE, OUT_RESIDUALS):
        bd = BatchDecoder(76, max_slots=1200)
        for s in range(76):
            bd.write(s, small)
        bd.reset_stats()
        assert bd.decode(6, flags) == 76 * 6
        st = bd.stats()
        counts.append((st["kernel_launches"], st["recon_launches"]))
        bd.close()
    (off_l, off_r), (on_l, on_r) = counts
    assert on_l == off_l + 1 and on_r == off_r == 6, counts
    counts = []
    for flags in (OUT_DEVICE, OUT_RESIDUALS):
        bd = BatchDecoder(len(MIXED), decode_b=True)
        for s, name in enumerate(MIXED):
            bd.write(s, stream(name))
        bd.reset_stats()
        for _ in range(3):
            bd.decode(6, flags)
        st = bd.stats()
        counts.append((st["kernel_launches"], st["recon_launches"]))
        bd.close()
    assert counts[0] == counts[1] and counts[0][1] > 0, counts


def test_the_bench_shape():
    """64 x 1080p x 60 through one decode(n, OUT_RESIDUALS) up to the last listed picture: every stream's residual is
    decode_residuals of that picture (compared on the device)."""
    import torch
    import bench
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips), max_slots=len(clips) * bench.PICTURES + 8)
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    last = min(max(e["picture"] for e in bd.macroblock_index(s)) for s in range(len(clips)))
    assert last >= bench.PICTURES - 2
    want = bd.decode_residuals([(s, last) for s in range(len(clips))])
    assert bd.decode(last + 1, OUT_RESIDUALS) == len(clips) * (last + 1)  # (I and P pictures: picture `last` is the last)
    for s in range(len(clips)):
        assert torch.equal(bd.device_residuals(s), want[s]), s
    assert bd.last_error() is None
    bd.close()
