"""Accumulated maps of the playback path (decode() and seek_pictures with OUT_ACCUMULATED, include/jsmpeg_b200.h):
after every I/P picture decode() reconstructs, the map equals decode_accumulated of that picture on every clean stream of
the key-picture and B corpora and an .mpg, with the slice walk and decode_b each on and off, and B pictures leave it as
it is; on damaged streams it is the model's fold over the device's own exports of the pictures decode() reconstructed;
calls without the flag, reset and a start on a P picture break the trace; seeks; the flag moves nothing else and adds
one launch per reconstruct step with an I/P picture; and the bench's shape."""
import numpy as np
import pytest

import accumulate_model
import chain_model
import helpers
import synth_es
from jsmpeg_b200.batch import (OUT_ACCUMULATED, OUT_DEVICE, OUT_HOST, OUT_MACROBLOCKS, OUT_RGBA, BatchDecoder,
                               accumulated_view)
from test_gpu_intra import CORPUS, _damage, ffmpeg_es, host
from test_gpu_macroblocks import B_CORPUS, MIXED, geometry, stream

pytestmark = pytest.mark.gpu


def untraced(bd, s):
    m = np.zeros((bd.stream_info(s)["coded_size"] * 3 // 2, 4), np.int16)
    m[:, 3] = -1
    return m


def listed_maps(bd, s):
    """{picture: host map} of decode_accumulated for every I/P picture of stream s's picture index"""
    pics = [e["picture"] for e in bd.picture_index(s) if e["type"] in (1, 2)]
    got = bd.decode_accumulated([(s, k) for k in pics])
    assert all(i["status"] == 1 for i in bd.last_accumulated_info)
    return {k: host(t) for k, t in zip(pics, got)}


def step_through(bd, es, flags=OUT_ACCUMULATED, s=0):
    """decode(1, flags) through stream s of `bd` (holding `es`): per consumed picture (picture number, picture type,
    whether it was reconstructed, map read back)."""
    starts = chain_model.picture_positions(es)
    out = []
    while True:
        at = (bd.get_index(s) + 7) >> 3
        before = bd.stats()["pictures_decoded"]
        if bd.decode(1, flags) != 1:
            return out
        k = next(i for i, p in enumerate(starts) if p >= at)
        out.append((k, bd.last_picture(s)[0], bd.stats()["pictures_decoded"] > before, bd.read_accumulated(s)))


def assert_follows(steps, want, prev_map, what):
    """Every reconstructed I/P picture's map is want[k] where listed; every other step leaves the map as it was"""
    compared = 0
    for k, ptype, decoded, got in steps:
        if decoded and ptype in (1, 2):
            if k in want:  # (an unclosed tail picture is not listed)
                assert np.array_equal(got, want[k]), (what, k)
                compared += 1
        else:
            assert np.array_equal(got, prev_map), (what, k, ptype)
        prev_map = got
    return compared


@pytest.mark.parametrize("name", CORPUS + B_CORPUS + ["mpg"])
def test_every_reconstructed_picture_equals_decode_accumulated(name):
    import gen_streams
    es = gen_streams.make_clip_m1v(320, 240, 24) if name == "mpg" else stream(name)

    def batch(**options):
        bd = BatchDecoder(1, **options)
        if name == "mpg":
            bd.write_ps(0, gen_streams.make_clip_ps(320, 240, 24, form="mpg"))
        else:
            bd.write(0, es)
        return bd

    ref = batch()
    want = listed_maps(ref, 0)  # (the same whatever the options: test_gpu_accumulated.py)
    ref.close()
    for slice_walk in (0, 1):
        for decode_b in (0, 1):
            bd = batch(slice_walk=slice_walk, decode_b=decode_b)
            steps = step_through(bd, es)
            n_ip = sum(d and t in (1, 2) for _, t, d, _ in steps)
            compared = assert_follows(steps, want, untraced(bd, 0), (name, slice_walk, decode_b))
            assert compared >= n_ip - 1 and compared > 0, (name, slice_walk, decode_b)
            view = bd.device_accumulated(0)
            assert view.is_cuda and str(view.dtype) == "torch.int16" and tuple(view.shape) == steps[-1][3].shape
            assert np.array_equal(host(view), steps[-1][3])
            assert tuple(accumulated_view(view, bd.stream_info(0))[0]["back"].shape) == tuple(
                x * 16 for x in geometry(bd, 0))
            assert bd.last_error() is None
            bd.close()


def device_fold(bd, s, pictures, mbw, mbh):
    """{picture: map}: accumulate_model.step folded over `pictures` (I/P picture numbers, the first traced from
    nothing) with the records and residuals of the device's own decode_macroblocks / decode_residuals"""
    reqs = [(s, k) for k in pictures]
    res = dict(zip(reqs, [host(r) for r in bd.decode_residuals(reqs)]))
    mbs = dict(zip(reqs, [host(m) for m in bd.decode_macroblocks(reqs)]))
    out, prev = {}, None
    for k in pictures:
        ent = mbs[(s, k)].reshape(-1, 16)
        rec = np.zeros((mbw * mbh, 16), np.uint8)  # mb_record_t of the entries: the forward vector, PRESENT / INTRA
        rec[:, 0:4] = ent[:, 0:4]
        rec[:, 4] = ent[:, 8] & 3
        prev = out[k] = accumulate_model.step(prev, rec, res[(s, k)], mbw, mbh)
    return out


@pytest.mark.parametrize("seed", [1, 2])
def test_damaged_streams_follow_the_fold_of_the_devices_own_exports(seed):
    import macroblock_model
    clean = ffmpeg_es(320, 240, 24) + synth_es.make_case("i_only_320x240")[-4:]  # end code: the last picture closes
    b_clean = synth_es.make_case("b_one_slice_fcodes")
    streams = [(_damage(clean, macroblock_model.macroblock_index(clean)[::3], seed), 0),
               (_damage(b_clean, macroblock_model.macroblock_index(b_clean)[1::2], seed, flips=3), 1)]
    for es, decode_b in streams:
        bd = BatchDecoder(1, decode_b=decode_b)
        bd.write(0, es)
        mbh, mbw = geometry(bd, 0)
        listed = {e["picture"] for e in bd.macroblock_index(0)}
        steps = step_through(bd, es)
        recon = [k for k, t, d, _ in steps if d and t in (1, 2)]
        want = device_fold(bd, 0, [k for k in recon if k in listed], mbw, mbh)
        compared = assert_follows(steps, want, untraced(bd, 0), (seed, decode_b))
        assert compared >= max(1, len(recon) - 1), (seed, decode_b)
        assert bd.last_error() is None
        bd.close()


def test_a_call_without_the_flag_breaks_the_trace_up_to_the_next_i_picture():
    """P picture m reconstructed without the flag: its map reads untraced; the next P picture starts a new trace from
    nothing (the fold with a break before it); the next I picture is decode_accumulated's again."""
    es = stream("ffmpeg_320x240")
    bd = BatchDecoder(1)
    bd.write(0, es)
    mbh, mbw = geometry(bd, 0)
    want = listed_maps(bd, 0)
    index = [e for e in bd.picture_index(0) if e["type"] in (1, 2)]
    i_pics = [e["picture"] for e in index if e["type"] == 1]
    gop = [e["picture"] for e in index if i_pics[0] < e["picture"] < i_pics[1]]  # the P pictures of the first GOP
    assert len(gop) >= 4
    for _ in range(3):  # i_pics[0], gop[0], gop[1]
        assert bd.decode(1, OUT_ACCUMULATED) == 1
    assert np.array_equal(bd.read_accumulated(0), want[gop[1]])
    assert bd.decode(1, OUT_DEVICE) == 1  # gop[2]
    assert np.array_equal(bd.read_accumulated(0), untraced(bd, 0))
    fold = device_fold(bd, 0, gop[3:], mbw, mbh)  # (gop[3] is predicted from a set without a map)
    for k in gop[3:]:
        assert bd.decode(1, OUT_ACCUMULATED) == 1
        got = bd.read_accumulated(0)
        assert np.array_equal(got, fold[k]), k
        assert (got[:, 3] == -1).sum() > (want[k][:, 3] == -1).sum(), k
    assert bd.decode(1, OUT_ACCUMULATED) == 1  # i_pics[1]
    assert np.array_equal(bd.read_accumulated(0), want[i_pics[1]])
    assert bd.last_error() is None
    bd.close()


def test_untraced_before_the_flag_and_after_reset():
    es = stream("ffmpeg_320x240")
    bd = BatchDecoder(2)
    bd.write(0, es)
    empty = untraced(bd, 0)
    assert np.array_equal(bd.read_accumulated(0), empty)  # before any decode()
    assert bd.decode(2) == 2
    assert np.array_equal(bd.read_accumulated(0), empty)  # before any call with the flag
    assert np.array_equal(host(bd.device_accumulated(0)), empty)
    bd.reset()
    bd.write(0, es)
    want = listed_maps(bd, 0)
    steps = step_through(bd, es)
    assert assert_follows(steps, want, empty, "before reset") >= 10
    bd.reset()
    assert np.array_equal(bd.read_accumulated(0), empty)
    bd.write(0, es)
    assert np.array_equal(bd.read_accumulated(0), empty)
    assert assert_follows(step_through(bd, es), want, empty, "after reset") >= 10
    for s, call in ((1, bd.read_accumulated), (1, bd.device_accumulated), (2, bd.read_accumulated),
                    (-1, bd.device_accumulated)):
        with pytest.raises(ValueError):
            call(s)
    for s in (1, 2, -1):
        assert bd.lib.jsmpeg_b200_batch_get_accumulated(bd.handle, s, None) != 0
        assert bd.lib.jsmpeg_b200_batch_read_accumulated(bd.handle, s, None) != 0
    assert bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("decode_b", [0, 1])
def test_a_start_on_a_p_picture_follows_the_sequential_model(decode_b):
    """set_index to the first P picture: every I/P map equals accumulate_model.sequential of the oracle from the same
    index -- untraced predicted samples up to the next I picture, decode_accumulated's maps after it."""
    name = "b_clip_1280x720" if decode_b else "ffmpeg_320x240"  # (I P B B P B B P B B I ...)
    es = stream(name)
    first_p = next(e for e in chain_model.picture_index(es) if e["type"] == 2)
    model = {start - 4: m for start, _, m in accumulate_model.sequential(helpers.oracle_lib(), es, decode_b,
                                                                          index=first_p["byte_pos"] * 8)}
    bd = BatchDecoder(1, decode_b=decode_b)
    bd.write(0, es)
    want = listed_maps(bd, 0)
    bd.set_index(0, first_p["byte_pos"] * 8)
    starts = chain_model.picture_positions(es)
    steps = step_through(bd, es)
    compared, untraced_run = 0, 0
    for k, ptype, decoded, got in steps:
        if decoded and ptype in (1, 2) and starts[k] in model:
            assert np.array_equal(got, model[starts[k]]), (name, k)
            compared += 1
            untraced_run += k in want and not np.array_equal(got, want[k])
    assert compared >= len(model) - 1 and untraced_run >= 2, (compared, len(model), untraced_run)
    assert bd.last_error() is None
    bd.close()


def _fresh_maps(es, entry, decode_b):
    """The device's own decode() with OUT_ACCUMULATED of chain_model.seek_bytes(es, entry) in a new batch: status and
    the map right after the decode() that consumes picture k (or the last one before, when none does), then after
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
        assert bd.decode(1, OUT_ACCUMULATED) == 1
        if nxt == target:
            status = 1
            break
    run = [bd.read_accumulated(0)]
    while bd.decode(1, OUT_ACCUMULATED) == 1:
        run.append(bd.read_accumulated(0))
    bd.close()
    return status, run


def test_seek_with_the_flag():
    """Status 1 (clean streams, decode_b on and off) and status 0 (a damaged and a cut stream): the map the fresh
    decoder has, and on clean streams decode_accumulated of picture k, or of the newer reference for a B picture k;
    then every decode(1, flag) after it goes on as that decoder does.  A seek without the flag leaves untraced maps."""
    import test_gpu_seek
    cases = [(name, es, 0, False) for name, es, _ in test_gpu_seek.damaged_streams()]
    cases += [("b_clip_1280x720", stream("b_clip_1280x720"), 1, True),
              ("mini_enc_open_gop", stream("mini_enc_open_gop"), 1, True), ("rows_ip", stream("rows_ip"), 0, True)]
    statuses = {0: 0, 1: 0}
    for name, es, decode_b, clean in cases:
        bd = BatchDecoder(1, decode_b=decode_b)
        bd.write(0, es)
        want = listed_maps(bd, 0) if clean else {}
        entries = chain_model.picture_index(es, decode_b)
        for n, e in enumerate(entries):
            bd.decode(n % 3, OUT_ACCUMULATED if n % 2 else OUT_DEVICE)  # an arbitrary state before the seek
            assert bd.seek_pictures([(0, e["picture"])], OUT_HOST | OUT_ACCUMULATED) == 1
            status, run = _fresh_maps(es, e, decode_b)
            assert bd.last_seek_info[0]["status"] == status, (name, e["picture"])
            statuses[status] += 1
            got = bd.read_accumulated(0)
            assert np.array_equal(got, run[0]), (name, e["picture"])
            if clean:
                assert status == 1
                newest = max(k for k in want if k <= e["picture"])  # (k itself for an I/P picture)
                assert np.array_equal(got, want[newest]), (name, e["picture"])
            for i, after in enumerate(run[1:4]):
                assert bd.decode(1, OUT_ACCUMULATED) == 1
                assert np.array_equal(bd.read_accumulated(0), after), (name, e["picture"], i)
            if n % 4 == 0:  # the same seek without the flag: no map
                assert bd.seek_pictures([(0, e["picture"])], OUT_DEVICE) == 1
                assert np.array_equal(bd.read_accumulated(0), untraced(bd, 0)), (name, e["picture"])
        assert bd.last_error() is None
        bd.close()
    assert statuses[0] >= 1 and statuses[1] >= 10


def _observed(bd, n_streams, flags):
    return [(bd.get_index(s), bd.last_picture(s), np.concatenate(bd.read_planes(s)),
             np.concatenate([p.copy() for p in bd.host_planes(s)]), bd.read_rgba(s), bd.read_macroblocks(s),
             bd.host_macroblocks(s).copy())
            for s in range(n_streams)]


def test_nothing_else_moves():
    """Planes, RGBA, host ring, entries, bit index and last_picture after every call, and the stats minus
    kernel_launches, are those of a twin batch without the flag, on a multi-stream batch with decode(n) for n > 1 under
    OUT_HOST | OUT_RGBA | OUT_MACROBLOCKS; the flag adds at most one launch per reconstruct step."""
    flags = OUT_HOST | OUT_RGBA | OUT_MACROBLOCKS
    runs, stats = [], []
    for extra in (0, OUT_ACCUMULATED):
        bd = BatchDecoder(len(MIXED), decode_b=True)
        for s, name in enumerate(MIXED):
            bd.write(s, stream(name))
        seen = []
        for n in [1, 3, 2, 5, 1, 4] * 6:
            got = bd.decode(n, flags | extra)
            seen.append((got, _observed(bd, len(MIXED), flags)))
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
    assert 0 < on["kernel_launches"] - off["kernel_launches"] <= on["recon_launches"]
    for key in off:
        if key != "kernel_launches" and not key.endswith("_ms"):
            assert on[key] == off[key], key


def test_launch_counts():
    """decode(1, flag) over I/P/B streams with decode_b: one more launch for each call whose step has an I/P picture,
    none for a step of B pictures alone; decode(n) over I/P streams: one more per reconstruct step."""
    names = ["b_rows", "mini_enc_open_gop"]
    runs = []
    for extra in (0, OUT_ACCUMULATED):
        bd = BatchDecoder(len(names), decode_b=True)
        for s, name in enumerate(names):
            bd.write(s, stream(name))
        ip_steps = 0
        while True:
            before = [bd.get_index(s) for s in range(len(names))]
            decoded = bd.stats()["pictures_decoded"]
            if not bd.decode(1, extra):
                break
            moved = [s for s in range(len(names)) if bd.get_index(s) != before[s]]
            ip_steps += bd.stats()["pictures_decoded"] > decoded and any(bd.last_picture(s)[0] in (1, 2) for s in moved)
        runs.append((bd.stats(), ip_steps))
        bd.close()
    (off, ip_steps), (on, _) = runs
    assert 0 < ip_steps < on["recon_launches"]  # (some steps reconstruct B pictures alone)
    assert (on["kernel_launches"] - off["kernel_launches"], on["recon_launches"]) == (ip_steps, off["recon_launches"])
    counts = []
    for extra in (0, OUT_ACCUMULATED):
        bd = BatchDecoder(3)
        for s, name in enumerate(["ffmpeg_320x240", "rows_ip", "ffmpeg_1280x720"]):
            bd.write(s, stream(name))
        while bd.decode(4, extra):
            pass
        counts.append(bd.stats())
        bd.close()
    assert counts[1]["kernel_launches"] - counts[0]["kernel_launches"] == counts[1]["recon_launches"] > 0


def test_the_bench_shape():
    """64 x 1080p x 60 through decode(60, OUT_ACCUMULATED): the last map of every stream equals decode_accumulated of
    its picture 59 (compared on the device; a sequence end code after each clip closes that picture, so that the
    picture index lists it)."""
    import sys

    import torch
    sys.path.insert(0, helpers.ROOT)
    import bench
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips), max_slots=len(clips) * bench.PICTURES + 8)
    for s, clip in enumerate(clips):
        bd.write(s, clip + b"\x00\x00\x01\xb7")
    assert bd.decode(bench.PICTURES, OUT_ACCUMULATED) == len(clips) * bench.PICTURES
    last = [bd.picture_index(s)[bench.PICTURES - 1] for s in range(len(clips))]
    assert all(e["picture"] == bench.PICTURES - 1 and e["type"] in (1, 2) for e in last)
    want = bd.decode_accumulated([(s, bench.PICTURES - 1) for s in range(len(clips))])
    assert all(i["status"] == 1 for i in bd.last_accumulated_info)
    for s in range(len(clips)):
        assert torch.equal(bd.device_accumulated(s), want[s]), s
    assert int((want[0][:, 3] >= 1).sum()) > 0
    assert bd.last_error() is None
    bd.close()
