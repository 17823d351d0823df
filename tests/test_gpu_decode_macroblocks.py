"""Macroblock entries of the playback path (decode() and seek_pictures with OUT_MACROBLOCKS, include/jsmpeg_b200.h)
against decode_macroblocks of the picture decode() consumed: every stream of the key-picture and B corpora with the
slice walk and decode_b on and off, an .mpg, damaged streams, the host ring, seeks, the reference-ABI decoder and the
bench's shape; and the flag moves nothing else and adds exactly one launch per reconstruct step."""
from collections import Counter

import numpy as np
import pytest

import chain_model
import synth_es
import test_gpu_launch_counts as launch_counts
from jsmpeg_b200.batch import OUT_DEVICE, OUT_HOST, OUT_MACROBLOCKS, OUT_RGBA, BatchDecoder, macroblocks_view
from jsmpeg_b200.decoder import MPEG1Video
from test_gpu_intra import CORPUS, _damage, ffmpeg_es, host
from test_gpu_macroblocks import B_CORPUS, MIXED, stream

pytestmark = pytest.mark.gpu


def listed_entries(bd, s):
    """{picture: host entries [mb_height, mb_width, 16]} of every picture decode_macroblocks lists for stream s, and
    {picture: n_present}."""
    pics = [e["picture"] for e in bd.macroblock_index(s)]
    got = bd.decode_macroblocks([(s, k) for k in pics])
    return ({k: host(t) for k, t in zip(pics, got)},
            {k: i["n_present"] for k, i in zip(pics, bd.last_macroblocks_info)})


def step_through(bd, es, flags=OUT_MACROBLOCKS):
    """decode(1, flags) through stream 0 of `bd` (holding `es`): per picture decode() reconstructs, (picture number,
    entries read back, stats' macroblock count of the step, Y | Cr | Cb)."""
    starts = chain_model.picture_positions(es)
    out = []
    while True:
        at = (bd.get_index(0) + 7) >> 3
        before = bd.stats()
        if bd.decode(1, flags) != 1:
            return out
        after = bd.stats()
        if after["pictures_decoded"] > before["pictures_decoded"]:
            k = next(i for i, p in enumerate(starts) if p >= at)
            out.append((k, bd.read_macroblocks(0), after["macroblocks"] - before["macroblocks"],
                        np.concatenate(bd.read_planes(0))))


@pytest.mark.parametrize("name", CORPUS + B_CORPUS + ["mpg"])
def test_every_reconstructed_picture_equals_decode_macroblocks(name):
    import gen_streams
    es = gen_streams.make_clip_m1v(320, 240, 24) if name == "mpg" else stream(name)
    for slice_walk in (0, 1):
        for decode_b in (0, 1):
            bd = BatchDecoder(1, slice_walk=slice_walk, decode_b=decode_b)
            if name == "mpg":
                bd.write_ps(0, gen_streams.make_clip_ps(320, 240, 24, form="mpg"))
            else:
                bd.write(0, es)
            want, _ = listed_entries(bd, 0)
            steps = step_through(bd, es)
            compared = 0
            for k, got, _, _ in steps:
                if k in want:  # (an unclosed tail picture is not listed)
                    assert np.array_equal(got, want[k]), (name, k, slice_walk, decode_b)
                    compared += 1
            assert compared >= len(steps) - 1 and compared > 0, (name, slice_walk, decode_b)
            view = bd.device_macroblocks(0)
            assert view.is_cuda and tuple(view.shape) == steps[-1][1].shape
            assert np.array_equal(host(view), steps[-1][1])
            assert macroblocks_view(view)["flags"].shape == view.shape[:2]
            assert bd.last_error() is None
            bd.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_damaged_streams(seed):
    """The walk that starts at k's start code on both paths: the same entries and the same n_present."""
    import macroblock_model
    clean = ffmpeg_es(320, 240, 24) + synth_es.make_case("i_only_320x240")[-4:]  # end code: the last picture closes
    b_clean = synth_es.make_case("b_one_slice_fcodes")
    streams = [(_damage(clean, macroblock_model.macroblock_index(clean)[::3], seed), 0),
               (_damage(b_clean, macroblock_model.macroblock_index(b_clean)[1::2], seed, flips=3), 1)]
    for es, decode_b in streams:
        bd = BatchDecoder(1, decode_b=decode_b)
        bd.write(0, es)
        want, n_present = listed_entries(bd, 0)
        steps = step_through(bd, es)
        compared = 0
        for k, got, macroblocks, _ in steps:
            if k in want:
                assert np.array_equal(got, want[k]) and macroblocks == n_present[k], (seed, decode_b, k)
                compared += 1
        assert compared >= max(5, len(steps) - 1), (seed, decode_b)
        assert bd.last_error() is None
        bd.close()


def _observed(bd, n_streams, flags):
    return [(bd.get_index(s), bd.last_picture(s), np.concatenate(bd.read_planes(s)),
             np.concatenate([p.copy() for p in bd.host_planes(s)]), bd.read_rgba(s) if flags & OUT_RGBA else None)
            for s in range(n_streams)]


def test_nothing_else_moves():
    """Planes, RGBA, host ring, bit index and last_picture after every call, and the stats minus the entries' bytes and
    launches, are those of a twin batch without the flag, on a multi-stream batch with decode(n) for n > 1."""
    flags = OUT_HOST | OUT_RGBA
    runs, stats = [], []
    for extra in (0, OUT_MACROBLOCKS):
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
        mb_bytes = [bd.read_macroblocks(s).nbytes for s in range(len(MIXED))] if extra else None
        bd.close()
    assert len(runs[0]) == len(runs[1]) and runs[0][-1][0] == 0
    for (ga, a), (gb, b) in zip(*runs):
        assert ga == gb
        for x, y in zip(a, b):
            assert x[:2] == y[:2]
            for u, v in zip(x[2:], y[2:]):
                assert (u is None and v is None) or np.array_equal(u, v)
    off, on = stats
    # every picture reconstructed: its entries copied out once; every reconstruct step: one export launch
    decoded = []
    for name in MIXED:
        single = BatchDecoder(1, decode_b=True)
        single.write(0, stream(name))
        single.decode(10 ** 6)
        decoded.append(single.stats()["pictures_decoded"])
        single.close()
    assert sum(decoded) == on["pictures_decoded"]
    assert on["d2h_bytes"] - off["d2h_bytes"] == sum(d * m for d, m in zip(decoded, mb_bytes))
    assert on["kernel_launches"] - off["kernel_launches"] == on["recon_launches"] > 0
    for key in off:
        if key not in ("d2h_bytes", "kernel_launches") and not key.endswith("_ms"):
            assert on[key] == off[key], key


@pytest.mark.parametrize("name,decode_b", [("ffmpeg_320x240", 0), ("b_clip_1280x720", 1), ("mini_enc_open_gop", 1)])
def test_host_ring_slot_holds_the_entries_of_its_planes(name, decode_b):
    """OUT_HOST | OUT_MACROBLOCKS with decode(n), n = 1 ... 6 (several turns of the four-slot ring in one call): the
    host entries are those of the picture host_planes shows, the last one the call reconstructed."""
    es = stream(name)
    ref = BatchDecoder(1, decode_b=decode_b)
    ref.write(0, es)
    sequence = [(got, planes) for _, got, _, planes in step_through(ref, es)]  # per reconstruction
    ref.close()
    bd = BatchDecoder(1, decode_b=decode_b)
    bd.write(0, es)
    calls = 0
    for n in [1, 2, 3, 4, 5, 6] * 10:
        if not bd.decode(n, OUT_HOST | OUT_MACROBLOCKS):
            break
        calls += 1
        done = bd.stats()["pictures_decoded"]
        entries, planes = sequence[done - 1]
        assert np.array_equal(np.concatenate([p.copy() for p in bd.host_planes(0)]), planes), (name, calls)
        assert np.array_equal(bd.host_macroblocks(0), entries), (name, calls)
        assert np.array_equal(bd.read_macroblocks(0), entries), (name, calls)
    assert calls >= 4 and bd.stats()["pictures_decoded"] == len(sequence)
    bd.close()


def _fresh_entries(es, entry, decode_b):
    """The device's own decode() with OUT_MACROBLOCKS of chain_model.seek_bytes(es, entry) in a new batch: status and
    the entries right after the decode() that consumes picture k (or the last one before, when none does), then after
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
        assert bd.decode(1, OUT_MACROBLOCKS) == 1
        if nxt == target:
            status = 1
            break
    run = [bd.read_macroblocks(0)]
    while bd.decode(1, OUT_MACROBLOCKS) == 1:
        run.append(bd.read_macroblocks(0))
    bd.close()
    return status, run


def test_seek_with_the_flag():
    """Status 1 (clean streams, decode_b on and off) and status 0 (a damaged and a cut stream): the entries of the
    picture the state ends on, as the fresh decoder has them, and those of every decode() after it; under OUT_HOST the
    host ring's slot too."""
    import test_gpu_seek
    cases = [(name, es, 0) for name, es, _ in test_gpu_seek.damaged_streams()]
    cases += [("b_clip_1280x720", stream("b_clip_1280x720"), 1), ("mini_enc_open_gop", stream("mini_enc_open_gop"), 1),
              ("rows_ip", stream("rows_ip"), 0)]
    statuses = Counter()
    for name, es, decode_b in cases:
        bd = BatchDecoder(1, decode_b=decode_b)
        bd.write(0, es)
        want, _ = listed_entries(bd, 0)
        entries = chain_model.picture_index(es, decode_b)
        for n, e in enumerate(entries):
            bd.decode(n % 3, OUT_MACROBLOCKS if n % 2 else OUT_DEVICE)  # an arbitrary state before the seek
            assert bd.seek_pictures([(0, e["picture"])], OUT_HOST | OUT_MACROBLOCKS) == 1
            status, run = _fresh_entries(es, e, decode_b)
            assert bd.last_seek_info[0]["status"] == status, (name, e["picture"])
            statuses[status] += 1
            if status:
                assert np.array_equal(run[0], want[e["picture"]]), (name, e["picture"])
                assert np.array_equal(bd.host_macroblocks(0), run[0]), (name, e["picture"])
            assert np.array_equal(bd.read_macroblocks(0), run[0]), (name, e["picture"])
            for i, entries_after in enumerate(run[1:4]):
                assert bd.decode(1, OUT_MACROBLOCKS) == 1
                assert np.array_equal(bd.read_macroblocks(0), entries_after), (name, e["picture"], i)
        assert bd.last_error() is None
        bd.close()
    assert statuses[0] >= 1 and statuses[1] >= 10


def test_entries_are_zero_before_the_flag_and_after_reset_and_calls_without_it_write_none():
    es = stream("ffmpeg_320x240")
    bd = BatchDecoder(2)
    bd.write(0, es)
    assert bd.decode(2) == 2
    assert not bd.read_macroblocks(0).any() and not bd.host_macroblocks(0).any()
    assert bd.decode(1, OUT_MACROBLOCKS) == 1
    first = bd.read_macroblocks(0)
    assert first.any()
    # pictures 3 and 4 without the flag: picture 4's planes went to the set of picture 2 (the I/P ping-pong), whose
    # entries were not written again -- they describe picture 2
    assert bd.decode(2, OUT_DEVICE) == 2
    assert np.array_equal(bd.read_macroblocks(0), first)
    bd.reset()
    assert not bd.read_macroblocks(0).any() and not bd.host_macroblocks(0).any()
    for s, call in ((1, bd.read_macroblocks), (1, bd.host_macroblocks), (1, bd.device_macroblocks),
                    (2, bd.read_macroblocks), (-1, bd.device_macroblocks)):
        with pytest.raises(ValueError):
            call(s)
    for fn in (bd.lib.jsmpeg_b200_batch_get_macroblocks, bd.lib.jsmpeg_b200_batch_get_host_macroblocks):
        for s in (1, 2, -1):
            assert fn(bd.handle, s, None) != 0
    assert bd.lib.jsmpeg_b200_batch_read_macroblocks(bd.handle, 5, None) != 0
    assert bd.last_error() is None
    bd.close()


def test_launch_counts():
    """The mixed workload of test_gpu_launch_counts.py (its two decode() calls of six steps each) with the flag: one
    more launch per reconstruct step, the export's; without the flag, that file pins the counts."""
    small = b"".join(p for _, p in launch_counts.helpers.clip_packets(320, 240, 12))
    big = open(launch_counts.FIXTURE_720P, "rb").read()
    bd = BatchDecoder(launch_counts.N_SMALL + launch_counts.N_720P, max_slots=1200, decode_b=1, slice_walk=1)
    for s in range(launch_counts.N_SMALL):
        bd.write(s, small)
    for s in range(launch_counts.N_720P):
        bd.write(launch_counts.N_SMALL + s, big)
    bd.reset_stats()
    for name, flags in (("decode plain", OUT_MACROBLOCKS), ("decode rgba", OUT_RGBA | OUT_MACROBLOCKS)):
        bd.decode(6, flags)
        _, launches, recon, _ = next(x for x in launch_counts.EXPECTED if x[0] == name)
        st = bd.stats()  # (counted from the reset: one more launch per reconstruct step so far)
        assert (st["kernel_launches"], st["recon_launches"]) == (launches + recon, recon), name
    bd.close()


@pytest.mark.parametrize("name,decode_b", [("ffmpeg_320x240", 0), ("b_clip_1280x720", 1)])
def test_reference_abi_decoder_option(name, decode_b):
    es = stream(name)
    bd = BatchDecoder(1, decode_b=decode_b)
    bd.write(0, es)
    plain = MPEG1Video({"decodeFirstFrame": False, "decodeBPictures": bool(decode_b)})
    dec = MPEG1Video({"decodeFirstFrame": False, "exportMacroblocks": True, "decodeBPictures": bool(decode_b)})
    for d in (plain, dec):
        d.write(0, [es])
    n = 0
    while bd.decode(1, OUT_HOST | OUT_MACROBLOCKS):
        assert dec.decode() and plain.decode()
        assert plain.macroblocks() is None
        got = dec.macroblocks()
        assert got.shape == bd.host_macroblocks(0).shape
        assert np.array_equal(got, bd.host_macroblocks(0)), (name, n)
        assert all(np.array_equal(a, b) for a, b in zip(dec.planes(), bd.host_planes(0)))
        n += 1
    assert not dec.decode() and n >= 6
    dec.destroy()
    plain.destroy()
    bd.close()


def test_the_bench_shape():
    """64 x 1080p x 60 through decode(1, OUT_MACROBLOCKS), every step's entries of every stream against
    decode_macroblocks of all listed pictures (compared on the device)."""
    import torch
    import bench
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips), max_slots=len(clips) * bench.PICTURES + 8)
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    listed = [bd.macroblock_index(s) for s in range(len(clips))]
    assert all([e["picture"] for e in index] == list(range(len(index))) and {e["type"] for e in index} <= {1, 2}
               for index in listed)
    reqs = [(s, e["picture"]) for s, index in enumerate(listed) for e in index]
    want = dict(zip(reqs, bd.decode_macroblocks(reqs)))
    compared = 0
    for k in range(bench.PICTURES):  # I and P pictures only: step k reconstructs picture k of every stream
        assert bd.decode(1, OUT_MACROBLOCKS) == len(clips)
        for s in range(len(clips)):
            if (s, k) in want:
                assert torch.equal(bd.device_macroblocks(s), want[(s, k)]), (s, k)
                compared += 1
    assert compared >= len(clips) * (bench.PICTURES - 1)
    assert bd.last_error() is None
    bd.close()
