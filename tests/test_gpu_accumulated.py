"""Accumulated motion and residuals on the device (jsmpeg_b200_batch_decode_accumulated) against the serial model
(tools/accumulate_model.py) of the oracle's fresh decode with B pictures off, bit for bit: every listed I/P picture of
the key-picture corpus and of I/P/B streams, with the slice walk and decode_b each off and on; a first P picture's map
rebuilt from the device's own decode_macroblocks and decode_residuals; an .mpg; mixed sizes with duplicates, many
requests on one chain and on many chains, slot pressure, chain groups, damaged streams, the decode() state the call
must leave alone, invalid requests, launch counts, and the bench's shape."""
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

import helpers  # (first: it puts tools/ on the path, also when the file runs as a script)
import accumulate_model  # noqa: E402
import synth_es  # noqa: E402
from jsmpeg_b200.batch import OUT_HOST, BatchDecoder, accumulated_view
from test_gpu_intra import CORPUS, _assert_same_state, _damage, _state, host
from test_gpu_macroblocks import B_CORPUS, MIXED, geometry, stream

pytestmark = pytest.mark.gpu


def ip_index(bd, s):
    """The I and P entries of stream s's picture index: what decode_accumulated accepts"""
    return [e for e in bd.picture_index(s) if e["type"] in (1, 2)]


def model_entry(es, picture):
    import chain_model
    return next(e for e in chain_model.picture_index(es) if e["picture"] == picture)


@functools.lru_cache(maxsize=None)
def expected(name, picture):
    """(status, n_present, error, int16 map) of I/P picture `picture` of corpus stream `name`"""
    es = stream(name)
    return accumulate_model.oracle_chain(helpers.oracle_lib(), es, model_entry(es, picture))


def check(name, picture, t, info):
    status, n_present, error, want = expected(name, picture)
    assert str(t.dtype) == "torch.int16" and t.is_cuda and tuple(t.shape) == want.shape
    assert (info["status"], info["n_present"], info["error"]) == (status, n_present, error), (name, picture)
    assert np.array_equal(host(t), want), (name, picture)


@pytest.mark.parametrize("name", CORPUS + B_CORPUS)
def test_every_listed_picture_equals_the_model_with_every_option(name):
    """All listed I/P pictures in one call, with the slice walk and decode_b each off and on: the model's map of the
    oracle's fresh decode with B pictures off, whatever the options (the listing does not change with decode_b)."""
    es = stream(name)
    listings = []
    for slice_walk, decode_b in ((0, 0), (1, 0), (0, 1), (1, 1)):
        bd = BatchDecoder(1, slice_walk=slice_walk, decode_b=decode_b)
        bd.write(0, es)
        entries = ip_index(bd, 0)
        listings.append([(e["picture"], e["chain_start"]) for e in entries])
        got = bd.decode_accumulated([(0, e["picture"]) for e in entries])
        for e, t, i in zip(entries, got, bd.last_accumulated_info):
            check(name, e["picture"], t, i)
        assert bd.last_error() is None
        bd.close()
    assert listings[0] and all(x == listings[0] for x in listings)


@pytest.mark.parametrize("name", ["ffmpeg_320x240", "mini_enc_fcodes_2_4_fullpel_bwd"])
def test_a_first_p_picture_rebuilt_from_the_devices_own_exports(name):
    """The map of a P picture right after its key picture, rebuilt from decode_macroblocks and decode_residuals of the
    same picture on the same decoder: back 1, the exported vector, the exported residual."""
    bd = BatchDecoder(1)
    bd.write(0, stream(name))
    mbh, mbw = geometry(bd, 0)
    info = bd.stream_info(0)
    entries = ip_index(bd, 0)
    firsts = [e for e, before in zip(entries[1:], entries) if e["type"] == 2 and before["type"] == 1
              and e["chain_start"] == before["picture"]]
    assert firsts
    reqs = [(0, e["picture"]) for e in firsts]
    maps = bd.decode_accumulated(reqs)
    res = bd.decode_residuals(reqs)
    mbs = bd.decode_macroblocks(reqs)
    key_rec = np.zeros((mbw * mbh, 16), np.uint8)  # a key picture: every macroblock PRESENT and INTRA
    key_rec[:, 4] = 3
    key = accumulate_model.step(None, key_rec, np.zeros(mbw * mbh * 384, np.int16), mbw, mbh)
    for t, r, m in zip(maps, res, mbs):
        ent = host(m).reshape(-1, 16)
        rec = np.zeros((mbw * mbh, 16), np.uint8)  # mb_record_t of the entries: the forward vector, PRESENT / INTRA
        rec[:, 0:4] = ent[:, 0:4]
        rec[:, 4] = ent[:, 8] & 3
        assert np.array_equal(host(t), accumulate_model.step(key, rec, host(r), mbw, mbh))
        y = accumulated_view(t, info)[0]
        assert tuple(y["motion"].shape) == (mbh * 16, mbw * 16, 2) and bool((y["back"] <= 1).all())
    bd.close()


def test_program_stream_through_write_ps():
    import gen_streams
    data = gen_streams.make_clip_ps(320, 240, 24, form="mpg")
    m1v = gen_streams.make_clip_m1v(320, 240, 24)
    bd = BatchDecoder(1)
    bd.write_ps(0, data)
    entries = ip_index(bd, 0)
    assert len(entries) >= 10
    got = bd.decode_accumulated([(0, e["picture"]) for e in entries])
    for e, t, i in zip(entries, got, bd.last_accumulated_info):
        status, _, _, want = accumulate_model.oracle_chain(helpers.oracle_lib(), m1v, model_entry(m1v, e["picture"]))
        assert i["status"] == status and np.array_equal(host(t), want), e["picture"]
    bd.close()


def test_mixed_sizes_many_chains_and_duplicates():
    """Streams of five sizes shuffled in one call: many requests on one chain, requests on many chains of one stream,
    and the same picture two and three times."""
    bd = BatchDecoder(len(MIXED))
    for s, name in enumerate(MIXED):
        bd.write(s, stream(name))
    rng = random.Random(7)
    reqs = []
    for s in range(len(MIXED)):
        pics = [e["picture"] for e in ip_index(bd, s)]
        reqs += [(s, k) for k in rng.sample(pics, min(len(pics), 7))]
    reqs += [reqs[2], reqs[9], reqs[9]]
    rng.shuffle(reqs)
    got = bd.decode_accumulated(reqs)
    for (s, k), t, i in zip(reqs, got, bd.last_accumulated_info):
        check(MIXED[s], k, t, i)
    assert len({(s, e["chain_start"]) for s in range(len(MIXED)) for e in ip_index(bd, s)}) > len(MIXED)
    bd.close()


def test_slot_pressure_and_chain_groups_give_the_same_bytes():
    """Three record slots (several waves per chain, the look-ahead flushed), and default slots: the same maps."""
    names = ["ffmpeg_320x240", "rows_ip", "b_rows", "mini_enc_open_gop"]
    outs = []
    for max_slots in (0, 3):
        bd = BatchDecoder(len(names), max_slots=max_slots)
        for s, name in enumerate(names):
            bd.write(s, stream(name))
        reqs = [(s, e["picture"]) for s in range(len(names)) for e in ip_index(bd, s)]
        reqs += reqs[::5]
        bd.decode(2)
        got = bd.decode_accumulated(reqs)
        outs.append(([host(t) for t in got], bd.last_accumulated_info, reqs))
        bd.close()
    assert len(outs[0][0]) == len(outs[1][0]) >= 40
    assert outs[0][1] == outs[1][1]
    for (s, k), a, b in zip(outs[0][2], outs[0][0], outs[1][0]):
        assert np.array_equal(a, b)
        assert np.array_equal(a, expected(names[s], k)[3]), (names[s], k)


def test_a_request_cut_into_chain_groups():
    """More chains than a wave has slots: the chains run in groups, with the same maps."""
    es = stream("ffmpeg_320x240")
    n = 12
    bd = BatchDecoder(n, max_slots=8)
    for s in range(n):
        bd.write(s, es)
    entries = ip_index(bd, 0)
    reqs = [(s, entries[(3 * s) % len(entries)]["picture"]) for s in range(n)]
    got = bd.decode_accumulated(reqs)
    for (s, k), t, i in zip(reqs, got, bd.last_accumulated_info):
        check("ffmpeg_320x240", k, t, i)
    bd.close()


def test_damaged_streams_follow_the_model():
    """Bit flips in I/P and B streams, three seeds: the model of the oracle fed everything from the chain start on (the
    bits the walks read past a closing code), status 0 (every record untraced) where it never consumes the picture."""
    import chain_model
    clean = stream("ffmpeg_320x240") + synth_es.make_case("i_only_320x240")[-4:]
    b_clean = synth_es.make_case("b_one_slice_fcodes")
    streams = []
    for seed in (1, 2, 3):
        streams += [_damage(clean, chain_model.picture_index(clean)[::3], seed),
                    _damage(b_clean, chain_model.picture_index(b_clean)[1::2], seed, flips=3)]
    bd = BatchDecoder(len(streams))
    statuses = Counter()
    for s, es in enumerate(streams):
        bd.write(s, es)
        entries = [e for e in chain_model.picture_index(es) if e["type"] in (1, 2)]
        assert [e["picture"] for e in entries] == [e["picture"] for e in ip_index(bd, s)]
        got = bd.decode_accumulated([(s, e["picture"]) for e in entries])
        for e, t, i in zip(entries, got, bd.last_accumulated_info):
            status, n_present, error, want = accumulate_model.oracle_chain(helpers.oracle_lib(), es, e, rest=True)
            assert i["status"] == status and bool(i["error"]) == bool(error), (s, e["picture"])
            assert np.array_equal(host(t), want), (s, e["picture"])
            statuses[status] += 1
    assert statuses[1] and bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("name,decode_b", [("ffmpeg_320x240", False), ("b_rows", True)])
def test_decode_state_is_untouched(name, decode_b):
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
                bd.decode_accumulated([(s, e["picture"]) for s in (0, 1) for e in ip_index(bd, s)])
                _assert_same_state(before, _state(bd, 0))
        runs.append(frames)
        bd.close()
    assert len(runs[0]) == len(runs[1])
    for a, b in zip(*runs):
        assert np.array_equal(a, b)


def test_invalid_requests_are_refused_and_change_nothing():
    import intra_model
    es = synth_es.make_case("b_rows")  # I B B P B B I B B P B B I
    bd = BatchDecoder(3, decode_b=True)
    bd.write(0, es)
    bd.write(1, es[intra_model.first_sequence_header(es)[0] + 4:])  # no sequence header
    bd.write(2, synth_es.make_case("ignored_pictures_userdata"))  # picture 2: P with forward_f_code 0; 6: D
    assert bd.decode(1, OUT_HOST)
    before = _state(bd, 0)
    ip = ip_index(bd, 0)
    b_pics = [e["picture"] for e in bd.picture_index(0) if e["type"] == 3]
    assert b_pics  # listed by decode_pictures with decode_b on, refused here
    good = ip[1]["picture"]
    mark = bd.decode_accumulated([(0, good)])[0].clone().fill_(7)

    def call(reqs, dsts):
        n = len(reqs)
        return bd.lib.jsmpeg_b200_batch_decode_accumulated(
            bd.handle, n, (ctypes.c_int * n)(*[s for s, _ in reqs]), (ctypes.c_uint32 * n)(*[p for _, p in reqs]),
            (ctypes.c_void_p * n)(*dsts), None, None, None)

    # with a valid request in front: a B picture, no sequence header, no stream, no picture, f_code 0, D
    for stream_, pic in ((0, b_pics[0]), (1, 0), (3, 0), (-1, 0), (0, 99), (2, 2), (2, 6)):
        assert call([(0, good), (stream_, pic)], [mark.data_ptr(), mark.data_ptr()]) == -2, (stream_, pic)
        with pytest.raises(ValueError):
            bd.decode_accumulated([(0, good), (stream_, pic)])
    assert call([(0, good)], [None]) == -2                 # NULL destination
    assert call([(0, good)], [mark.data_ptr() + 8]) == -2  # misaligned destination
    assert bool((mark == 7).all())
    _assert_same_state(before, _state(bd, 0))
    assert bd.last_error() is None
    assert call([(0, good)], [mark.data_ptr()]) == 1
    assert np.array_equal(host(mark), expected("b_rows", good)[3])
    assert call([], []) == 0
    bd.close()


def launch_counts():
    """({kernel: launches} of one decode_accumulated call of one wave, the most reference pictures of its two chains),
    counted by torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    import chain_model
    from test_macroblock_index import pictures
    bd = BatchDecoder(2, max_slots=64, decode_b=1)
    refs, reqs = [], []
    for s, name in enumerate(("ffmpeg_320x240", "b_rows")):
        es = stream(name)
        bd.write(s, es)
        last = ip_index(bd, s)[-1]
        reqs.append((s, last["picture"]))
        refs.append(sum(chain_model.is_reference(es, p) for p in pictures(es)[last["chain_start"]:last["picture"] + 1]))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        bd.decode_accumulated(reqs)
        torch.cuda.synchronize()
    kernels = Counter()
    for ev in prof.events():
        m = re.search(r"(\w+_kernel)\(", ev.name)
        if ev.device_type == torch.autograd.DeviceType.CUDA and m:
            kernels[m.group(1)] += 1
    bd.close()
    return dict(kernels), max(refs)


def test_launch_counts():
    """One wave: one accumulate launch per chain depth, no reconstruct launch.  (Counted in a process of its own.)"""
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "launch-counts"], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    kernels, depth = json.loads(r.stdout.strip().splitlines()[-1])
    assert kernels.get("accumulate_kernel") == depth > 1
    assert not any("reconstruct" in k for k in kernels), kernels


def test_the_bench_shape():
    """16 consecutive I/P pictures from each of the bench's 64 distinct 1080p clips in one call; the last picture of
    every fourth clip equals the model of the oracle."""
    sys.path.insert(0, helpers.ROOT)
    import bench
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips))
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    reqs = [(s, e["picture"]) for s in range(len(clips)) for e in ip_index(bd, s)[:16]]
    got = bd.decode_accumulated(reqs)
    assert bd.last_error() is None and len(got) == 1024
    assert all(i["status"] == 1 for i in bd.last_accumulated_info)
    for j in range(15, len(reqs), 64):
        s, k = reqs[j]
        assert tuple(got[j].shape) == (68 * 120 * 384, 4)
        _, _, _, want = accumulate_model.oracle_chain(helpers.oracle_lib(), clips[s], model_entry(clips[s], k))
        assert np.array_equal(host(got[j]), want), (s, k)
    bd.close()


if __name__ == "__main__" and sys.argv[1:] == ["launch-counts"]:
    print(json.dumps(launch_counts()))
