"""The buffers of one decoder regrow while it works, and what it computes stays the same.

A decoder first sizes everything for a 176x144 stream: the record slot pool, the parse and export task lists, the
chain plane sets and the zeroed forward set of a chain of one.  A 1280x720 stream then arrives on another stream of
the same decoder in growing pieces, so the ES mirror regrows, and every size above regrows too.  A stream dense in
start codes overflows the scan's position list (the scan runs again with room for all) and restages the device's
start-code lists with longer rows.  The device TS and PS demuxers' scratch regrows with bigger chunks.  Every
result is checked against what the other GPU suites compare with."""
import hashlib
import json
import os

import numpy as np
import pytest

import bench
import chain_model
import gen_streams
import helpers
import intra_model
import macroblock_model
import mini_ps
from jsmpeg_b200 import ts
from jsmpeg_b200.batch import OUT_HOST, BatchDecoder
from test_gpu_intra import host
from test_gpu_ps_demux import _feed
from test_macroblock_index import oracle_fresh
from test_picture_index import fresh_decode

pytestmark = pytest.mark.gpu

SMALL = os.path.join(helpers.GOLDEN, "ffmpeg_176x144_ip")
CLIP_720P = os.path.join(helpers.ROOT, "tests", "fixtures", "b_clip_1280x720")


def growing_cuts(n, first):
    """Cut positions in (0, n) with every piece twice as long as the one before."""
    cuts, at, size = [], first, first
    while at < n:
        cuts.append(at)
        size *= 2
        at += size
    return cuts


def planes_sha(bd, s):
    return {k: hashlib.sha256(p.tobytes()).hexdigest() for k, p in zip(("y", "cr", "cb"), bd.read_planes(s))}


def check_macroblocks(bd, streams):
    """decode_macroblocks of the first `pick` listed pictures of each (stream, es, pick) against the model's
    conversion of the oracle's records."""
    reqs, want = [], []
    for s, es, pick in streams:
        for e in macroblock_model.macroblock_index(es)[:pick]:
            info, rec = oracle_fresh(es, e)
            reqs.append((s, e["picture"]))
            want.append((info.n_present, info.error, macroblock_model.export(rec, e["type"])))
    got = bd.decode_macroblocks(reqs)
    for r, t, i, (n_present, error, mb) in zip(reqs, got, bd.last_macroblocks_info, want):
        assert (i["n_present"], i["error"]) == (n_present, error), r
        assert np.array_equal(host(t).reshape(-1, 16), mb), r


def check_pictures(bd, streams):
    """decode_pictures of the first `pick` listed pictures of each (stream, es, pick) against the oracle fed the
    fresh bytes of each picture."""
    reqs, want = [], []
    for s, es, pick in streams:
        for e in chain_model.picture_index(es, True)[:pick]:
            planes, _, _ = fresh_decode(es, e, True)
            reqs.append((s, e["picture"]))
            want.append(np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in planes]))
    got = bd.decode_pictures(reqs)
    for r, t, i, w in zip(reqs, got, bd.last_pictures_info, want):
        assert i["status"] == 1 and np.array_equal(host(t), w), r


def test_engine_buffers_regrow_within_one_decoder():
    small = open(SMALL + ".es", "rb").read()
    golden = json.load(open(SMALL + ".json"))["pictures"]
    big = open(CLIP_720P + ".m1v", "rb").read()
    meta = json.load(open(CLIP_720P + ".json"))
    bd = BatchDecoder(2, decode_b=1)
    bd.write(0, small)
    for k in range(2):
        assert bd.decode(1, OUT_HOST) == 1
        assert planes_sha(bd, 0) == {c: golden[k][c] for c in ("y", "cr", "cb")}, k
    check_macroblocks(bd, [(0, small, 2)])
    check_pictures(bd, [(0, small, 2)])
    prev = 0
    for c in growing_cuts(len(big), 4096) + [len(big)]:
        bd.write(1, big[prev:c])
        prev = c
        assert [e["byte_pos"] for e in bd.picture_index(1)] == [e["byte_pos"] for e in chain_model.picture_index(big[:c], True)]
    check_macroblocks(bd, [(0, small, None), (1, big, None)])
    check_pictures(bd, [(0, small, None), (1, big, None)])
    n0, n1 = len(golden) - 2, len(meta["fnv1a64"])
    for step in range(max(n0, n1)):
        assert bd.decode(1, OUT_HOST) == (step < n0) + (step < n1), step
        if step < n0:
            assert planes_sha(bd, 0) == {c: golden[2 + step][c] for c in ("y", "cr", "cb")}, step
        if step < n1:
            assert format(bench.fnv1a64_planes(*bd.read_planes(1)), "016x") == meta["fnv1a64"][step], step
    assert bd.decode(1, OUT_HOST) == 0
    assert bd.last_error() is None and bd.stats()["parse_errors"] == 0
    bd.close()


def test_dense_start_codes_rescan_and_restage():
    """20,000 user-data start codes between two pictures: more than the scan's first position list holds, and more
    than the device's start-code rows staged for the first stream.  The pictures decode as without them."""
    small = open(SMALL + ".es", "rb").read()
    golden = json.load(open(SMALL + ".json"))["pictures"]
    second = [p for p in intra_model.prefixes(small) if small[p + 3] == 0][1]
    dense = small[:second] + b"\x00\x00\x01\xb2" * 20000 + small[second:]
    bd = BatchDecoder(2)
    bd.write(0, small)
    assert bd.decode(1, OUT_HOST) == 1
    bd.write(1, dense)
    assert [e["byte_pos"] for e in bd.picture_index(1)] == [e["byte_pos"] for e in chain_model.picture_index(dense)]
    want = {c: golden[0][c] for c in ("y", "cr", "cb")}
    assert bd.decode(1, OUT_HOST) == 2 and planes_sha(bd, 1) == want
    for k in range(1, len(golden)):
        assert bd.decode(1, OUT_HOST) >= 1
        assert planes_sha(bd, 1) == {c: golden[k][c] for c in ("y", "cr", "cb")}, k
    assert bd.last_error() is None
    bd.close()


def test_demux_scratch_regrows_with_bigger_chunks():
    """TS on stream 0 and PS on stream 1 of one decoder, each in pieces that double: the ES and PES tables equal
    the host demuxers' of the whole input."""
    bd = BatchDecoder(2)
    data = gen_streams.make_clip_ts(320, 240, 24, seed=1234, noise=9)
    es = b"".join(p for _, p in ts.demux_video_es(data))
    total, prev = 0, 0
    for c in growing_cuts(len(data), 188 * 4) + [len(data)]:
        total += bd.write_ts(0, data[prev:c])[0]
        prev = c
    assert total == len(es) and bd.read_es(0) == es
    data = gen_streams.make_clip_ps(320, 240, 24, form="mpg")
    want_es, want_pes = mini_ps.demux_chunked(data, [])
    total, pes = _feed(bd, 1, data, growing_cuts(len(data), 2048))
    assert total == len(want_es) and bd.read_es(1) == want_es and pes == want_pes
    assert bd.last_error() is None
    bd.close()
