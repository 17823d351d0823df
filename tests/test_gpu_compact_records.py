"""Stage 1b -> stage 2 through compact coefficient records (jsmpeg_b200/csrc/coef_records.h) on the device, where
both forms occur: a stream coded at quantiser scale 1 (most coded blocks carry more than 12 values and take the dense
form) alone and in a batch with bench-like streams (nearly every block compact), through decode(), OUT_RGBA,
decode_pictures, decode_intra, the B-picture walk and the slice walk, against the oracle.  The CPU twin is
tests/test_compact_records.py."""
import numpy as np
import pytest

import helpers
import test_oracle_golden as golden
from jsmpeg_b200.batch import OUT_DEVICE, OUT_RGBA, BatchDecoder

pytestmark = pytest.mark.gpu


def qscale1_stream(b_frames=0, frames=10):
    pytest.importorskip("cv2")
    import mini_enc
    es, types, _, _ = mini_enc.make_b_clip(width=176, height=144, frames=frames, b_frames=b_frames, qscale=(1, 1, 1))
    return es, types


def bench_like(width, height, frames, seed):
    pytest.importorskip("cv2")
    return b"".join(p for _, p in helpers.clip_packets(width, height, frames, seed=seed, noise=9))


def oracle_frames(es, decode_b=False):
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(1 if decode_b else 0)
    try:
        frames, _, d = helpers.decode_all(lib, [(0, es)])
        d.destroy()
    finally:
        lib.oracle_set_decode_b(0)
    return [np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in f]) for f in frames]


def flat(planes):
    return np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in planes])


def decode_batch(streams, flags=OUT_DEVICE, **options):
    """every stream picture by picture (decode(1) steps), Y | Cr | Cb per step"""
    bd = BatchDecoder(len(streams), **options)
    for i, es in enumerate(streams):
        bd.write(i, es)
    got = [[] for _ in streams]
    while bd.decode(1, flags):
        for i in range(len(streams)):
            got[i].append(flat(bd.read_planes(i)))
    assert bd.last_error() is None
    bd.close()
    return got


def assert_streams_equal(got, want, what):
    for i, (g, w) in enumerate(zip(got, want)):
        assert len(g) >= len(w), f"{what}: stream {i}: {len(g)} of {len(w)} pictures"
        for k in range(len(w)):
            assert np.array_equal(g[k], w[k]), f"{what}: stream {i} picture {k}: {np.count_nonzero(g[k] != w[k])} bytes differ"


@pytest.mark.parametrize("flags", [OUT_DEVICE, OUT_RGBA], ids=["planes", "rgba"])
def test_qscale1_stream_alone_and_in_a_bench_like_batch(flags):
    es, _ = qscale1_stream()
    streams = [es, bench_like(640, 360, 8, 1234), bench_like(320, 240, 12, 1235), es]
    want = [oracle_frames(s) for s in streams]
    assert_streams_equal(decode_batch(streams[:1], flags), want[:1], "alone")
    assert_streams_equal(decode_batch(streams, flags), want, "batch")


def test_decode_pictures_and_decode_intra():
    es, types = qscale1_stream()
    clip = bench_like(320, 240, 12, 1236)
    want = {0: oracle_frames(es), 1: oracle_frames(clip)}
    bd = BatchDecoder(2)
    bd.write(0, es)
    bd.write(1, clip)
    # (a stream's last picture is listed once a start code closes it: the index may stop one picture short)
    reqs = [(s, e["picture"]) for s in (0, 1) for e in bd.picture_index(s)]
    assert len(reqs) >= len(want[0]) + len(want[1]) - 2
    for (s, k), t in zip(reqs, bd.decode_pictures(reqs)):
        assert np.array_equal(t.cpu().numpy(), want[s][k]), ("decode_pictures", s, k)
    reqs = [(s, e["picture"]) for s in (0, 1) for e in bd.intra_index(s)]
    assert reqs
    for (s, k), t in zip(reqs, bd.decode_intra(reqs)):
        assert np.array_equal(t.cpu().numpy(), want[s][k]), ("decode_intra", s, k)
    assert bd.last_error() is None
    bd.close()


def test_b_pictures():
    es, types = qscale1_stream(b_frames=2, frames=10)
    assert 3 in types
    streams = [es, bench_like(320, 240, 12, 1237)]
    want = [oracle_frames(es, decode_b=True), oracle_frames(streams[1])]
    assert_streams_equal(decode_batch(streams, decode_b=1), want, "decode_b")


def test_slice_walk():
    es, _ = qscale1_stream()
    rows, _ = golden.load_case("rows_ip")
    streams = [es, rows]
    assert_streams_equal(decode_batch(streams, slice_walk=1), [oracle_frames(s) for s in streams], "slice_walk")
