"""decode_frames (include/jsmpeg_b200.h, jsmpeg_b200_batch_decode_frames) against its twins: frame j of a stream equals
what a twin batch reads back (planes, RGBA, residual, entries, last_picture) after the decode(1) that reconstructed that
picture, on the key-picture and B corpora with the slice walk and decode_b on and off, an .mpg, damaged streams and a
batch of mixed streams; and a third twin's decode(n, flags) leaves the same batch state under every flag combination."""
import ctypes

import numpy as np
import pytest

import chain_model
import synth_es
from jsmpeg_b200.batch import (MB_PRESENT, OUT_ACCUMULATED, OUT_DEVICE, OUT_HOST, OUT_MACROBLOCKS, OUT_RESIDUALS, OUT_RGBA,
                               BatchDecoder, Frame)
from test_gpu_intra import CORPUS, _damage, host
from test_gpu_macroblocks import B_CORPUS, MIXED, stream

pytestmark = pytest.mark.gpu
ALL = OUT_HOST | OUT_RGBA | OUT_MACROBLOCKS | OUT_ACCUMULATED | OUT_RESIDUALS
KINDS = ("planes", "rgba", "residuals", "macroblocks")


def make(es_list, ps=False, **opts):
    bd = BatchDecoder(len(es_list), **opts)
    for s, es in enumerate(es_list):
        if ps:
            bd.write_ps(s, es)
        else:
            bd.write(s, es)
    return bd


def per_picture(bd, n, flags=OUT_DEVICE):
    """n x decode(1, flags | OUT_RGBA | OUT_RESIDUALS | OUT_MACROBLOCKS) of the one-stream batch `bd`: per reconstructed
    picture {kind: what the read calls give, "type", "temporal_reference", "byte_pos"}"""
    out, at = [], []
    for _ in range(n):
        before_index, before = bd.get_index(0), bd.stats()["pictures_decoded"]
        if bd.decode(1, flags | OUT_RGBA | OUT_RESIDUALS | OUT_MACROBLOCKS) != 1:
            break
        if bd.stats()["pictures_decoded"] > before:
            t, r = bd.last_picture(0)
            out.append({"planes": np.concatenate(bd.read_planes(0)), "rgba": bd.read_rgba(0),
                        "residuals": bd.read_residuals(0), "macroblocks": bd.read_macroblocks(0), "type": t,
                        "temporal_reference": r})
            at.append((before_index + 7) >> 3)
    starts = chain_model.picture_positions(bd.read_es(0)) if out else []
    for o, a in zip(out, at):
        o["byte_pos"] = next(p for p in starts if p >= a)
    return out


def check_frames(got, want, label):
    """decode_frames' result `got` for one stream against per_picture's `want`"""
    assert got["n_frames"] == len(want), label
    for j, w in enumerate(want):
        for kind in KINDS:
            if got.get(kind) is not None:
                assert np.array_equal(host(got[kind][j]), w[kind]), (label, j, kind)
        info = got["info"][j]
        assert (info["type"], info["temporal_reference"], info["byte_pos"]) == (w["type"], w["temporal_reference"], w["byte_pos"]), (label, j)
        assert info["n_present"] == int((w["macroblocks"][..., 8] & MB_PRESENT).astype(bool).sum()), (label, j)


@pytest.mark.parametrize("name", CORPUS + B_CORPUS + ["mpg"])
def test_every_frame_equals_the_per_picture_twin(name):
    import gen_streams
    if name == "mpg":
        es, ps = gen_streams.make_clip_ps(320, 240, 24, form="mpg"), True
    else:
        es, ps = stream(name), False
    n = len(chain_model.picture_positions(gen_streams.make_clip_m1v(320, 240, 24) if ps else es)) + 2
    for slice_walk in (0, 1):
        for decode_b in (0, 1):
            a = make([es], ps, slice_walk=slice_walk, decode_b=decode_b)
            got = a.decode_frames(n, planes=True, rgba=True, residuals=True, macroblocks=True)
            b = make([es], ps, slice_walk=slice_walk, decode_b=decode_b)
            want = per_picture(b, n)
            assert want, name
            check_frames(got[0], want, (name, slice_walk, decode_b))
            if not decode_b:
                assert all(i["type"] != 3 for i in got[0]["info"])
            assert a.last_error() is None and b.last_error() is None
            a.close()
            b.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_damaged_streams(seed):
    import macroblock_model
    from test_gpu_intra import ffmpeg_es
    clean = ffmpeg_es(320, 240, 24) + synth_es.make_case("i_only_320x240")[-4:]
    b_clean = synth_es.make_case("b_one_slice_fcodes")
    errors = 0
    for es, decode_b in ((_damage(clean, macroblock_model.macroblock_index(clean)[::3], seed), 0),
                         (_damage(b_clean, macroblock_model.macroblock_index(b_clean)[1::2], seed, flips=3), 1)):
        n = len(chain_model.picture_positions(es)) + 1
        got = make([es], decode_b=decode_b).decode_frames(n, planes=True, rgba=True, residuals=True, macroblocks=True)
        check_frames(got[0], per_picture(make([es], decode_b=decode_b), n), (seed, decode_b))
        errors += sum(i["error"] != 0 for i in got[0]["info"])
    assert errors > 0


def observed(bd, flags):
    """Everything decode() leaves that a reader can see, per stream"""
    out = []
    for s in range(bd.n_streams):
        if not bd.stream_info(s)["has_sequence_header"]:
            out.append(None)
            continue
        o = [bd.get_index(s), bd.last_picture(s), np.concatenate(bd.read_planes(s)), bd.read_macroblocks(s),
             bd.read_accumulated(s), bd.read_residuals(s)]
        if flags & OUT_HOST:
            o += [np.concatenate([p.copy() for p in bd.host_planes(s)]), bd.host_macroblocks(s).copy()]
        rgba = ctypes.c_void_p()
        o.append(bd.read_rgba(s) if bd.lib.jsmpeg_b200_batch_get_rgba(bd.handle, s, ctypes.byref(rgba)) == 0 else None)
        out.append(o)
    return out


def same(x, y):
    if isinstance(x, np.ndarray):
        return np.array_equal(x, y)
    return x == y


@pytest.mark.parametrize("flags", [OUT_DEVICE, OUT_HOST, OUT_RGBA, OUT_MACROBLOCKS, OUT_ACCUMULATED, OUT_RESIDUALS,
                                   OUT_RGBA | OUT_RESIDUALS, ALL])
def test_batch_state_equals_decode(flags):
    """decode_frames(n, flags) with every destination, call after call, against decode(n, flags): every stats field but
    kernel_launches and the device times, and all a reader sees."""
    es_list = [stream(name) for name in MIXED]
    runs, stats = [], []
    for frames in (False, True):
        bd = make(es_list, decode_b=True)
        seen = []
        for n in [1, 3, 2, 5, 4, 8] * 4:
            if frames:
                out = bd.decode_frames(n, flags, planes=True, rgba=True, residuals=True, macroblocks=True)
                total = sum(o["n_frames"] for o in out)
                seen.append((total, observed(bd, flags)))
            else:
                before = bd.stats()["pictures_decoded"]
                bd.decode(n, flags)
                seen.append((bd.stats()["pictures_decoded"] - before, observed(bd, flags)))
        runs.append(seen)
        stats.append(bd.stats())
        assert bd.last_error() is None
        bd.close()
    for (na, a), (nb, b) in zip(*runs):
        assert na == nb
        for x, y in zip(a, b):
            assert (x is None) == (y is None)
            for u, v in zip(x or [], y or []):
                assert same(u, v)
    off, on = stats
    for key in off:
        if not key.endswith("_ms") and key != "kernel_launches":
            assert on[key] == off[key], key


def test_return_value_equals_decode():
    es_list = [stream(name) for name in MIXED]
    a, c = make(es_list, decode_b=True), make(es_list, decode_b=True)
    S = len(es_list)
    for n in (0, 1, 4, 7, 30):
        n_frames = (ctypes.c_int32 * S)()
        got = a.lib.jsmpeg_b200_batch_decode_frames(a.handle, n, 0, None, None, None, None, None, n_frames)
        assert got == c.decode(n), n
    a.close()
    c.close()


def test_mixed_streams_null_entries_and_short_streams():
    """Streams of different coded sizes and an odd display size in one batch, each destination array with a NULL entry,
    streams that run out at different counts, and n larger than any stream has: each stream's frames equal its own
    twin's, NULL entries get nothing, and memory past n_frames is untouched."""
    import torch
    names = MIXED + ["odd 101x51"]
    es_list = [stream(name) for name in MIXED]
    es_list.append(synth_es.SynthStream(synth_es.Knobs(width=101, height=51, pictures=6, gop=3, slices="random"), 19).generate())
    S, n = len(es_list), max(len(chain_model.picture_positions(es)) for es in es_list) + 3
    bd = make(es_list, decode_b=True)
    infos = [bd.stream_info(s) for s in range(S)]
    assert len({(i["width"], i["height"]) for i in infos}) > 2 and any(i["width"] & 1 or i["height"] & 1 for i in infos)
    dev = torch.device("cuda", 0)
    shapes = {"planes": lambda i: (i["coded_size"] * 3 // 2,), "rgba": lambda i: (i["height"], i["width"], 4),
              "residuals": lambda i: (i["coded_size"] * 3 // 2,),
              "macroblocks": lambda i: ((i["height"] + 15) // 16, (i["width"] + 15) // 16, 16)}
    dtypes = {"planes": torch.uint8, "rgba": torch.uint8, "residuals": torch.int16, "macroblocks": torch.uint8}
    null = {"planes": 1, "rgba": 2, "residuals": 3, "macroblocks": 4}  # the stream whose entry is NULL, per kind
    bufs = {k: [None if s == null[k] else torch.full((n, *shapes[k](infos[s])), 0x5A, dtype=dtypes[k], device=dev)
                for s in range(S)] for k in KINDS}
    arr = {k: (ctypes.c_void_p * S)(*[None if t is None else t.data_ptr() for t in bufs[k]]) for k in KINDS}
    info_out = (Frame * (S * n))()
    n_frames = (ctypes.c_int32 * S)()
    torch.cuda.synchronize()
    got = bd.lib.jsmpeg_b200_batch_decode_frames(bd.handle, n, OUT_DEVICE, arr["planes"], arr["rgba"], arr["residuals"],
                                                 arr["macroblocks"], info_out, n_frames)
    assert got > 0 and bd.last_error() is None
    counts = list(n_frames)
    assert len(set(counts)) > 2 and max(counts) < n
    for s in range(S):
        want = per_picture(make([es_list[s]], decode_b=True), n)
        assert counts[s] == len(want), names[s]
        for k in KINDS:
            t = bufs[k][s]
            if t is None:
                continue
            for j, w in enumerate(want):
                assert np.array_equal(host(t[j]), w[k]), (names[s], k, j)
            assert (host(t[counts[s]:]) == 0x5A).all(), (names[s], k)
        for j, w in enumerate(want):
            f = info_out[s * n + j]
            assert (f.byte_pos, f.picture_type, f.temporal_reference) == (w["byte_pos"], w["type"], w["temporal_reference"])
    bd.close()


def test_several_rounds_seek_and_reset():
    """A small max_slots cuts a call into many rounds: frames continue across them.  Frames after seek_pictures and
    after reset equal the twin's, which took the same seek or reset."""
    names = ["ffmpeg_320x240", "b_rows", "mini_enc_open_gop"]
    es_list = [stream(name) for name in names]
    a = make(es_list, decode_b=True, max_slots=4)
    outs = a.decode_frames(40, planes=True, residuals=True, macroblocks=True, rgba=True)
    for s, es in enumerate(es_list):
        check_frames(outs[s], per_picture(make([es], decode_b=True), 40), ("rounds", names[s]))
    a.close()
    for s, es in enumerate(es_list):
        entries = chain_model.picture_index(es, True)
        k = entries[len(entries) // 2]["picture"]
        a, b = make([es], decode_b=True), make([es], decode_b=True)
        for bd in (a, b):
            bd.decode(3)
            assert bd.seek_pictures([(0, k)]) == 1
        check_frames(a.decode_frames(6, rgba=True, residuals=True, macroblocks=True)[0], per_picture(b, 6), ("seek", names[s]))
        for bd in (a, b):
            bd.reset()
            bd.write(0, es)
        check_frames(a.decode_frames(5, rgba=True, residuals=True, macroblocks=True)[0], per_picture(b, 5), ("reset", names[s]))
        a.close()
        b.close()


def test_refusals_change_nothing():
    import torch
    es_list = [stream("ffmpeg_320x240"), stream("rows_ip")]
    bd = make(es_list)
    bd.decode(2, OUT_RGBA)
    before = observed(bd, OUT_RGBA)
    stats = bd.stats()
    t = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    good, bad = t.data_ptr(), t.data_ptr() + 8
    n_frames = (ctypes.c_int32 * 2)(7, 7)
    f = bd.lib.jsmpeg_b200_batch_decode_frames
    assert f(bd.handle, -1, 0, None, None, None, None, None, n_frames) == -2
    for pos in range(4):
        args = [None] * 4
        args[pos] = (ctypes.c_void_p * 2)(good, bad)
        assert f(bd.handle, 1, 0, *args, None, n_frames) == -2, pos
    assert list(n_frames) == [7, 7]
    with pytest.raises(ValueError):
        bd.decode_frames(-1)
    after = observed(bd, OUT_RGBA)
    for x, y in zip(before, after):
        for u, v in zip(x, y):
            assert same(u, v)
    assert bd.stats() == stats
    assert bd.last_error() is None
    bd.close()


def test_shared_geometry_is_one_tensor():
    """Two streams of one geometry, the second cut short: each kind is one [S, n, ...] tensor, each stream's frames a
    view of its row, as many as its twin reconstructs."""
    es = stream("ffmpeg_320x240")
    es_list = [es, es[:len(es) // 6]]
    bd = make(es_list)
    out = bd.decode_frames(10, planes=True, macroblocks=True)
    whole = bd.last_frames_batch["planes"]
    assert tuple(whole.shape) == (2, 10, 320 * 240 * 3 // 2)
    assert tuple(bd.last_frames_batch["macroblocks"].shape) == (2, 10, 15, 20, 16)
    for s in range(2):
        assert out[s]["planes"].data_ptr() == whole[s].data_ptr()
        check_frames(out[s], per_picture(make([es_list[s]]), 10), ("shared", s))
    assert out[0]["n_frames"] == 10 and 0 < out[1]["n_frames"] < 10
    bd.close()


def test_the_bench_shape():
    """64 x 1080p x 60 planar frames in one call against the per-picture twin on sampled frames."""
    import torch
    import bench
    clips = bench.load_streams(bench.rank_seeds(0))
    S, n = len(clips), bench.PICTURES
    a = BatchDecoder(S, max_slots=S * n + 8)
    b = BatchDecoder(S)
    for s, clip in enumerate(clips):
        a.write(s, clip)
        b.write(s, clip)
    out = a.decode_frames(n)
    assert {o["n_frames"] for o in out} == {n}
    sample = {0, 1, n // 2, n - 1}
    for j in range(n):
        assert b.decode(1) == S
        if j in sample:
            for s in range(0, S, 7):
                want = torch.as_tensor(np.concatenate(b.read_planes(s))).cuda()
                assert torch.equal(out[s]["planes"][j], want), (s, j)
    assert a.last_error() is None and b.last_error() is None
    a.close()
    b.close()
