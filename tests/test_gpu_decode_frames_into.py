"""decode_frames_into (include/jsmpeg_b200.h, jsmpeg_b200_batch_decode_frames_into) against its twins: coefficient frame j
of a stream equals decode_coefficients of that picture, and map frame j what read_accumulated gives right after the
decode(1, flags | OUT_ACCUMULATED) that reconstructed it in a twin batch (all untraced for a B picture) -- on the
key-picture and B corpora with the slice walk and decode_b on and off, an .mpg, damaged streams, mixed streams, many
rounds and calls, and after seek, reset and calls without the flag; a third twin's decode(n, flags) leaves the same batch
state, maps included, and the chain of maps carries into the next decode()."""
import ctypes

import numpy as np
import pytest

import chain_model
import synth_es
from jsmpeg_b200.batch import (OUT_ACCUMULATED, OUT_DEVICE, OUT_HOST, OUT_MACROBLOCKS, OUT_RESIDUALS, OUT_RGBA,
                               BatchDecoder, Frame, FrameDst)
from test_gpu_decode_frames import ALL, make, observed, same
from test_gpu_intra import CORPUS, _damage, host
from test_gpu_macroblocks import B_CORPUS, MIXED, stream

pytestmark = pytest.mark.gpu
NEW = ("coefficients", "accumulated")


def untraced(coded_size):
    m = np.zeros((coded_size * 3 // 2, 4), np.int16)
    m[:, 3] = -1
    return m


def twin(bd, n, flags=OUT_DEVICE, slice_walk=0):
    """n x decode(1, flags | OUT_ACCUMULATED) of the one-stream batch `bd`: per reconstructed picture {"type",
    "byte_pos", "accumulated": read_accumulated right after that decode (all untraced for a B picture), "coefficients":
    decode_coefficients of the picture (picture k: the k-th picture start code).  decode_coefficients lists only closed
    pictures, and decode() also reconstructs a last picture that runs to the end of the buffer, so the coefficients come
    from a batch (with bd's `slice_walk`) that holds bd's stream closed by a sequence end code."""
    out, at = [], []
    cs = bd.stream_info(0)["coded_size"] if bd.stream_info(0)["has_sequence_header"] else 0
    for _ in range(n):
        before_index, before = bd.get_index(0), bd.stats()["pictures_decoded"]
        if bd.decode(1, flags | OUT_ACCUMULATED) != 1:
            break
        if bd.stats()["pictures_decoded"] > before:
            t, _ = bd.last_picture(0)
            out.append({"type": t, "accumulated": untraced(cs) if t == 3 else bd.read_accumulated(0)})
            at.append((before_index + 7) >> 3)
    if out:
        es = bd.read_es(0)
        starts = chain_model.picture_positions(es)
        closed = BatchDecoder(1, slice_walk=slice_walk)
        closed.write(0, es + b"\x00\x00\x01\xb7")
        pics = []
        for o, a in zip(out, at):
            k = next(k for k, p in enumerate(starts) if p >= a)
            o["byte_pos"] = starts[k]
            pics.append(k)
        listed = {e["picture"]: e["byte_pos"] for e in closed.macroblock_index(0)}
        assert all(listed.get(k) == o["byte_pos"] for k, o in zip(pics, out))
        for o, c in zip(out, closed.decode_coefficients([(0, k) for k in pics])):
            o["coefficients"] = host(c)
        assert closed.last_error() is None
        closed.close()
    return out


def check(got, want, label, kinds=NEW):
    """decode_frames' result `got` for one stream against twin's `want`"""
    assert got["n_frames"] == len(want), label
    for j, w in enumerate(want):
        assert (got["info"][j]["type"], got["info"][j]["byte_pos"]) == (w["type"], w["byte_pos"]), (label, j)
        for kind in kinds:
            assert np.array_equal(host(got[kind][j]), w[kind]), (label, j, kind)


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
            got = a.decode_frames(n, OUT_ACCUMULATED, planes=False, coefficients=True, accumulated=True)
            want = twin(make([es], ps, slice_walk=slice_walk, decode_b=decode_b), n, slice_walk=slice_walk)
            assert want, name
            check(got[0], want, (name, slice_walk, decode_b))
            assert decode_b or all(i["type"] != 3 for i in got[0]["info"])
            assert a.last_error() is None
            a.close()


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
        got = make([es], decode_b=decode_b).decode_frames(n, OUT_ACCUMULATED, coefficients=True, accumulated=True)
        check(got[0], twin(make([es], decode_b=decode_b), n), (seed, decode_b))
        errors += sum(i["error"] != 0 for i in got[0]["info"])
    assert errors > 0


@pytest.mark.parametrize("flags", [OUT_DEVICE, OUT_MACROBLOCKS, OUT_ACCUMULATED, OUT_ACCUMULATED | OUT_HOST,
                                   OUT_ACCUMULATED | OUT_RGBA | OUT_RESIDUALS, ALL])
def test_batch_state_equals_decode(flags):
    """decode_frames_into(n, flags) with every destination, call after call, against decode(n, flags): every stats field
    but kernel_launches and the device times, and all a reader sees, maps included; then the next
    decode(1, OUT_ACCUMULATED) gives the same maps, so the chain carries on from the call's map frames."""
    es_list = [stream(name) for name in MIXED]
    acc = bool(flags & OUT_ACCUMULATED)
    runs, stats = [], []
    for frames in (False, True):
        bd = make(es_list, decode_b=True)
        seen = []
        for n in [1, 3, 2, 5, 4, 8] * 3:
            if frames:
                out = bd.decode_frames(n, flags, planes=False, rgba=True, residuals=True, macroblocks=True,
                                       coefficients=True, accumulated=acc)
                seen.append((sum(o["n_frames"] for o in out), observed(bd, flags)))
            else:
                before = bd.stats()["pictures_decoded"]
                bd.decode(n, flags)
                seen.append((bd.stats()["pictures_decoded"] - before, observed(bd, flags)))
        for _ in range(3):
            bd.decode(1, OUT_ACCUMULATED)
            seen.append((0, [bd.read_accumulated(s) if bd.stream_info(s)["has_sequence_header"] else None
                             for s in range(len(es_list))]))
        runs.append(seen)
        stats.append(bd.stats())
        assert bd.last_error() is None
        bd.close()
    for (na, a), (nb, b) in zip(*runs):
        assert na == nb
        for x, y in zip(a, b):
            assert (x is None) == (y is None)
            if isinstance(x, np.ndarray):
                assert np.array_equal(x, y)
                continue
            for u, v in zip(x or [], y or []):
                assert same(u, v)
    off, on = stats
    for key in off:
        if not key.endswith("_ms") and key != "kernel_launches":
            assert on[key] == off[key], key
    assert on["kernel_launches"] > off["kernel_launches"]  # (the coefficient exports)


def test_rounds_and_calls_in_a_row():
    """max_slots=4 cuts each call into many rounds, and five calls follow one another: each stream's frames of all calls,
    one after the other, equal its twin's, so maps chain across rounds and calls."""
    names = ["ffmpeg_320x240", "b_rows", "mini_enc_open_gop", "rows_ip"]
    es_list = [stream(name) for name in names]
    a = make(es_list, decode_b=True, max_slots=4)
    calls = [7, 1, 12, 3, 20]
    got = [{k: [] for k in NEW + ("info",)} for _ in names]
    for n in calls:
        for s, o in enumerate(a.decode_frames(n, OUT_ACCUMULATED | OUT_RGBA, planes=False, coefficients=True,
                                              accumulated=True)):
            for k in got[s]:
                got[s][k] += list(o[k]) if o[k] is not None else []
    for s, es in enumerate(es_list):
        want = twin(make([es], decode_b=True), sum(calls), OUT_RGBA)
        g = got[s]
        check({"n_frames": len(g["info"]), **g}, want, ("rounds", names[s]))
    assert a.last_error() is None
    a.close()


@pytest.mark.parametrize("before", ["seek", "seek_acc", "reset", "no_flag", "no_flag_into"])
def test_after_seek_reset_and_a_call_without_the_flag(before):
    """The same operation on both batches first; then the map frames follow OUT_ACCUMULATED's prev rule exactly as the
    twin's decode(1) loop does: a trace broken by a seek or a call without the flag, or by reset, stays untraced up to
    the next I picture."""
    for name in ["ffmpeg_320x240", "b_rows", "mini_enc_open_gop"]:
        es = stream(name)
        a, b = make([es], decode_b=True), make([es], decode_b=True)
        entries = chain_model.picture_index(es, True)
        k = entries[len(entries) // 2]["picture"]
        for bd in (a, b):
            if before.startswith("seek"):
                bd.decode(3, OUT_ACCUMULATED)
                assert bd.seek_pictures([(0, k)], OUT_ACCUMULATED if before == "seek_acc" else OUT_DEVICE) == 1
            elif before == "reset":
                bd.decode(4, OUT_ACCUMULATED)
                bd.reset()
                bd.write(0, es)
            elif before == "no_flag":
                bd.decode(2, OUT_ACCUMULATED)
                bd.decode(2)
            elif bd is a:  # decode_frames_into without map frames and without the flag breaks it the same way
                a.decode_frames(2, OUT_ACCUMULATED, planes=False, coefficients=True, accumulated=True)
                a.decode_frames(2, planes=False, coefficients=True)
            else:
                b.decode(2, OUT_ACCUMULATED)
                b.decode(2)
        got = a.decode_frames(8, OUT_ACCUMULATED, planes=False, coefficients=True, accumulated=True)[0]
        check(got, twin(b, 8), (before, name))
        a.close()
        b.close()


def test_mixed_streams_null_entries_and_short_streams():
    """Streams of different coded sizes and an odd display size in one batch, each new array with a NULL entry, streams
    that run out at different counts, and n larger than any stream has: each stream's frames equal its own twin's, NULL
    entries get nothing, and memory past n_frames is untouched."""
    import torch
    names = MIXED + ["odd 101x51"]
    es_list = [stream(name) for name in MIXED]
    es_list.append(synth_es.SynthStream(synth_es.Knobs(width=101, height=51, pictures=6, gop=3, slices="random"), 19).generate())
    S, n = len(es_list), max(len(chain_model.picture_positions(es)) for es in es_list) + 3
    bd = make(es_list, decode_b=True)
    infos = [bd.stream_info(s) for s in range(S)]
    assert len({(i["width"], i["height"]) for i in infos}) > 2 and any(i["width"] & 1 or i["height"] & 1 for i in infos)
    dev = torch.device("cuda", 0)
    shapes = {"coefficients": lambda i: ((i["height"] + 15) // 16, (i["width"] + 15) // 16, 6, 8, 8),
              "accumulated": lambda i: (i["coded_size"] * 3 // 2, 4)}
    null = {"coefficients": 1, "accumulated": 4}  # the stream whose entry is NULL, per kind
    bufs = {k: [None if s == null[k] else torch.full((n, *shapes[k](infos[s])), 0x5A5A, dtype=torch.int16, device=dev)
                for s in range(S)] for k in NEW}
    arr = {k: (ctypes.c_void_p * S)(*[None if t is None else t.data_ptr() for t in bufs[k]]) for k in NEW}
    dst = FrameDst(None, None, None, None, ctypes.addressof(arr["coefficients"]), ctypes.addressof(arr["accumulated"]))
    info_out = (Frame * (S * n))()
    n_frames = (ctypes.c_int32 * S)()
    torch.cuda.synchronize()
    got = bd.lib.jsmpeg_b200_batch_decode_frames_into(bd.handle, n, OUT_ACCUMULATED, ctypes.byref(dst), info_out, n_frames)
    assert got > 0 and bd.last_error() is None
    counts = list(n_frames)
    assert len(set(counts)) > 2 and max(counts) < n
    for s in range(S):
        want = twin(make([es_list[s]], decode_b=True), n)
        assert counts[s] == len(want), names[s]
        for k in NEW:
            t = bufs[k][s]
            if t is None:
                continue
            for j, w in enumerate(want):
                assert np.array_equal(host(t[j]), w[k]), (names[s], k, j)
            assert (host(t[counts[s]:]) == 0x5A5A).all(), (names[s], k)
        for j, w in enumerate(want):
            f = info_out[s * n + j]
            assert (f.byte_pos, f.picture_type) == (w["byte_pos"], w["type"])
    bd.close()


def test_refusals_change_nothing():
    import torch
    es_list = [stream("ffmpeg_320x240"), stream("rows_ip")]
    bd = make(es_list)
    bd.decode(2, OUT_ACCUMULATED | OUT_RGBA)
    before = observed(bd, OUT_RGBA)
    stats = bd.stats()
    t = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda")
    good, bad = t.data_ptr(), t.data_ptr() + 8
    n_frames = (ctypes.c_int32 * 2)(7, 7)
    f = bd.lib.jsmpeg_b200_batch_decode_frames_into
    assert f(bd.handle, 1, OUT_ACCUMULATED, None, None, n_frames) == -2  # NULL dst
    for field in ("coef", "acc"):
        arr = (ctypes.c_void_p * 2)(good, bad)
        dst = FrameDst(**{field: ctypes.addressof(arr)})
        assert f(bd.handle, 1, OUT_ACCUMULATED, ctypes.byref(dst), None, n_frames) == -2, field
    arr = (ctypes.c_void_p * 2)(None, good)
    for flags in (OUT_DEVICE, ALL & ~OUT_ACCUMULATED):  # a map destination without the flag
        assert f(bd.handle, 1, flags, ctypes.byref(FrameDst(acc=ctypes.addressof(arr))), None, n_frames) == -2, flags
    assert f(bd.handle, -1, OUT_ACCUMULATED, ctypes.byref(FrameDst()), None, n_frames) == -2
    assert list(n_frames) == [7, 7]
    with pytest.raises(ValueError):
        bd.decode_frames(1, OUT_RGBA, accumulated=True)
    after = observed(bd, OUT_RGBA)
    for x, y in zip(before, after):
        for u, v in zip(x, y):
            assert same(u, v)
    assert bd.stats() == stats
    assert bd.last_error() is None
    bd.close()


def test_the_old_kinds_alone_equal_decode_frames():
    """decode_frames_into with only decode_frames' four arrays (and NULL coef / acc) is decode_frames: the same frames,
    the same batch state and the same stats, kernel_launches included."""
    import torch
    es_list = [stream(name) for name in MIXED]
    S, n, flags = len(es_list), 9, OUT_RGBA | OUT_MACROBLOCKS | OUT_ACCUMULATED
    results = []
    for into in (False, True):
        bd = make(es_list, decode_b=True)
        bufs, seen = [], []
        for _ in range(3):
            infos = [bd.stream_info(s) for s in range(S)]
            kinds = [[torch.zeros((n, i["coded_size"] * 3 // 2), dtype=torch.uint8, device="cuda") for i in infos],
                     [torch.zeros((n, i["height"], i["width"], 4), dtype=torch.uint8, device="cuda") for i in infos],
                     [torch.zeros((n, i["coded_size"] * 3 // 2), dtype=torch.int16, device="cuda") for i in infos],
                     [torch.zeros((n, i["coded_size"] // 256, 16), dtype=torch.uint8, device="cuda") for i in infos]]
            arrs = [(ctypes.c_void_p * S)(*[t.data_ptr() for t in ts]) for ts in kinds]
            info_out, n_frames = (Frame * (S * n))(), (ctypes.c_int32 * S)()
            torch.cuda.synchronize()
            if into:
                dst = FrameDst(*[ctypes.addressof(a) for a in arrs])
                got = bd.lib.jsmpeg_b200_batch_decode_frames_into(bd.handle, n, flags, ctypes.byref(dst), info_out, n_frames)
            else:
                got = bd.lib.jsmpeg_b200_batch_decode_frames(bd.handle, n, flags, *arrs, info_out, n_frames)
            bufs.append([[host(t) for t in ts] for ts in kinds])
            seen.append((got, list(n_frames), bytes(info_out), observed(bd, flags)))
        results.append((bufs, seen, bd.stats()))
        assert bd.last_error() is None
        bd.close()
    (ba, sa, ta), (bb, sb, tb) = results
    for x, y in zip(ba, bb):
        for u, v in zip(x, y):
            assert all(np.array_equal(p, q) for p, q in zip(u, v))
    for (ga, na, ia, oa), (gb, nb, ib, ob) in zip(sa, sb):
        assert (ga, na, ia) == (gb, nb, ib)
        for x, y in zip(oa, ob):
            for u, v in zip(x or [], y or []):
                assert same(u, v)
    assert {k: v for k, v in ta.items() if not k.endswith("_ms")} == {k: v for k, v in tb.items() if not k.endswith("_ms")}


def test_shared_geometry_is_one_tensor():
    """Two streams of one geometry, the second cut short: each new kind is one [S, n, ...] tensor, each stream's frames a
    view of its row, as many as its twin reconstructs."""
    es = stream("ffmpeg_320x240")
    es_list = [es, es[:len(es) // 6]]
    bd = make(es_list)
    out = bd.decode_frames(10, OUT_ACCUMULATED, planes=False, coefficients=True, accumulated=True)
    assert tuple(bd.last_frames_batch["coefficients"].shape) == (2, 10, 15, 20, 6, 8, 8)
    assert tuple(bd.last_frames_batch["accumulated"].shape) == (2, 10, 320 * 240 * 3 // 2, 4)
    assert "planes" not in bd.last_frames_batch
    for s in range(2):
        for kind in NEW:
            assert out[s][kind].data_ptr() == bd.last_frames_batch[kind][s].data_ptr()
        check(out[s], twin(make([es_list[s]]), 10), ("shared", s))
    assert out[0]["n_frames"] == 10 and 0 < out[1]["n_frames"] < 10
    bd.close()
