"""decode_frames_display and flush_frames (include/jsmpeg_b200.h) against a twin batch that runs decode_frames(1, flags)
per picture with every kind, its frames put in presentation order by tools/display_model.py across the calls and the
flush: every kind and every info field byte for byte -- the B fixture, the mini_enc I/P/B streams and an .mpg with B
pictures with the slice walk on and off cut into calls of 1, 2, 7 and 60; damaged B streams; decode_b off, where the
call is decode_frames_into and nothing is held; mixed sizes with an odd display size, NULL entries and short streams;
holds across round boundaries; the batch state against decode(n, flags); holds dropped by reset, seek_pictures,
set_index and decode(); flush_frames with and without holds; the -2 rules; and presentation order on closed GOPs."""
import ctypes

import numpy as np
import pytest

import chain_model
import display_model
import mini_ps
import synth_es
from jsmpeg_b200.batch import (OUT_ACCUMULATED, OUT_DEVICE, OUT_HOST, OUT_MACROBLOCKS, OUT_RESIDUALS, OUT_RGBA, Frame,
                               FrameDst)
from test_gpu_decode_frames import ALL, make, observed, same
from test_gpu_intra import _damage, host
from test_gpu_macroblocks import stream
from test_macroblock_index import MINI_ENC

pytestmark = pytest.mark.gpu
KINDS = ("planes", "rgba", "residuals", "macroblocks", "coefficients", "accumulated")
INFO = ("byte_pos", "type", "temporal_reference", "n_present", "error")
CUTS = ([1], [2], [7], [60])


def asked(flags, kinds=KINDS):
    """decode_frames' keyword arguments for `kinds` (map frames only under OUT_ACCUMULATED)"""
    return {k: k in kinds and (k != "accumulated" or bool(flags & OUT_ACCUMULATED)) for k in KINDS}


def frames_of(o):
    """One stream's result of decode_frames / flush_frames as a list of frames: info fields and host arrays"""
    return [{**{k: o["info"][j][k] for k in INFO}, **{k: host(o[k][j]) for k in KINDS if o.get(k) is not None}}
            for j in range(o["n_frames"])]


def coded_steps(es_list, n_steps, flags, kinds=KINDS, ps=False, **opts):
    """Per stream, per decode_frames(1, flags) of a twin batch: the frames it reconstructs (coded order)"""
    tw = make(es_list, ps, **opts)
    steps = [[] for _ in es_list]
    for _ in range(n_steps):
        for s, o in enumerate(tw.decode_frames(1, flags, **asked(flags, kinds))):
            steps[s].append(frames_of(o))
    assert tw.last_error() is None
    tw.close()
    return steps


def run_display(bd, calls, flags, kinds=KINDS, flush=True):
    """Per stream, per call of decode_frames(n, flags, display_order=True) (then flush_frames): its frames"""
    got = [[] for _ in range(bd.n_streams)]
    for n in calls:
        for s, o in enumerate(bd.decode_frames(n, flags, display_order=True, **asked(flags, kinds))):
            assert o["n_frames"] <= n + 1
            got[s].append(frames_of(o))
    if flush:
        for s, o in enumerate(bd.flush_frames(**asked(flags, kinds))):
            assert o["n_frames"] <= 1
            got[s].append(frames_of(o))
    return got


def expect(steps, calls, decode_b=True, flush=True):
    """The model's presentation of one stream's twin `steps`, cut into `calls`, then flushed"""
    m, out, at = display_model.DisplayModel(decode_b), [], 0
    for n in calls:
        out.append(m.call([f for step in steps[at:at + n] for f in step]))
        at += n
    if flush:
        out.append(m.flush())
    return out


def assert_same(got, want, label):
    assert [len(c) for c in got] == [len(c) for c in want], label
    for i, (gc, wc) in enumerate(zip(got, want)):
        for j, (g, w) in enumerate(zip(gc, wc)):
            assert g.keys() == w.keys(), (label, i, j)
            for k in g:
                assert same(g[k], w[k]), (label, i, j, k)


def calls_for(cut, total):
    return (cut * total)[:max(1, -(-total // cut[0]))]


def source(name):
    if name == "mpg":
        return mini_ps.mux(stream("b_clip_1280x720"), form="mpg")[0], True
    return stream(name), False


@pytest.mark.parametrize("name", ["b_clip_1280x720", "mpg"] + sorted(MINI_ENC))
def test_every_frame_in_presentation_order(name):
    es, ps = source(name)
    total = len(chain_model.picture_positions(stream("b_clip_1280x720") if ps else es)) + 2
    flags = OUT_ACCUMULATED | OUT_RGBA
    for slice_walk in (0, 1):
        steps = coded_steps([es], total, flags, ps=ps, decode_b=True, slice_walk=slice_walk)[0]
        assert any(f["type"] == 3 for st in steps for f in st)
        for cut in CUTS:
            calls = calls_for(cut, total)
            bd = make([es], ps, decode_b=True, slice_walk=slice_walk)
            got = run_display(bd, calls, flags)[0]
            assert_same(got, expect(steps, calls), (name, slice_walk, cut))
            assert bd.last_error() is None
            bd.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_damaged_b_streams(seed):
    import macroblock_model
    errors = 0
    for case in ("b_one_slice_fcodes", "b_rows"):
        clean = synth_es.make_case(case)
        es = _damage(clean, macroblock_model.macroblock_index(clean)[1::2], seed, flips=3)
        total = len(chain_model.picture_positions(es)) + 1
        steps = coded_steps([es], total, OUT_ACCUMULATED, decode_b=True)[0]
        for cut in ([1], [3], [60]):
            calls = calls_for(cut, total)
            got = run_display(make([es], decode_b=True), calls, OUT_ACCUMULATED)[0]
            assert_same(got, expect(steps, calls), (case, seed, cut))
        errors += sum(f["error"] != 0 for st in steps for f in st)
    assert errors > 0


def test_without_decode_b_the_call_is_decode_frames_into():
    """decode_b off: each call gives decode_frames_into's frames in its order, and flush_frames finds nothing held."""
    for name in ("b_clip_1280x720", "mini_enc_open_gop", "ffmpeg_320x240"):
        es = stream(name)
        total = len(chain_model.picture_positions(es)) + 1
        calls = calls_for([3], total)
        a, b = make([es]), make([es])
        for n in calls:
            got = frames_of(a.decode_frames(n, OUT_ACCUMULATED, display_order=True, **asked(OUT_ACCUMULATED))[0])
            want = frames_of(b.decode_frames(n, OUT_ACCUMULATED, **asked(OUT_ACCUMULATED))[0])
            assert_same([got], [want], (name, n))
        assert [o["n_frames"] for o in a.flush_frames()] == [0]
        a.close()
        b.close()


def test_mixed_streams_null_entries_and_short_streams():
    """Streams of different coded sizes and an odd display size in one batch, each kind with a NULL entry, streams that
    run out at different counts: each stream's frames are its twin's in presentation order, a NULL entry gets nothing,
    and memory past n_frames is untouched."""
    import torch
    from test_gpu_macroblocks import MIXED
    es_list = [stream(name) for name in MIXED + ["b_clip_1280x720"]]
    es_list.append(synth_es.SynthStream(synth_es.Knobs(width=101, height=51, pictures=7, gop=3, slices="random", b_frames=1),
                                        19).generate())
    S, flags = len(es_list), OUT_ACCUMULATED
    calls = [5, 9, 40]
    steps = coded_steps(es_list, sum(calls), flags, decode_b=True)
    bd = make(es_list, decode_b=True)
    infos = [bd.stream_info(s) for s in range(S)]
    assert any(i["width"] & 1 or i["height"] & 1 for i in infos)
    shapes = {"planes": (lambda i: (i["coded_size"] * 3 // 2,), torch.uint8), "rgba": (lambda i: (i["height"], i["width"], 4), torch.uint8),
              "residuals": (lambda i: (i["coded_size"] * 3 // 2,), torch.int16),
              "macroblocks": (lambda i: (i["coded_size"] // 256, 16), torch.uint8),
              "coefficients": (lambda i: (i["coded_size"] // 256, 384), torch.int16),
              "accumulated": (lambda i: (i["coded_size"] * 3 // 2, 4), torch.int16)}
    field = {"planes": "planes", "rgba": "rgba", "residuals": "res", "macroblocks": "mb", "coefficients": "coef", "accumulated": "acc"}
    null = {k: i % S for i, k in enumerate(KINDS)}  # per kind the stream whose entry is NULL
    got = [[] for _ in range(S)]
    for n in calls:
        bufs = {k: [None if s == null[k] else torch.full((n + 1, *shapes[k][0](infos[s])), 0x5A, dtype=shapes[k][1], device="cuda")
                    for s in range(S)] for k in KINDS}
        arr = {k: (ctypes.c_void_p * S)(*[None if t is None else t.data_ptr() for t in bufs[k]]) for k in KINDS}
        dst = FrameDst(**{field[k]: ctypes.addressof(arr[k]) for k in KINDS})
        info_out, n_frames = (Frame * (S * (n + 1)))(), (ctypes.c_int32 * S)()
        torch.cuda.synchronize()
        r = bd.lib.jsmpeg_b200_batch_decode_frames_display(bd.handle, n, flags, ctypes.byref(dst), info_out, n_frames)
        assert r > 0 and bd.last_error() is None
        for s in range(S):
            f = n_frames[s]
            frames = []
            for j in range(f):
                row = info_out[s * (n + 1) + j]
                fr = {"byte_pos": row.byte_pos, "type": row.picture_type, "temporal_reference": row.temporal_reference,
                      "n_present": row.n_present, "error": row.error}
                for k in KINDS:
                    if bufs[k][s] is not None:
                        fr[k] = host(bufs[k][s][j]).reshape(-1)
                frames.append(fr)
            for k in KINDS:
                if bufs[k][s] is not None:
                    assert (host(bufs[k][s][f:]) == 0x5A).all(), (s, k)
            got[s].append(frames)
    assert len({sum(len(c) for c in g) for g in got}) > 2  # streams end at different counts
    bd.close()
    for s in range(S):
        want = expect(steps[s], calls, flush=False)
        for c, (gc, wc) in enumerate(zip(got[s], want)):
            assert len(gc) == len(wc), (s, c)
            for g, w in zip(gc, wc):
                assert set(g) == {k for k in w if k in INFO or null.get(k) != s}, (s, c)
                for k in g:
                    assert np.array_equal(np.asarray(g[k]).reshape(-1), np.asarray(w[k]).reshape(-1)), (s, c, k)


def test_holds_cross_round_boundaries():
    """max_slots=3 cuts each call into many rounds: held pictures go through the store at every round's end."""
    names = ["b_rows", "mini_enc_open_gop", "b_clip_1280x720", "ffmpeg_320x240"]
    es_list = [stream(name) for name in names]
    flags = OUT_ACCUMULATED | OUT_RGBA | OUT_RESIDUALS
    calls = [7, 1, 12, 3, 20]
    steps = coded_steps(es_list, sum(calls), flags, decode_b=True)
    bd = make(es_list, decode_b=True, max_slots=3)
    got = run_display(bd, calls, flags)
    for s, name in enumerate(names):
        assert_same(got[s], expect(steps[s], calls), name)
    assert bd.last_error() is None
    bd.close()


@pytest.mark.parametrize("flags", [OUT_DEVICE, OUT_HOST, OUT_RGBA, OUT_MACROBLOCKS, OUT_ACCUMULATED, OUT_RESIDUALS, ALL])
def test_batch_state_equals_decode(flags):
    """decode_frames_display(n, flags) with every kind, call after call, against a third twin's decode(n, flags): every
    stats field but kernel_launches and the device times, and all a reader sees (the RGBA and residual of the last
    reconstructed picture, held or not)."""
    from test_gpu_macroblocks import MIXED
    es_list = [stream(name) for name in MIXED + ["b_clip_1280x720"]]
    runs, stats = [], []
    for display in (False, True):
        bd = make(es_list, decode_b=True)
        seen = []
        for n in [1, 3, 2, 5, 4, 8] * 2:
            if display:
                r = bd.decode_frames(n, flags, display_order=True, **asked(flags))
                seen.append(observed(bd, flags))
            else:
                bd.decode(n, flags)
                seen.append(observed(bd, flags))
        runs.append(seen)
        stats.append(bd.stats())
        assert bd.last_error() is None
        bd.close()
    for a, b in zip(*runs):
        for x, y in zip(a, b):
            assert (x is None) == (y is None)
            for u, v in zip(x or [], y or []):
                assert same(u, v)
    off, on = stats
    for key in off:
        if not key.endswith("_ms") and key != "kernel_launches":
            assert on[key] == off[key], key


@pytest.mark.parametrize("op", ["reset", "seek", "set_index", "decode"])
def test_holds_are_dropped(op):
    es = stream("b_clip_1280x720")
    bd = make([es], decode_b=True)
    first = bd.decode_frames(4, display_order=True)[0]
    assert first["n_frames"] == 3  # I B B presented after P arrives; P held
    if op == "reset":
        bd.reset()
        bd.write(0, es)
    elif op == "seek":
        entries = chain_model.picture_index(es, True)
        assert bd.seek_pictures([(0, entries[len(entries) // 2]["picture"])]) == 1
    elif op == "set_index":
        bd.set_index(0, bd.get_index(0))
    else:
        bd.decode(1)
    assert [o["n_frames"] for o in bd.flush_frames()] == [0]
    bd.close()


def test_flush_with_and_without_holds():
    es = stream("b_clip_1280x720")
    steps = coded_steps([es], 4, OUT_DEVICE, decode_b=True)[0]
    bd = make([es], decode_b=True)
    assert [o["n_frames"] for o in bd.flush_frames()] == [0]  # nothing held yet
    bd.decode_frames(4, display_order=True)
    before = observed(bd, OUT_RGBA)
    fl = bd.flush_frames(rgba=False)[0]
    held = [f for st in steps for f in st if f["type"] != 3][-1]
    assert fl["n_frames"] == 1 and fl["info"][0]["byte_pos"] == held["byte_pos"]
    assert np.array_equal(host(fl["planes"][0]), held["planes"])
    for u, v in zip(before[0], observed(bd, OUT_RGBA)[0]):
        assert same(u, v)
    assert [o["n_frames"] for o in bd.flush_frames()] == [0]  # released
    bd.close()


def test_refusals_change_nothing():
    import torch
    es_list = [stream("b_clip_1280x720"), stream("rows_ip")]
    bd = make(es_list, decode_b=True)
    bd.decode_frames(3, OUT_ACCUMULATED | OUT_RGBA, display_order=True, planes=True, macroblocks=True)  # holds planes + entries
    before = observed(bd, OUT_RGBA)
    stats = bd.stats()
    t = torch.zeros(1 << 24, dtype=torch.uint8, device="cuda")
    good, bad = t.data_ptr(), t.data_ptr() + 8
    n_frames = (ctypes.c_int32 * 2)(7, 7)
    f = bd.lib.jsmpeg_b200_batch_decode_frames_display
    assert f(bd.handle, 1, OUT_DEVICE, None, None, n_frames) == -2  # NULL dst
    assert f(bd.handle, -1, OUT_DEVICE, ctypes.byref(FrameDst()), None, n_frames) == -2
    arr = (ctypes.c_void_p * 2)(good, bad)
    assert f(bd.handle, 1, OUT_DEVICE, ctypes.byref(FrameDst(planes=ctypes.addressof(arr))), None, n_frames) == -2
    one = (ctypes.c_void_p * 2)(None, good)
    assert f(bd.handle, 1, OUT_DEVICE, ctypes.byref(FrameDst(acc=ctypes.addressof(one))), None, n_frames) == -2  # no flag
    held_only = (ctypes.c_void_p * 2)(good, None)
    assert f(bd.handle, 1, OUT_DEVICE, ctypes.byref(FrameDst(res=ctypes.addressof(held_only))), None, n_frames) == -2
    fl = bd.lib.jsmpeg_b200_batch_flush_frames
    assert fl(bd.handle, None, None, n_frames) == -2
    assert fl(bd.handle, ctypes.byref(FrameDst(rgba=ctypes.addressof(held_only))), None, n_frames) == -2
    assert list(n_frames) == [7, 7]
    for u, v in zip(before, observed(bd, OUT_RGBA)):
        for x, y in zip(u or [], v or []):
            assert same(x, y)
    assert bd.stats() == stats
    # the hold survived every refusal: planes and entries are still there to flush
    out = bd.flush_frames(planes=True, macroblocks=True)
    assert out[0]["n_frames"] == 1
    assert bd.last_error() is None
    bd.close()


def test_closed_gops_are_presented_in_temporal_order():
    """On clean one-GOP streams the frames come in presentation order: temporal_reference counts 0, 1, 2, ... across
    calls and the flush, and every reconstructed picture is presented once."""
    for name in ("b_clip_1280x720", "mini_enc_fcodes_2_4_fullpel_bwd"):
        es = stream(name)
        total = len(chain_model.picture_positions(es)) + 1
        bd = make([es], decode_b=True)
        frames = [f for call in run_display(bd, calls_for([5], total), OUT_DEVICE, kinds=())[0] for f in call]
        bd.close()
        assert [f["temporal_reference"] for f in frames] == list(range(len(frames))), name
        assert len(frames) == sum(len(st) for st in coded_steps([es], total, OUT_DEVICE, kinds=(), decode_b=True)[0])
