"""tools/display_model.py against MPEG1Video(decodeBPictures, displayOrder) over the oracle library: the pictures the
host class renders, flush included, are the model's presentation of the oracle's coded-order pictures, picture for
picture, however the stream is cut into calls -- on the mini_enc I/P/B streams and the 720p B fixture, clean streams on
which every picture is reconstructed.  Without decode_b the model presents every picture at once and holds nothing."""
import os

import numpy as np
import pytest

import display_model
import helpers
from test_macroblock_index import MINI_ENC, corpus_stream

FIXTURE_720P = os.path.join(helpers.ROOT, "tests", "fixtures", "b_clip_1280x720.m1v")
NAMES = sorted(MINI_ENC) + ["b_clip_1280x720"]


@pytest.fixture
def oracle_b():
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(1)
    yield lib
    lib.oracle_set_decode_b(0)


def es_of(name):
    if name == "b_clip_1280x720":
        return open(FIXTURE_720P, "rb").read()
    pytest.importorskip("cv2")  # (mini_enc's scenes)
    return corpus_stream(name)


def coded(lib, es):
    """Every picture MPEG1Video decodes, in coded order: {"type", "temporal_reference", "y"}"""
    from jsmpeg_b200 import decoder
    d = decoder.MPEG1Video({"decodeFirstFrame": False, "decodeBPictures": True}, lib=lib)
    d.write(0, [es])
    out = []
    while d.decode():
        t, r = d.lastPicture()
        out.append({"type": t, "temporal_reference": r, "y": d.currentY.copy()})
    d.destroy()
    return out


def rendered(lib, es):
    """The luma planes MPEG1Video(decodeBPictures, displayOrder) renders, flush included"""
    from jsmpeg_b200 import decoder
    d = decoder.MPEG1Video({"decodeFirstFrame": False, "decodeBPictures": True, "displayOrder": True}, lib=lib)
    rec = decoder.PlaneRecorder()
    d.connect(rec)
    d.write(0, [es])
    while d.decode():
        pass
    d.flush()
    d.destroy()
    return [y for y, _, _ in rec.frames]


@pytest.mark.parametrize("name", NAMES)
def test_model_equals_the_display_order_renderer(oracle_b, name):
    es = es_of(name)
    pics = coded(oracle_b, es)
    assert all(p["type"] in (1, 2, 3) for p in pics) and any(p["type"] == 3 for p in pics)
    want = rendered(oracle_b, es)
    assert len(want) == len(pics)
    for calls in ([1], [2], [7], [60], [1, 2, 7, 60], [3, 1, 1, 5]):
        cuts = (calls * len(pics))[:len(pics)]
        per_call = display_model.present(pics, cuts)
        got = [p for call in per_call for p in call]
        assert len(got) == len(want), (name, calls)
        for k, (g, w) in enumerate(zip(got, want)):
            assert np.array_equal(g["y"], w), (name, calls, k)
        # a call presents at most one picture more than it reconstructs; the flush at most one
        assert all(len(c) <= n + 1 for c, n in zip(per_call, cuts)) and len(per_call[-1]) <= 1
        # one GOP, closed: temporal_reference counts the presentation positions
        assert [p["temporal_reference"] for p in got] == sorted(p["temporal_reference"] for p in got)


def test_without_decode_b_nothing_is_held():
    frames = [{"type": t} for t in (1, 2, 2, 1, 2)]
    m = display_model.DisplayModel(decode_b=False)
    assert m.call(frames[:2]) == frames[:2] and m.call(frames[2:]) == frames[2:]
    assert m.flush() == []


def test_held_pictures_cross_calls_and_drop():
    f = [{"type": t, "k": k} for k, t in enumerate((1, 3, 3, 2, 3, 3, 2))]
    m = display_model.DisplayModel()
    assert m.call(f[:1]) == []  # the I picture waits for its successor
    assert m.call(f[1:4]) == [f[1], f[2], f[0]]
    m.drop()  # (reset, a seek, a call in coded order)
    assert m.call(f[4:]) == [f[4], f[5]]
    assert m.flush() == [f[6]] and m.flush() == []
