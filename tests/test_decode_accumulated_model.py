"""The accumulated maps of the playback path (decode() with OUT_ACCUMULATED, include/jsmpeg_b200.h) WITHOUT a GPU: the
serial model's sequential fold (tools/accumulate_model.py) -- one step per I/P picture the oracle's own decode()
reconstructs, from the map of the one before -- equals decode_accumulated's chain fold (oracle_chain) for every listed
I/P picture, with B pictures off and on; and a start on a P picture traces nothing back before it, up to the next I
picture."""
import numpy as np
import pytest

import accumulate_model
import chain_model
import helpers
from test_macroblock_index import GOLDEN, MINI_ENC, corpus_stream

STREAMS = GOLDEN + ["ffmpeg_320x240", "ffmpeg_1280x720"] + sorted(MINI_ENC)


def listed_maps(es):
    """{header start byte: decode_accumulated's map} of every I/P picture of the picture index (B pictures off)"""
    lib = helpers.oracle_lib()
    out = {}
    for e in chain_model.picture_index(es, False):
        if e["type"] in (1, 2):
            status, _, _, m = accumulate_model.oracle_chain(lib, es, e)
            assert status == 1, e
            out[e["byte_pos"] + 4] = m
    return out


@pytest.mark.parametrize("name", STREAMS)
def test_the_sequential_fold_equals_decode_accumulated(name):
    es = corpus_stream(name)
    want = listed_maps(es)
    assert want, name
    for decode_b in (False, True):
        got = accumulate_model.sequential(helpers.oracle_lib(), es, decode_b)
        starts = [start for start, _, _ in got]
        assert set(want) <= set(starts), (name, decode_b)  # (an unclosed tail picture is not listed)
        assert len(starts) - len(want) <= 1, (name, decode_b)
        for start, info, m in got:
            assert info.picture_type in (1, 2)
            if start in want:
                assert np.array_equal(m, want[start]), (name, decode_b, start)


@pytest.mark.parametrize("decode_b", [False, True])
def test_a_start_on_a_p_picture_traces_nothing_before_it(decode_b):
    """set_index to the first P picture after a key picture: that picture's predicted samples are untraced, every map
    up to the next I picture is the fold from nothing (fewer samples traced than decode_accumulated's, and no trace
    longer than the pictures since the start), and from the next I picture on the maps are decode_accumulated's."""
    es = corpus_stream("ffmpeg_320x240")
    want = listed_maps(es)
    index = chain_model.picture_index(es, False)
    first_p = next(e for e in index if e["type"] == 2)
    next_i = next(e for e in index if e["type"] == 1 and e["picture"] > first_p["picture"])
    got = accumulate_model.sequential(helpers.oracle_lib(), es, decode_b, index=first_p["byte_pos"] * 8)
    assert got[0][0] == first_p["byte_pos"] + 4 and got[0][1].picture_type == 2
    run = [(start, m) for start, _, m in got if start < next_i["byte_pos"] + 4]
    assert len(run) >= 2
    for n, (start, m) in enumerate(run):
        assert m[:, 3].max() <= n, (start, n)
        assert (m[:, 3] == -1).sum() > (want[start][:, 3] == -1).sum(), start
    assert (run[0][1][:, 3] <= 0).all() and not run[0][1][:, :3].any()
    after = [(start, m) for start, _, m in got if start >= next_i["byte_pos"] + 4 and start in want]
    assert len(after) >= 2
    for start, m in after:
        assert np.array_equal(m, want[start]), start
