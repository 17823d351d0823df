"""The seek model of tools/chain_model.py (seek_start, seek_bytes) against the oracle: for every listed picture k of the
golden, FFmpeg and mini_enc I/P/B streams, with decode_b off and on, the oracle fed the seek bytes and decoded until it
consumes k goes on picture for picture -- planes, consumed picture and translated bit index -- exactly as the
oracle's sequential decode() of the whole stream, wherever the stream starts with an I picture and every picture from
the seek chain start on codes every macroblock.  An open-GOP clip sought at an I picture pins why the seek chain start
of an I picture reaches one reference back under decode_b."""
import numpy as np
import pytest

import chain_model
import helpers
import intra_model
import synth_es
from jsmpeg_b200 import decoder
from test_picture_index import ffmpeg_es, open_gop_clip


def oracle_run(data, decode_b):
    """decode() of the oracle over `data` until it returns false: per consumed picture (start byte of its header, bit
    index after it, its planes, n_present), and mb_size."""
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(1 if decode_b else 0)
    try:
        d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=lib)
        rec = decoder.PlaneRecorder()
        d.connect(rec)
        d.write(0.0, [data])
        steps = []
        while d.decode():
            info = lib.oracle_last_picture_info(d.decoder).contents
            steps.append((info.start_byte, d.bufferGetIndex(), rec.frames[-1], info.status, info.n_present))
        mb_size = lib.oracle_seq_params(d.decoder).contents.mb_size if steps else 0
        d.destroy()
    finally:
        lib.oracle_set_decode_b(0)
    return steps, mb_size


def seek_run(es, entry, decode_b):
    """The oracle fed chain_model.seek_bytes, from the decode() that consumes picture k to the end, translated to the
    positions of `es`: [(start byte, bit index, planes)]; and whether every picture it decoded codes every
    macroblock.  None when it never consumes k."""
    data = chain_model.seek_bytes(es, entry, decode_b)
    delta = len(es) - len(data)
    steps, mb_size = oracle_run(data, decode_b)
    at = next((i for i, s in enumerate(steps) if s[0] + delta == entry["byte_pos"] + 4), None)
    if at is None:
        return None
    full = all(n == mb_size for _, _, _, status, n in steps if status == 1)
    return [(b + delta, idx + 8 * delta, planes) for b, idx, planes, _, _ in steps[at:]], full


def assert_same_run(got, want, what):
    assert len(got) == len(want), what
    for (b, idx, planes), (wb, widx, wplanes) in zip(got, want):
        assert (b, idx) == (wb, widx), what
        for p, q in zip(planes, wplanes):
            assert np.array_equal(p, q), what


STREAMS = sorted(synth_es.CASES) + sorted(synth_es.B_CASES) + ["ffmpeg_320x240", "ffmpeg_1280x720", "open_gop"]
FULL = {"rows_ip", "fcodes_fullpel", "escapes_matrices", "b_rows", "ffmpeg_320x240", "ffmpeg_1280x720", "open_gop"}


def stream(name):
    if name == "open_gop":
        return open_gop_clip()
    if name.startswith("ffmpeg_"):
        return ffmpeg_es(*{"ffmpeg_320x240": (320, 240, 24), "ffmpeg_1280x720": (1280, 720, 6)}[name])
    return synth_es.make_case(name)


@pytest.mark.parametrize("decode_b", [False, True])
@pytest.mark.parametrize("name", STREAMS)
def test_a_seek_goes_on_as_the_sequential_decode(name, decode_b):
    es = stream(name)
    sequential, _ = oracle_run(es, decode_b)
    pics = chain_model.picture_positions(es)
    starts_with_i = chain_model.picture_type(es, pics[0]) == 1
    by_start = {b: i for i, (b, _, _, _, _) in enumerate(sequential)}
    checked = 0
    for e in chain_model.picture_index(es, decode_b):
        j = chain_model.seek_start(es, e, decode_b)
        assert j <= e["chain_start"] and (j == e["chain_start"] or e["type"] == 1)
        run = seek_run(es, e, decode_b)
        assert run is not None, (name, e["picture"])  # clean streams: the fresh decoder always consumes k
        got, full = run
        if not (starts_with_i and full):
            continue
        want = [(b, idx, planes) for b, idx, planes, _, _ in sequential[by_start[e["byte_pos"] + 4]:]]
        assert_same_run(got, want, (name, decode_b, e["picture"]))
        checked += 1
    if name in FULL:
        assert checked == len(chain_model.picture_index(es, decode_b)) > 0, name


def test_seek_start_literal():
    es = open_gop_clip()  # I P B B I B B P B B I B B
    starts = {e["picture"]: chain_model.seek_start(es, e, True) for e in chain_model.picture_index(es, True)}
    assert starts == {0: 0, 1: 0, 2: 0, 3: 0, 4: 0, 5: 0, 6: 0, 7: 4, 8: 4, 9: 4, 10: 4, 11: 4, 12: 4}
    # without decode_b an I picture is its own seek chain start
    assert all(chain_model.seek_start(es, e, False) == e["chain_start"] for e in chain_model.picture_index(es, False))
    b_rows = synth_es.make_case("b_rows")  # I B B P B B I B B P B B I: the first I picture has no reference before it
    assert {e["picture"]: chain_model.seek_start(b_rows, e, True) for e in chain_model.picture_index(b_rows, True)
            if e["type"] == 1} == {0: 0, 6: 0, 12: 6}


def test_open_gop_seek_at_an_i_picture_needs_one_reference_back():
    """Sought at I picture 4 of the open-GOP clip with decode_b: from the seek chain start (0) the B pictures 5 and 6
    after it equal the sequential decode; from the I picture itself they would not (their forward reference, P 1,
    would be a zeroed set)."""
    es = open_gop_clip()
    entry = next(e for e in chain_model.picture_index(es, True) if e["picture"] == 4)
    sequential, _ = oracle_run(es, True)
    want = [(b, idx, planes) for b, idx, planes, _, _ in sequential[4:]]
    got, full = seek_run(es, entry, True)
    assert full
    assert_same_run(got, want, "seek chain start 0")
    own = seek_run(es, dict(entry, type=2, chain_start=4), True)[0]  # (type 2: seek_start keeps chain_start)
    assert own[0][1] == want[0][1] and np.array_equal(own[0][2][0], want[0][2][0])  # picture 4 itself is the same
    assert not all(np.array_equal(p, q) for p, q in zip(own[1][2], want[1][2]))  # B picture 5 is not


def test_seek_bytes_run_to_the_end_of_the_buffer():
    es = synth_es.make_case("rows_ip")
    for e in chain_model.picture_index(es):
        data = chain_model.seek_bytes(es, e)
        start = chain_model.picture_positions(es)[chain_model.seek_start(es, e)]
        h = intra_model.first_sequence_header(es)[0]
        assert data.endswith(es[start:]) and data.startswith(es[h:h + 4])
        assert len(data) - (len(es) - start) == len(chain_model.fresh_bytes(es, e)) - (e["close"] + 4 - e["chain_start_pos"])
