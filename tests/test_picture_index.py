"""The picture index and the fresh-decoder result of tools/chain_model.py: literal index expectations (I/P streams,
skipped B / D / forward_f_code 0 pictures, open-GOP I/P/B streams with decode_b on and off), and the oracle run as the
fresh decoder of every listed I/P picture pinned to the stored reference decodes (tests/golden/reference/decodes.json)
wherever every picture of its chain codes every macroblock."""
import functools

import numpy as np
import pytest

import chain_model
import helpers
import intra_model
import synth_es
from jsmpeg_b200 import decoder


def fresh_decode(es, entry, decode_b=False):
    """The oracle fed chain_model.fresh_bytes(es, entry), decoding until it consumes picture k.  Returns (Y, Cr, Cb)
    of picture k or None when the decoder never consumes it, [(status, picture_type, n_present, error)] of every
    picture it consumed, and mb_size."""
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(1 if decode_b else 0)
    try:
        d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=lib)
        rec = decoder.PlaneRecorder()
        d.connect(rec)
        d.write(0.0, [chain_model.fresh_bytes(es, entry)])
        target = chain_model.target_start_byte(es, entry)
        infos, at = [], None
        while d.decode():
            info = lib.oracle_last_picture_info(d.decoder).contents
            infos.append((info.status, info.picture_type, info.n_present, info.error))
            at = info.start_byte
            if at >= target:
                break
        mb_size = lib.oracle_seq_params(d.decoder).contents.mb_size
        planes = rec.frames[-1] if at == target else None
        d.destroy()
    finally:
        lib.oracle_set_decode_b(0)
    return planes, infos, mb_size


def ffmpeg_es(w, h, n, seed=1234):
    return b"".join(p for _, p in helpers.clip_packets(w, h, n, seed=seed))


@functools.lru_cache(maxsize=None)
def open_gop_clip():
    """mini_enc I/P/B, two B pictures per reference, an I picture every second reference: coded order
    I P B B I B B P B B I B B -- the B pictures behind each later I picture refer to the GOP before (open GOP)."""
    pytest.importorskip("cv2")
    import mini_enc
    return mini_enc.make_b_clip(176, 144, 13, 2, gop_refs=2)[0]


def index_triples(es, decode_b=False):
    return [(e["picture"], e["type"], e["chain_start"]) for e in chain_model.picture_index(es, decode_b)]


def test_i_p_stream_literal():
    # rows_ip: I P P P I P P P I P -- every P picture chains from the I picture before it
    assert index_triples(synth_es.make_case("rows_ip")) == \
        [(0, 1, 0), (1, 2, 0), (2, 2, 0), (3, 2, 0), (4, 1, 4), (5, 2, 4), (6, 2, 4), (7, 2, 4), (8, 1, 8), (9, 2, 8)]
    # FFmpeg, GOP 12: the last picture is never closed (no sequence end code)
    es = ffmpeg_es(320, 240, 24)
    assert index_triples(es) == [(k, 1 if k % 12 == 0 else 2, k // 12 * 12) for k in range(23)]


def test_ignored_pictures_are_not_listed():
    """ignored_pictures_userdata: I P P(forward_f_code 0) P I P D P I P D P -- the f_code-0 P picture and the D
    pictures are consumed by decode() and never reconstructed, so they are not listed (with decode_b on or off);
    they are no references either."""
    es = synth_es.make_case("ignored_pictures_userdata")
    want = [(0, 1, 0), (1, 2, 0), (3, 2, 0), (4, 1, 4), (5, 2, 4), (7, 2, 4), (8, 1, 8), (9, 2, 8), (11, 2, 8)]
    assert index_triples(es, False) == index_triples(es, True) == want
    pics = [p for p in intra_model.prefixes(es) if es[p + 3] == 0]
    assert chain_model.picture_type(es, pics[2]) == 2 and chain_model.header_bits(es, pics[2], 30, 3) == 0
    assert chain_model.picture_type(es, pics[6]) == chain_model.picture_type(es, pics[10]) == 4


def test_b_stream_first_b_pictures_have_no_chain_start():
    """b_rows: I B B P B B I B B P B B I.  Without decode_b no B picture is listed.  With it, the first two B
    pictures (one reference before them) have no chain start; the B pictures behind the second I picture chain
    from the first one."""
    es = synth_es.make_case("b_rows")
    assert index_triples(es, False) == [(0, 1, 0), (3, 2, 0), (6, 1, 6), (9, 2, 6), (12, 1, 12)]
    assert index_triples(es, True) == [(0, 1, 0), (3, 2, 0), (4, 3, 0), (5, 3, 0), (6, 1, 6), (7, 3, 0), (8, 3, 0),
                                       (9, 2, 6), (10, 3, 6), (11, 3, 6), (12, 1, 12)]


def test_open_gop_literal():
    es = open_gop_clip()
    assert index_triples(es, False) == [(0, 1, 0), (1, 2, 0), (4, 1, 4), (7, 2, 4), (10, 1, 10)]
    # the B pictures 5, 6 (after I 4) and 11, 12 (after I 10) refer to P 1 / P 7 of the GOP before: one GOP back
    assert index_triples(es, True) == [(0, 1, 0), (1, 2, 0), (2, 3, 0), (3, 3, 0), (4, 1, 4), (5, 3, 0), (6, 3, 0),
                                       (7, 2, 4), (8, 3, 4), (9, 3, 4), (10, 1, 10), (11, 3, 4), (12, 3, 4)]


@pytest.mark.parametrize("name", sorted(synth_es.CASES) + sorted(synth_es.B_CASES))
@pytest.mark.parametrize("decode_b", [False, True])
def test_the_intra_index_is_the_type_1_entries(name, decode_b):
    es = synth_es.make_case(name)
    entries = chain_model.picture_index(es, decode_b)
    assert [(e["picture"], e["byte_pos"], e["temporal_reference"], e["close"]) for e in entries if e["type"] == 1] == \
        [(e["picture"], e["byte_pos"], e["temporal_reference"], e["close"]) for e in intra_model.intra_index(es)]
    assert all(e["chain_start"] == e["picture"] for e in entries if e["type"] == 1)
    assert all(e["chain_start"] < e["picture"] for e in entries if e["type"] != 1)


def test_a_tail_picture_is_listed_once_its_closing_code_arrives():
    es = synth_es.make_case("rows_ip")
    for e in chain_model.picture_index(es):
        for cut in (e["close"], e["close"] + 3):
            assert e["picture"] not in [x["picture"] for x in chain_model.picture_index(es[:cut])]
        assert e in chain_model.picture_index(es[:e["close"] + 4])


FFMPEG = {"ffmpeg_320x240": (320, 240, 24), "ffmpeg_1280x720": (1280, 720, 6)}
PINNED = sorted(synth_es.CASES) + list(FFMPEG)


@functools.lru_cache(maxsize=None)
def stream(name):
    return ffmpeg_es(*FFMPEG[name]) if name in FFMPEG else synth_es.make_case(name)


@pytest.mark.parametrize("name", PINNED)
def test_fresh_decoder_matches_the_reference_where_every_macroblock_is_coded(name):
    """Pinned to the reference: for every listed picture whose chain (j through k) codes every macroblock, the fresh
    decode from the chain start has the stored reference hash of picture k -- what decode() gives there."""
    es = stream(name)
    want = helpers.reference_decode([(0.0, es)], "whole")["fnv1a64"]
    full = 0
    for e in chain_model.picture_index(es):
        planes, infos, mb_size = fresh_decode(es, e)
        assert planes is not None and infos[-1][:2] == (1, e["type"]) and infos[-1][3] == 0, (name, e["picture"])
        if all(n_present == mb_size for status, _, n_present, _ in infos if status == 1):
            assert helpers.frame_hashes([planes])[0] == want[e["picture"]], (name, e["picture"])
            full += e["type"] == 2
    if name in FFMPEG or name in ("fcodes_fullpel", "rows_ip", "escapes_matrices"):
        assert full >= 1, name  # some P picture took this path


def test_open_gop_b_pictures_equal_the_sequential_decode():
    """decode_b on: every listed picture of the open-GOP clip (every picture codes every macroblock) decoded fresh
    from its chain start equals the oracle's own decode() of the whole clip at that point."""
    es = open_gop_clip()
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(1)
    try:
        frames, _, d = helpers.decode_all(lib, [(0, es)])
        d.destroy()
    finally:
        lib.oracle_set_decode_b(0)
    entries = chain_model.picture_index(es, True)
    assert sum(e["type"] == 3 for e in entries) == 8
    for e in entries:
        planes, infos, mb_size = fresh_decode(es, e, decode_b=True)
        assert all(n == mb_size for _, _, n, _ in infos)
        for p, q in zip(planes, frames[e["picture"]]):
            assert np.array_equal(p, q), e["picture"]
