"""The key-picture index and the fresh-decoder result of tools/intra_model.py: literal index expectations on the
synthetic corner streams and FFmpeg clips, and the fresh-decoder pictures pinned to the stored reference decodes
(tests/golden/reference/decodes.json) wherever a picture codes every macroblock."""
import ctypes
import functools

import numpy as np
import pytest

import helpers
import intra_model
import synth_es
from jsmpeg_b200 import decoder


def fresh_decode(es, entry):
    """The oracle fed fresh_bytes: (Y, Cr, Cb), picture_info, macroblock records [mb_size, 16], mb_width."""
    lib = helpers.oracle_lib()
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=lib)
    rec = decoder.PlaneRecorder()
    d.connect(rec)
    d.write(0.0, [intra_model.fresh_bytes(es, entry)])
    assert d.decode()
    sp = lib.oracle_seq_params(d.decoder).contents
    info = lib.oracle_last_picture_info(d.decoder).contents
    hdr = np.ctypeslib.as_array(ctypes.cast(lib.oracle_last_mb_records(d.decoder), ctypes.POINTER(ctypes.c_uint8)),
                                shape=(sp.mb_size, 16)).copy()
    out = (rec.frames[0], (info.status, info.picture_type, info.n_present, info.error), hdr, sp.mb_width)
    d.destroy()
    return out


def random_stream(seed):
    """The random syntax streams of test_oracle_vs_reference.py (same knobs, same seeds)."""
    k = synth_es.Knobs(width=int(16 * (2 + seed)), height=int(16 * (1 + seed % 3)) + 2 * seed, pictures=7, gop=3,
                       slices=["one", "rows", "random"][seed % 3], slice_gap_prob=0.2, stuffing_prob=0.2,
                       skip_prob=0.3, f_codes=(1, 2, 3, 4), full_pel_prob=0.3, escape_prob=0.3,
                       custom_matrices=bool(seed & 1), extension_user_data=True, ignored_pictures=bool(seed & 2))
    return synth_es.SynthStream(k, 1000 + seed).generate()


FFMPEG = {"ffmpeg_320x240": (320, 240, 24), "ffmpeg_1280x720": (1280, 720, 6)}
PINNED = sorted(synth_es.CASES) + [f"random_{seed}" for seed in range(6)] + list(FFMPEG)


@functools.lru_cache(maxsize=None)
def stream(name):
    """Every stream whose reference decode is stored: synth_es.CASES, the random streams, two FFmpeg clips."""
    if name in FFMPEG:
        return b"".join(p for _, p in helpers.clip_packets(*FFMPEG[name]))
    if name.startswith("random_") and name[7:].isdigit():
        return random_stream(int(name[7:]))
    return synth_es.make_case(name)


def pinned_streams():
    return [(name, stream(name)) for name in PINNED]


EXPECTED = {
    "escapes_matrices": [0, 4], "fcodes_fullpel": [0, 5], "i_only_320x240": list(range(8)),
    "ignored_pictures_userdata": [0, 4, 8], "odd_size": [0, 3], "random_slices_gaps": [0, 5], "rows_ip": [0, 4, 8],
    "skips_stuffing_escape_mba": [0, 4],
    # TS-demuxed FFmpeg encodes (GOP 12) end without a sequence end code: their last picture is never closed
    "ffmpeg_320x240": [0, 12], "ffmpeg_1280x720": [0],
}


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_index_literal(name):
    es = stream(name)
    assert [e["picture"] for e in intra_model.intra_index(es)] == EXPECTED[name]


def test_user_data_and_extensions_after_a_picture_header_do_not_close_it():
    """In ignored_pictures_userdata and the random streams, some listed picture has an extension or user data between
    its header and its first slice; it is listed, and its closing code is neither."""
    seen = 0
    for name, es in pinned_streams():
        codes = intra_model.prefixes(es)
        for e in intra_model.intra_index(es):
            after = [es[q + 3] for q in codes if e["byte_pos"] < q < e["close"]]
            assert all(0x01 <= c <= 0xAF or c in (0xB2, 0xB5) for c in after), name
            assert es[e["close"] + 3] not in (0xB2, 0xB5)
            if after and after[0] in (0xB2, 0xB5):
                seen += 1
                # cut right after the user data / extension: nothing closes the picture yet
                first_slice = next(q for q in codes if q > e["byte_pos"] and 0x01 <= es[q + 3] <= 0xAF)
                assert e["picture"] not in [x["picture"] for x in intra_model.intra_index(es[:first_slice + 4])]
    assert seen >= 2


@pytest.mark.parametrize("name", ["i_only_320x240", "rows_ip", "ffmpeg_320x240"])
def test_a_tail_picture_is_listed_once_its_closing_code_arrives(name):
    es = stream(name)
    for e in intra_model.intra_index(es):
        close = e["close"]
        for cut in (close, close + 1, close + 3):  # the last slice is complete, the code is not
            assert e["picture"] not in [x["picture"] for x in intra_model.intra_index(es[:cut])], (name, e["picture"], cut)
        again = [x for x in intra_model.intra_index(es[:close + 4]) if x["picture"] == e["picture"]]
        assert again == [e]


def test_no_sequence_header_no_index():
    es = synth_es.make_case("i_only_320x240")
    h = intra_model.first_sequence_header(es)[0]
    assert intra_model.intra_index(es[h + 4:]) == []  # (the header's start code is cut off)


@pytest.mark.parametrize("name", PINNED)
def test_fresh_decoder_matches_the_reference_where_every_macroblock_is_coded(name):
    """Pinned to the reference: for every listed picture that codes every macroblock, the fresh decode's hash is the
    stored reference hash at that ordinal.  Elsewhere (slice gaps) the fresh decode differs from the sequential one
    only in macroblocks the picture does not reach, and is zero there."""
    es = stream(name)
    want = helpers.reference_decode([(0.0, es)], "whole")["fnv1a64"]
    seq_frames, _, od = helpers.decode_all(helpers.oracle_lib(), [(0.0, es)])
    od.destroy()
    full = 0
    for e in intra_model.intra_index(es):
        planes, (status, ptype, n_present, error), hdr, mbw = fresh_decode(es, e)
        assert (status, ptype, error) == (1, 1, 0), (name, e)
        k = e["picture"]
        if n_present == hdr.shape[0]:
            assert helpers.frame_hashes([planes])[0] == want[k], (name, k)
            full += 1
            continue
        absent = (hdr[:, 4] & 1) == 0
        for p, (got, seq) in enumerate(zip(planes, seq_frames[k])):
            s = 16 if p == 0 else 8
            rows, cols = got.size // (mbw * s), mbw * s
            mb = (np.arange(rows)[:, None] // s) * mbw + np.arange(cols)[None, :] // s
            mb = mb.reshape(-1)
            assert not np.any(got[absent[mb]]), (name, k, p)
            diff = got != seq
            assert np.all(absent[mb][diff]), (name, k, p)
    assert full >= 1, name


def test_some_pinned_pictures_have_gaps():
    """The gap rule above is exercised: a listed picture of random_slices_gaps or the random streams misses macroblocks."""
    gaps = 0
    for name, es in pinned_streams():
        if name.startswith(("random", "odd")):
            for e in intra_model.intra_index(es):
                _, (_, _, n_present, _), hdr, _ = fresh_decode(es, e)
                gaps += n_present < hdr.shape[0]
    assert gaps >= 1
