"""The picture's geometry and the spread of its bits over the macroblocks, WITHOUT a GPU (the GPU side:
tests/test_gpu_geometry_domain.py), on synth_es.GEOMETRY_CASES and GEOMETRY_B_CASES: one macroblock (one lane of the
lane walk) and a 1x1 display, a 16-sample column of 256 one-macroblock rows, a 4095-sample row of 256 macroblocks,
4095x4095 (256 x 256 macroblocks), 250 rows where the slice of start code 0xAF spans rows 174-249, an odd macroblock
width with cropped edges, letterboxed pictures and a fade to black.

  * the generator: every generated case stays byte for byte what it was (SHA-256 pins), and each geometry case reaches
    what its name promises, counted from the oracle's records;
  * the oracle against the compiled reference's recorded decodes (tests/golden/reference/decodes.json) on every I/P
    case whose taps stay inside the planes;
  * the device code built for the host: every walk (lane-parallel with the product's staging area, with a tiny one and
    with none, the slice walk) against the serial walk, record for record; walk, stage 1b and stage 2 against the
    oracle's planes; and the letterboxed I pictures keep the lane walk and store their records in its second pass
    (pass D of walk_slice_lanes: a lane owns more macroblocks than its share of the staging area).
"""
import functools
import hashlib

import numpy as np
import pytest

import accumulate_model
import helpers
import synth_es
from test_b_pictures import _emulated_b_pipeline
from test_motion_domain import stream  # (one generation per case and process, shared with the GPU tests)
from test_walk_emu import _pipeline_against_oracle_planes, emu_lib, picture_starts, stream_geometry, walk

IP_CASES = sorted(synth_es.GEOMETRY_CASES)
B_CASES = sorted(synth_es.GEOMETRY_B_CASES)
CASES = IP_CASES + B_CASES
LETTERBOX = sorted(n for n in IP_CASES if synth_es.GEOMETRY_CASES[n]["knobs"].get("profile") == "letterbox")
REFERENCE_CASES = synth_es.GEOMETRY_REFERENCE_CASES

# what the generated cases not committed under tests/golden/ are (SHA-256, first 16 hex digits): a change of the
# generator that moves any of them shows here
CASE_SHA256 = {
    "vec_mixed": "76bba1b9e603cc53", "vec_mixed_b": "f0db5d574b6f98a5", "vec_outside": "0a7140aea5af0742",
    "vec_outside_b": "49cab19d8eebea34", "vec_wide_1080p": "2ae15fd46fee81ce", "vec_wide_720p": "8da58e3079271df6",
    "vec_wide_b": "0ba8f1b2c4758f4e", "vec_wrap": "55d0c39376342443", "vec_wrap_b": "f1edce6251fc1bf0",
    "val_i_one_slice_300k": "6eab2dd2ac956c71", "val_i_one_slice_down": "2a7ef60b198c24e1",
    "val_i_random_slices": "57e8e1c1cf93da51", "val_i_rows_wander": "17e4515a423aecda",
    "val_lanes_640x480": "e192804bb7bafac2", "val_p_intra_resets": "542a3f18f5431562",
    "val_quant_default": "06c04796ab935349", "val_quant_matrices": "e4f6b27af900c9a5",
    "val_repro_96x16": "fbc1b4ca8c05e0be", "val_b_intra": "2ae804c549388448", "val_b_rows": "cf063920750022aa",
}
GEOMETRY_SHA256 = {
    "geo_1mb": "4de2d8407378363b", "geo_1mb_b": "7ef1a2dfa8330108", "geo_1x1": "cc1f11ae5c42cdcf",
    "geo_column": "ae7b5cb27645dbaa", "geo_column_b": "fce93451edb45479", "geo_flat_1080p": "b558190943effa05",
    "geo_letterbox_1080p": "0ad3cd8fefa42610", "geo_letterbox_720p": "076154ef92003f8b",
    "geo_letterbox_qcif": "43ce0f3244ca478d", "geo_max": "6c399fd716fa74b0", "geo_odd_4k": "c83700e62b06de2c",
    "geo_row": "ee2dbb924a829599", "geo_row_b": "9b6ad6d4f61f590f", "geo_tall_rows": "8d6377114c076c90",
}


@functools.lru_cache(maxsize=None)
def oracle_run(name, decode_b=False):
    """[(start byte, picture_info, records, coefficients, Y | Cr | Cb)] of every picture the oracle's decode() consumes,
    and the geometry in macroblocks"""
    return accumulate_model.oracle_decode(helpers.oracle_lib(), stream(name), decode_b=decode_b)


def packets(name):
    """The stream in writes of 256 KiB: the reference grows its buffer to twice its size, or to the size of one write
    less the room it had, whichever is more (buffer.c:48-64), so that one write of more than twice its initial 512 KiB
    overruns it"""
    es = stream(name)
    return [(0.0, es[i:i + (1 << 18)]) for i in range(0, len(es), 1 << 18)]


def display_size(es):
    i = es.index(b"\x00\x00\x01\xb3") + 4
    return (es[i] << 4 | es[i + 1] >> 4), ((es[i + 1] & 15) << 8 | es[i + 2])


def slice_codes(es, start):
    """The slice start codes (1..0xAF) of the picture whose header begins at byte `start`, in stream order"""
    out, i = [], es.find(b"\x00\x00\x01", start)
    while i >= 0 and 1 <= es[i + 3] <= 0xAF:
        out.append(es[i + 3])
        i = es.find(b"\x00\x00\x01", i + 4)
    return out


# ---- the generator ---------------------------------------------------------------------------------------------------

def test_the_generated_cases_stay_put():
    for name, digest in CASE_SHA256.items():
        assert hashlib.sha256(synth_es.make_case(name)).hexdigest()[:16] == digest, name
    for name, digest in GEOMETRY_SHA256.items():
        assert hashlib.sha256(stream(name)).hexdigest()[:16] == digest, name
    assert sorted(GEOMETRY_SHA256) == sorted(CASES)


def test_the_slice_rule_past_row_174():
    """slices="rows" and "random" on a picture of more than 175 rows: rows 0-173 as the mode draws them, then one slice
    of start code 0xAF (row 174) to the picture's end; 175 rows or fewer draw what they always drew"""
    for slices in ("rows", "random"):
        s = synth_es.SynthStream(synth_es.Knobs(width=16, height=16 * 200, pictures=1, gop=1, slices=slices), 5)
        s.sequence_header()
        s.picture(0)
        es = s.out.tobytes()
        codes = slice_codes(es, es.index(b"\x00\x00\x01\x00") + 4)
        assert codes[-1] == 0xAF and max(codes) == 0xAF, (slices, codes[-4:])
        if slices == "rows":
            assert codes == list(range(1, 0xB0))


@pytest.mark.parametrize("name", CASES)
def test_each_case_reaches_its_geometry(name):
    """Every macroblock of every decoded picture present (decode_b on for the B twins), and what the name promises: the
    macroblock counts, mb_width 256, slice code 0xAF spanning rows past 174, cropped edges, black bars"""
    es = stream(name)
    got, mbw, mbh = oracle_run(name, name in B_CASES)
    width, height = display_size(es)
    decoded = [(start, info, rec) for start, info, rec, _, _ in got if info.status == 1]
    assert len(decoded) == {**synth_es.GEOMETRY_CASES, **synth_es.GEOMETRY_B_CASES}[name]["knobs"]["pictures"]
    for start, info, rec in decoded:
        assert info.n_present == mbw * mbh, (name, start)
    geometry = {"geo_1mb": (1, 1), "geo_1x1": (1, 1), "geo_column": (1, 256), "geo_row": (256, 1), "geo_max": (256, 256),
                "geo_tall_rows": (21, 250)}
    base = name[:-2] if name in B_CASES else name
    if base in geometry:
        assert (mbw, mbh) == geometry[base], name
    if name == "geo_1x1":
        assert (width, height) == (1, 1)
    if name == "geo_odd_4k":
        assert mbw % 2 == 1 and width % 16 and height % 16 and mbw * mbh > 32_000
    if mbh > 175 and base != "geo_max":  # the rows past 174 come from the slice of code 0xAF, which spans them
        for start, info, rec in decoded:
            codes = slice_codes(es, info.start_byte)
            assert codes[-1] == 0xAF and len(codes) == 175 and codes == sorted(codes), (name, start)
            flags = np.frombuffer(rec.tobytes(), accumulate_model.macroblock_model.RECORD)["flags"]
            assert (flags.reshape(mbh, mbw)[175:] & 1).all()
    if base == "geo_max":
        assert all(len(slice_codes(es, info.start_byte)) == 1 for _, info, _ in decoded)
    profile = synth_es.GEOMETRY_CASES.get(name, {"knobs": {}})["knobs"].get("profile")
    if profile:
        s = synth_es.SynthStream(synth_es.Knobs(**synth_es.GEOMETRY_CASES[name]["knobs"]), 0)
        bar = np.array([s.in_bar(mb) for mb in range(mbw * mbh)])
        assert bar.any() and (profile == "flat") == bar.all()
        for start, info, rec in decoded:
            r = np.frombuffer(rec.tobytes(), accumulate_model.macroblock_model.RECORD)
            if info.picture_type == 1:  # the bars: intra macroblocks of six DC-only blocks
                assert (r["cbp"][bar] == 0x3F).all() and (r["dc_only"][bar] == 0x3F).all(), name
            else:  # skipped, or a zero vector and no coded block
                assert (r["cbp"][bar] == 0).all() and (r["mv_h"][bar] == 0).all() and (r["mv_v"][bar] == 0).all(), name


# ---- the oracle against the compiled reference ------------------------------------------------------------------------

@pytest.mark.parametrize("name", REFERENCE_CASES)
def test_oracle_equals_the_compiled_reference(name):
    """The compiled reference (its decodes stored in tests/golden/reference/decodes.json) on every I/P case whose taps
    all lie inside its planes"""
    frames, idx, d = helpers.decode_all(helpers.oracle_lib(), packets(name))
    helpers.assert_frames_match_reference(frames, idx, packets(name), f"{name}: oracle vs compiled reference")
    d.destroy()


# ---- the device code, emulated ---------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def walks(name):
    """Every walk of every picture against the serial one (modes of tests/emu/walk_emu.cpp: 1 the lane walk with the
    product's staging area, 2 with a tiny one, 3 with none, 4 the slice walk): picture info, records and the parked
    data of every coded block equal.  Returns per decoded picture (picture type, the lane walk's picture info)."""
    es = stream(name)
    lib = emu_lib()
    mbw, mbh = stream_geometry(es)
    buf = np.frombuffer(es + b"\0" * 16, dtype=np.uint8).copy()
    out = []
    for k, s in enumerate(picture_starts(es)):
        h0, c0, i0 = walk(lib, buf, len(es), s, mbw, mbh, 0)
        hb = h0.view(np.uint8).reshape(-1, 16)
        coded = np.zeros(len(c0), dtype=bool)
        for blk in range(6):
            coded[blk::6] = ((hb[:, 4] & 1) != 0) & ((hb[:, 5] & (0x20 >> blk)) != 0)
        for mode in (1, 2, 3, 4):
            h1, c1, i1 = walk(lib, buf, len(es), s, mbw, mbh, mode)
            assert np.array_equal(i0[:9], i1[:9]), f"{name}: picture {k} mode {mode}: info {i0[:9]} vs {i1[:9]}"
            assert np.array_equal(h0, h1), \
                f"{name}: picture {k} mode {mode}: records differ at mb {np.nonzero((h0 != h1).any(axis=1))[0][:8]}"
            assert np.array_equal(c0[coded], c1[coded]), f"{name}: picture {k} mode {mode}: parked block data differ"
            if mode == 1 and i1[2] == 1:
                out.append((int(i1[3]), i1.copy()))
    return out


@pytest.mark.parametrize("name", CASES)
def test_every_walk_gives_the_serial_walks_records(name):
    assert walks(name)


@pytest.mark.parametrize("name", LETTERBOX)
def test_letterboxed_pictures_take_the_lane_walks_storing_pass(name):
    """The I pictures of a letterboxed stream keep the lane walk (info.reserved[0] == 1) but no slice of theirs is
    finished from the staged records (reserved[2] == 0): the lanes over the bars own more macroblocks than their share
    of the staging area, so the walk stores its records in pass D -- with the serial walk's records (walks())"""
    pics = [info for ptype, info in walks(name) if ptype == 1]
    assert len(pics) == 2
    for info in pics:
        assert (info[9], info[11]) == (1, 0), (name, info)


@pytest.mark.parametrize("name", IP_CASES)
def test_emulated_device_code_equals_the_oracle(name):
    """walk (lane-parallel) -> stage 1b -> stage 2, on the host, against the oracle's planes"""
    assert _pipeline_against_oracle_planes(stream(name), name, walk_mode=1) == synth_es.GEOMETRY_CASES[name]["knobs"]["pictures"]


@pytest.mark.parametrize("name", B_CASES)
def test_emulated_device_code_equals_the_oracle_b(name):
    lib = helpers.oracle_lib()
    lib.oracle_set_decode_b(1)
    try:
        checked, n_b = _emulated_b_pipeline(stream(name), name)
    finally:
        lib.oracle_set_decode_b(0)
    assert checked == synth_es.GEOMETRY_B_CASES[name]["knobs"]["pictures"] and n_b > 0
