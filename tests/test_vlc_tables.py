"""Pin tools/vlc_tables.py (ISO 11172-2 Annex B form) to the reference's tree tables.

The reference's trees (src/wasm/mpeg1.c:59-680 == src/mpeg1.js:1037-1663), parsed out of the
reference source by tools/make_golden.py into tests/golden/reference/tables.json (data only), and every
canonical code is walked through them exactly the way read_huffman does (src/wasm/mpeg1.c:1742-1748).
"""
import json
import os
import re

import pytest

import helpers
import vlc_tables as V

TABLES_GOLDEN = os.path.join(helpers.REFERENCE_DATA, "tables.json")


def parse_reference_arrays(tree):
    """The named constant arrays of the reference's src/wasm/mpeg1.c (tools/make_golden.py stores them)."""
    src = open(os.path.join(tree, "src", "wasm", "mpeg1.c")).read()
    out = {}
    for m in re.finditer(r"static const (?:int|uint8_t|float) (\w+)\[\] = \{(.*?)\};", src, re.S):
        body = re.sub(r"//[^\n]*", "", m.group(2))
        vals = []
        for tok in body.replace("\n", " ").split(","):
            tok = tok.strip()
            if tok:
                vals.append(eval(tok))  # tokens are literals like "13*3", "0x0a", "-1"
        out[m.group(1)] = vals
    return out


def _ref_arrays():
    if helpers.RECORD and helpers.REFERENCE_TREE:
        with open(TABLES_GOLDEN, "w") as f:
            json.dump(parse_reference_arrays(helpers.REFERENCE_TREE), f, sort_keys=True)
            f.write("\n")
    return json.load(open(TABLES_GOLDEN))


def _walk(tree, code):
    state = 0
    for i, ch in enumerate(code):
        state = tree[state + int(ch)]
        if state < 0:
            return None, i + 1
        if tree[state] == 0:
            return tree[state + 2], i + 1
    return "incomplete", len(code)


@pytest.mark.parametrize("name", sorted(V.ALL_VLC))
def test_prefix_free(name):
    V.check_prefix_free(V.ALL_VLC[name])


@pytest.mark.parametrize("name", sorted(V.ALL_VLC))
def test_codes_match_reference_trees(name):
    tree = _ref_arrays()[name]
    table = V.ALL_VLC[name]
    for code, value in table.items():
        got, used = _walk(tree, code)
        assert used == len(code), (name, code)
        assert got == value, (name, code, got, value)
    # same number of leaves => the tables are the same function on all valid codes
    leaves = sum(1 for i in range(0, len(tree), 3) if tree[i] == 0 and i != 0)
    assert leaves == len(table), (name, leaves, len(table))


def test_constant_matrices_match_reference():
    ref = _ref_arrays()
    assert ref["ZIG_ZAG"] == V.ZIG_ZAG
    assert ref["DEFAULT_INTRA_QUANT_MATRIX"] == V.DEFAULT_INTRA_QUANT_MATRIX
    assert ref["DEFAULT_NON_INTRA_QUANT_MATRIX"] == V.DEFAULT_NON_INTRA_QUANT_MATRIX
    assert ref["PREMULTIPLIER_MATRIX"] == V.PREMULTIPLIER_MATRIX
    assert [round(x, 3) for x in ref["PICTURE_RATE"]] == [round(x, 3) for x in V.PICTURE_RATE]


def test_run_level_table_size():
    assert len(V.DCT_RUN_LEVEL_CODE) == 111  # ISO 11172-2 table B.5c-g
    assert sorted(V.ZIG_ZAG) == list(range(64))
