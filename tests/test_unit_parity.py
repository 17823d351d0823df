"""Per-function parity of the oracle against the compiled reference (SURVEY section 4): the
reference's helper functions are non-static (prototypes src/wasm/mpeg1.c:754-769), so they can be
called directly through ctypes.  What the reference's idct() made of the blocks below is stored in
tests/golden/reference/idct.npz (recorded by tools/make_golden.py with oracle/_ref built)."""
import ctypes
import os

import numpy as np

import helpers

IDCT_GOLDEN = os.path.join(helpers.REFERENCE_DATA, "idct.npz")


def random_blocks():
    """300 blocks uniform over the full premultiplied coefficient range."""
    return np.random.default_rng(300).integers(-2048 * 62, 2047 * 62 + 1, size=(300, 64)).tolist()


def sparse_and_extreme_blocks():
    rng = np.random.default_rng(0)
    cases = [[0] * 64, [255 << 8] + [0] * 63, [-(2048 * 62)] * 64, [2047 * 62] * 64]
    for _ in range(200):
        blk = [0] * 64
        for i in rng.integers(0, 64, rng.integers(1, 6)):
            blk[int(i)] = int(rng.integers(-2048 * 62, 2047 * 62 + 1))
        cases.append(blk)
    return cases


def _idct(fn, blocks):
    out = []
    for block in blocks:
        a = (ctypes.c_int * 64)(*block)
        fn(a)
        out.append(list(a))
    return np.array(out, dtype=np.int32)


def reference_idct(name, blocks):
    if helpers.RECORD and helpers.ref_lib() is not None:
        stored = dict(np.load(IDCT_GOLDEN)) if os.path.exists(IDCT_GOLDEN) else {}
        stored[name + "_in"] = np.array(blocks, dtype=np.int32)
        stored[name + "_out"] = _idct(helpers.ref_lib().idct, blocks)
        np.savez_compressed(IDCT_GOLDEN, **stored)
    stored = np.load(IDCT_GOLDEN)
    assert np.array_equal(stored[name + "_in"], np.array(blocks, dtype=np.int32)), "blocks differ from the recorded ones"
    return stored[name + "_out"]


def test_idct_matches_reference_on_random_blocks():
    """src/mpeg1.js:916-983 / src/wasm/mpeg1.c:1673-1740 on the full premultiplied coefficient range."""
    blocks = random_blocks()
    want = reference_idct("random", blocks)
    got = _idct(helpers.oracle_lib().oracle_idct, blocks)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert not len(bad), f"blocks {bad[:8]} differ"


def test_idct_matches_reference_on_sparse_and_extreme_blocks():
    blocks = sparse_and_extreme_blocks()
    want = reference_idct("sparse_extreme", blocks)
    got = _idct(helpers.oracle_lib().oracle_idct, blocks)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert not len(bad), f"blocks {bad[:8]} differ"


def test_vlc_trie_matches_reference_read_huffman_on_random_bits():
    """Whole-stream comparisons already exercise the VLC paths; here the DCT coefficient table is
    hit with uniformly random bits through both decoders' block parsers by wrapping them in minimal
    one-macroblock intra pictures (every escape / long-code branch gets visited)."""
    import synth_es
    k = synth_es.Knobs(width=16, height=16, pictures=40, gop=1, slices="one", escape_prob=0.5, big_escape_prob=0.5,
                       max_coefs=30, dc_only_prob=0.05)
    es = synth_es.SynthStream(k, 4242).generate()
    orc_frames, orc_idx, od = helpers.decode_all(helpers.oracle_lib(), [(0.0, es)])
    helpers.assert_frames_match_reference(orc_frames, orc_idx, [(0.0, es)], "one-macroblock intra pictures")
    assert len(orc_frames) == 40
    od.destroy()
