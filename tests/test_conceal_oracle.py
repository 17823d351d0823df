"""The `conceal` option (include/jsmpeg_b200.h, DESIGN 3.19) without a GPU.  The rule's model (tools/conceal_model.py:
the oracle's decode() with the copy) is checked on a damaged corpus against the oracle itself and against the rule
stated macroblock by macroblock; the emulated product pipeline walk -> expand -> conceal -> reconstruct
(tests/emu/conceal_check.cpp) equals the model picture for picture; the option reaches the library from BatchDecoder and
MPEG1Video; and conceal_kernel compiles to the SASS profiles/sass_hashes_sm90a.txt records.

The damaged corpus: bit flips inside pictures of I/P and B streams (test_gpu_intra._damage: no start code is made or
broken) and lost transport packets, 184-byte runs cut from inside pictures of an FFmpeg-style elementary stream."""
import ctypes
import functools
import os
import shutil
import subprocess

import numpy as np
import pytest

import conceal_model
import helpers
import macroblock_model
import synth_es
from jsmpeg_b200 import batch, decoder
from test_compact_records import RECORD, stream_geometry
from test_gpu_intra import _damage, ffmpeg_es

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_SRC = os.path.join(HERE, "emu", "conceal_check.cpp")
CSRC = os.path.join(HERE, "..", "jsmpeg_b200", "csrc")
END = b"\x00\x00\x01\xb7"


@functools.lru_cache(maxsize=None)
def corpus_stream(name):
    """A stream of the damaged corpus by name"""
    if name.startswith("ip_flips_"):
        clean = ffmpeg_es(320, 240, 24) + END
        return _damage(clean, macroblock_model.macroblock_index(clean)[::3], int(name[-1]))
    if name.startswith("b_flips_"):
        clean = synth_es.make_case("b_one_slice_fcodes")
        return _damage(clean, macroblock_model.macroblock_index(clean)[1::2], int(name[-1]), flips=3)
    if name == "b_clip_flips":
        import mini_enc
        clean = mini_enc.make_b_clip(frames=12)[0]
        return _damage(clean, macroblock_model.macroblock_index(clean)[1::2], 5, flips=2)
    if name.startswith("ip_cuts_"):
        return conceal_model.lost_packets(ffmpeg_es(640, 480, 18, seed=int(name[-1])) + END, seed=int(name[-1]))
    if name == "repeated_row":
        return conceal_model.repeated_row(synth_es.make_case("rows_ip"))
    if name == "slice_gaps":
        return synth_es.make_case("random_slices_gaps")
    raise KeyError(name)


CORPUS = ["ip_flips_1", "ip_flips_2", "b_flips_1", "b_flips_2", "b_clip_flips", "ip_cuts_1", "ip_cuts_2", "slice_gaps",
          "repeated_row"]


def oracle_views(es, decode_b):
    """Y | Cr | Cb that the oracle's own MPEG1Video shows after each decode()"""
    olib = helpers.oracle_lib()
    olib.oracle_set_decode_b(1 if decode_b else 0)
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=olib)
    out = []
    try:
        d.write(0, [es])
        n = olib.mpeg1_decoder_get_coded_size(d.decoder)
        while d.decode():
            planes = [np.ctypeslib.as_array(ctypes.cast(f(d.decoder), ctypes.POINTER(ctypes.c_uint8)), shape=(m,)).copy()
                      for f, m in ((olib.mpeg1_decoder_get_y_ptr, n), (olib.mpeg1_decoder_get_cr_ptr, n >> 2),
                                   (olib.mpeg1_decoder_get_cb_ptr, n >> 2))]
            out.append(np.concatenate(planes))
    finally:
        d.destroy()
        olib.oracle_set_decode_b(0)
    return out


@pytest.mark.parametrize("decode_b", [0, 1])
@pytest.mark.parametrize("name", CORPUS)
def test_the_model_without_the_rule_is_the_oracle(name, decode_b):
    es = corpus_stream(name)
    got = [p["planes"] for p in conceal_model.decode(helpers.oracle_lib(), es, False, decode_b=decode_b, product=False)]
    want = oracle_views(es, decode_b)
    assert len(got) == len(want) > 0
    for k, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, w), (name, k)


@pytest.mark.parametrize("decode_b", [0, 1])
@pytest.mark.parametrize("name", CORPUS)
def test_the_rule_macroblock_by_macroblock(name, decode_b):
    """Every non-PRESENT macroblock of a decoded picture is its forward reference's co-located samples; every PRESENT
    one is what oracle_reconstruct (with stage 2's rule for unfinished intra blocks) makes of it from the same
    references into the set as the picture found it."""
    es = corpus_stream(name)
    olib = helpers.oracle_lib()
    mbw, mbh = stream_geometry(es)
    absent = 0
    for k, p in enumerate(conceal_model.decode(olib, es, True, decode_b=decode_b)):
        if not p["decoded"]:
            continue
        a = ~p["present"].reshape(mbh, mbw)
        got = conceal_model.macroblock_views(p["planes"], mbw, mbh)
        for g, f in zip(got, conceal_model.macroblock_views(p["fwd"], mbw, mbh)):
            assert np.array_equal(g[a], f[a]), (name, k, "absent")
        # the PRESENT macroblocks, reconstructed without the rule from the same references
        plain = p["before"].copy()
        cw, ch = mbw * 16, mbh * 16
        ref = conceal_model.PlaneSet(cw, ch)
        ref.data[:] = p["fwd"]
        dst = conceal_model.PlaneSet(cw, ch)
        dst.data[:] = plain
        _reconstruct(olib, es, p, ref, dst)
        for g, w in zip(got, conceal_model.macroblock_views(dst.data, mbw, mbh)):
            assert np.array_equal(g[~a], w[~a]), (name, k, "present")
        absent += int(a.sum())
    if name != "slice_gaps":  # (its pictures lack macroblocks by design; the damaged ones must lose some)
        assert absent > 0, name


def _reconstruct(olib, es, p, ref, dst):
    """oracle_reconstruct(_b) of picture `p`'s records, parsed again from `es`, from `ref` (and p["bwd"]) into `dst`"""
    seq_d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=olib)
    try:
        seq_d.write(0, [es])
        seq = olib.oracle_seq_params(seq_d.decoder)
        mb_size = seq.contents.mb_size
        info = helpers.PictureInfo()
        hdr = np.zeros(mb_size * 16, dtype=np.uint8)
        coef = np.zeros(mb_size * 384, dtype=np.int16)
        olib.oracle_parse_picture.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p,
                                              ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        buf = np.frombuffer(es, dtype=np.uint8)
        olib.oracle_parse_picture(buf.ctypes.data, len(es), p["start_byte"] * 8, ctypes.cast(seq, ctypes.c_void_p),
                                  ctypes.addressof(info), hdr.ctypes.data, coef.ctypes.data)
        assert np.array_equal((hdr.reshape(mb_size, 16)[:, 4] & 1) != 0, p["present"])
        mbw = seq.contents.mb_width
        w, h = mbw * 16, (mb_size // mbw) * 16
        seq_ptr = ctypes.cast(seq, ctypes.c_void_p)
        pf, pd = ref.planes(), dst.planes()
        if p["bwd"] is None:
            olib.oracle_reconstruct(seq_ptr, w, h, hdr.ctypes.data, coef.ctypes.data, ctypes.byref(pf), ctypes.byref(pd))
        else:
            bwd = conceal_model.PlaneSet(w, h)
            bwd.data[:] = p["bwd"]
            pb = bwd.planes()
            olib.oracle_reconstruct_b(seq_ptr, w, h, hdr.ctypes.data, coef.ctypes.data, ctypes.byref(pf), ctypes.byref(pb),
                                      ctypes.byref(pd))
        conceal_model.zero_unfinished_intra_blocks(dst.data, hdr, mbw, mb_size // mbw)
    finally:
        seq_d.destroy()


def conceal_lib():
    out = os.path.join(HERE, "emu", "libconceal_check.so")
    deps = [EMU_SRC, os.path.join(HERE, "emu", "compact_emu.cpp"), os.path.join(HERE, "emu", "walk_emu.cpp")] + \
        [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        tmp = out + ".%d.tmp" % os.getpid()
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-Wno-attributes",
                               "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-o", tmp, EMU_SRC])
        os.replace(tmp, out)
    lib = ctypes.CDLL(out)
    vp, i, u32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32
    lib.emu_walk_picture.argtypes = [vp, u32, u32, i, i, vp, vp, vp, i]
    lib.emu_walk_picture_b.argtypes = [vp, u32, u32, i, i, vp, vp, vp]
    lib.emu_expand_picture_compact.argtypes = [vp, u32, i, i, vp, vp, vp, vp, vp]
    lib.emu_reconstruct_picture_compact.argtypes = [vp, vp, vp, vp, vp, vp, i, i]
    lib.emu_conceal_picture.argtypes = [vp, vp, vp, i, i]
    return lib


def quantiser_matrices(es):
    """(intra, non-intra) matrices of `es`'s sequence header, as the oracle reads them"""
    olib = helpers.oracle_lib()
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=olib)
    try:
        d.write(0, [es])
        seq = olib.oracle_seq_params(d.decoder).contents
        return bytes(seq.intra_q), bytes(seq.non_intra_q)
    finally:
        d.destroy()


def emulated_pipeline(es, name):
    """walk -> expand -> conceal -> reconstruct on the host, with decode()'s plane-set rotation and B pictures on,
    against the model with the rule picture for picture.  Returns (pictures, B pictures, concealed macroblocks)."""
    lib = conceal_lib()
    lib.emu_set_quant(*quantiser_matrices(es))
    mbw, mbh = stream_geometry(es)
    mb = mbw * mbh
    buf = np.frombuffer(es + b"\0" * 16, dtype=np.uint8).copy()
    n = mb * 384
    size = n + mbw * 16 + 64
    sets = [np.zeros(size, dtype=np.uint8) for _ in range(4)]  # two I/P sets, two B sets
    cur, b_cur, seen = 0, 0, [0, 0, 0]
    for p in conceal_model.decode(helpers.oracle_lib(), es, True, decode_b=True):
        if not p["decoded"]:
            continue
        is_b = p["type"] == 3
        hdr = np.zeros(mb * 4, dtype=np.uint32)
        park = np.zeros(mb * 6 * 2, dtype=np.uint32)
        pinfo = np.zeros(12, dtype=np.int32)
        if is_b:
            lib.emu_walk_picture_b(buf.ctypes.data, len(es), p["start_byte"], mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                                   pinfo.ctypes.data)
        else:
            lib.emu_walk_picture(buf.ctypes.data, len(es), p["start_byte"], mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                                 pinfo.ctypes.data, 1)
        assert pinfo[2] == 1, (name, seen[0])
        coef = np.zeros(mb * 6 * 64, dtype=np.int16)
        compact = np.zeros(mb * 6, dtype=RECORD)
        lib.emu_expand_picture_compact(buf.ctypes.data, len(es), mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                                       coef.ctypes.data, compact.ctypes.data, pinfo.ctypes.data)
        if is_b:
            out, fwd, bwd = sets[2 + b_cur], sets[cur], sets[cur ^ 1]
        else:
            out, fwd, bwd = sets[cur], sets[cur ^ 1], None
        seen[2] += lib.emu_conceal_picture(hdr.ctypes.data, out.ctypes.data, fwd.ctypes.data, mbw, mbh)
        lib.emu_reconstruct_picture_compact(hdr.ctypes.data, coef.ctypes.data, compact.ctypes.data, out.ctypes.data,
                                            fwd.ctypes.data, None if bwd is None else bwd.ctypes.data, mbw, mbh)
        assert np.array_equal(out[:n], p["planes"]), (name, "picture", seen[0], "type", p["type"])
        if is_b:
            b_cur ^= 1
        else:
            cur ^= 1
        seen[0] += 1
        seen[1] += int(is_b)
    return seen


@pytest.mark.parametrize("name", CORPUS)
def test_the_emulated_pipeline_equals_the_model(name):
    pictures, _, concealed = emulated_pipeline(corpus_stream(name), name)
    assert pictures > 0 and concealed > 0, (name, pictures, concealed)


def test_a_repeated_row_lacks_a_row_with_a_whole_count():
    """The repeated-row stream has pictures that the walk's error and count alone would pass as whole: no invalid
    code, n_present == mb_size, yet a row not PRESENT.  The engine queues them because a slice goes back to an
    earlier row; the device tests (tests/test_gpu_conceal.py) check that they are concealed."""
    es = corpus_stream("repeated_row")
    lib = conceal_lib()
    lib.emu_set_quant(*quantiser_matrices(es))
    mbw, mbh = stream_geometry(es)
    mb = mbw * mbh
    buf = np.frombuffer(es + b"\0" * 16, dtype=np.uint8).copy()
    hidden = 0
    for p in conceal_model.decode(helpers.oracle_lib(), es, True):
        if not p["decoded"]:
            continue
        hdr = np.zeros(mb * 4, dtype=np.uint32)
        park = np.zeros(mb * 6 * 2, dtype=np.uint32)
        pinfo = np.zeros(12, dtype=np.int32)
        lib.emu_walk_picture(buf.ctypes.data, len(es), p["start_byte"], mbw, mbh, hdr.ctypes.data, park.ctypes.data,
                             pinfo.ctypes.data, 1)
        present = (hdr.view(np.uint8).reshape(mb, 16)[:, 4] & conceal_model.MBF_PRESENT) != 0
        assert np.array_equal(present, p["present"])
        hidden += int(pinfo[8] == 0 and pinfo[6] == mb and not present.all())
    assert hidden > 0


def test_the_corpus_has_concealed_b_pictures():
    total = [0, 0, 0]
    for name in ("b_flips_1", "b_flips_2", "b_clip_flips"):
        total = [a + b for a, b in zip(total, emulated_pipeline(corpus_stream(name), name))]
    assert total[1] > 0 and total[2] > 0, total


class FakeLib:
    """A stand-in for the library that records the options it is given"""

    def __init__(self):
        self.options = []

    def jsmpeg_b200_batch_create(self, n, device, max_slots):
        return 1

    def jsmpeg_b200_batch_last_error(self, handle):
        return None

    def jsmpeg_b200_batch_destroy(self, handle):
        pass

    def jsmpeg_b200_batch_set_option(self, handle, name, value):
        self.options.append((name, value))
        return 0 if name in (b"conceal", b"decode_b") else -1

    def mpeg1_decoder_create(self, size, mode):
        return 1

    def mpeg1_decoder_destroy(self, d):
        pass

    def jsmpeg_b200_decoder_last_error(self, d):
        return None

    def jsmpeg_b200_decoder_set_option(self, d, name, value):
        return self.jsmpeg_b200_batch_set_option(d, name, value)


def test_the_option_reaches_the_library():
    lib = FakeLib()
    batch.BatchDecoder(1, lib=lib, conceal=1)
    assert lib.options == [(b"conceal", 1)]
    lib = FakeLib()
    batch.BatchDecoder(1, lib=lib, decode_b=1, conceal=0).set_option("conceal", 1)
    assert lib.options == [(b"decode_b", 1), (b"conceal", 0), (b"conceal", 1)]
    lib = FakeLib()
    batch.BatchDecoder(1, lib=lib)
    assert lib.options == []
    lib = FakeLib()
    v = decoder.MPEG1Video({"concealErrors": True, "decodeBPictures": True}, lib=lib)
    assert v.concealErrors and lib.options == [(b"decode_b", 1), (b"conceal", 1)]
    lib = FakeLib()
    assert not decoder.MPEG1Video({}, lib=lib).concealErrors and lib.options == []


def test_a_library_without_the_option_is_refused():
    """The oracle restates the reference, which has no concealment: MPEG1Video says so instead of decoding without it,
    and frees the decoder it made"""
    with pytest.raises(ValueError, match="concealErrors"):
        decoder.MPEG1Video({"concealErrors": True}, lib=helpers.oracle_lib())


def test_the_conceal_kernel_is_the_measured_one():
    """profiles/sass_hashes_sm90a.txt records conceal_kernel's SASS md5 (tools/sass_hash.py) on the build its H100
    numbers were taken with; recompiling conceal.cu must give the same machine code."""
    if not (shutil.which("nvcc") and shutil.which("cuobjdump")):
        pytest.skip("nvcc / cuobjdump not available")
    import sass_hash
    line = next(x for x in open(os.path.join(helpers.ROOT, "profiles", "sass_hashes_sm90a.txt"))
                if "conceal.cu" in x and "conceal_kernel" in x)
    recorded = next(p for p in line.split() if len(p) == 32)
    now = {sass_hash.demangle(k): md5 for k, (md5, _) in sass_hash.kernel_hashes("conceal.cu").items()}
    assert now == {"conceal_kernel": recorded}
