"""Shared test helpers: library loading, clip access, oracle record access, stored reference decodes."""
import ctypes
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from jsmpeg_b200 import capi, decoder  # noqa: E402

ORACLE_LIB = os.path.join(ROOT, "oracle", "liboracle.so")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libjsmpeg_ref.so")
GOLDEN = os.path.join(ROOT, "tests", "golden")
REFERENCE_DATA = os.path.join(GOLDEN, "reference")
# JSMPEG_RECORD_REFERENCE=1 with oracle/_ref built: run the compiled reference and (re)write what the tests
# compare against under tests/golden/ (tools/make_golden.py); otherwise those files are only read.
RECORD = os.environ.get("JSMPEG_RECORD_REFERENCE") == "1"
# the reference's source tree (a checkout of phoboslab/jsmpeg), needed only to record its constant tables
REFERENCE_TREE = os.environ.get("JSMPEG_REFERENCE_TREE", "")


class PictureInfo(ctypes.Structure):
    _fields_ = [("start_byte", ctypes.c_uint32), ("end_bit", ctypes.c_uint32), ("status", ctypes.c_int32),
                ("picture_type", ctypes.c_int32), ("full_pel", ctypes.c_int32), ("f_code", ctypes.c_int32),
                ("n_present", ctypes.c_int32), ("n_coded_blocks", ctypes.c_int32), ("error", ctypes.c_int32),
                ("reserved", ctypes.c_int32 * 3)]


class SeqParamsOracle(ctypes.Structure):
    _fields_ = [("mb_width", ctypes.c_int), ("mb_size", ctypes.c_int),
                ("intra_q", ctypes.c_uint8 * 64), ("non_intra_q", ctypes.c_uint8 * 64)]


def build_oracle():
    if not os.path.exists(ORACLE_LIB) or os.path.getmtime(ORACLE_LIB) < os.path.getmtime(
            os.path.join(ROOT, "oracle", "mpeg1_oracle.c")):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])


_oracle = None


def oracle_lib():
    global _oracle
    if _oracle is None:
        build_oracle()
        lib = capi.load_library(ORACLE_LIB)
        lib.oracle_last_picture_info.restype = ctypes.POINTER(PictureInfo)
        lib.oracle_last_picture_info.argtypes = [ctypes.c_void_p]
        lib.oracle_last_mb_records.restype = ctypes.c_void_p
        lib.oracle_last_mb_records.argtypes = [ctypes.c_void_p]
        lib.oracle_last_coefficients.restype = ctypes.c_void_p
        lib.oracle_last_coefficients.argtypes = [ctypes.c_void_p]
        lib.oracle_seq_params.restype = ctypes.POINTER(SeqParamsOracle)
        lib.oracle_seq_params.argtypes = [ctypes.c_void_p]
        # the product's extension entry points, same names (B pictures: decodeBPictures / lastPicture of the host class)
        lib.jsmpeg_b200_decoder_set_option.restype = ctypes.c_int
        lib.jsmpeg_b200_decoder_set_option.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int]
        lib.jsmpeg_b200_decoder_last_picture.restype = ctypes.c_int
        lib.jsmpeg_b200_decoder_last_picture.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
        _oracle = lib
    return _oracle


def ref_lib():
    if not os.path.exists(REF_LIB):
        return None
    return capi.load_library(REF_LIB)


def decode_all(lib, packets, options=None, keep=True, max_frames=None):
    """Drive a 15-function-ABI library through the decoder surface: write everything, then decode()
    until it returns False.  Returns (frames, bit indices after each decode, decoder)."""
    opts = {"decodeFirstFrame": False}
    opts.update(options or {})
    d = decoder.MPEG1Video(opts, lib=lib)
    rec = decoder.PlaneRecorder(keep=keep)
    d.connect(rec)
    for pts, payload in packets:
        d.write(pts, [payload])
    idx = []
    while (max_frames is None or len(idx) < max_frames) and d.decode():
        idx.append(d.bufferGetIndex())
    return rec.frames, idx, d


def assert_frames_equal(a, b, what=""):
    assert len(a) == len(b), f"{what}: {len(a)} vs {len(b)} pictures"
    for k, (x, y) in enumerate(zip(a, b)):
        for name, p, q in zip(("Y", "Cr", "Cb"), x, y):
            if not np.array_equal(p, q):
                w = np.nonzero(p != q)[0]
                raise AssertionError(f"{what}: picture {k} plane {name}: {len(w)} bytes differ, first at {w[:8]}: "
                                     f"{p[w[:8]]} vs {q[w[:8]]}")


def clip_packets(width, height, frames, seed=1234, noise=9):
    import gen_streams
    return gen_streams.make_clip_es(width, height, frames, seed, noise)


def frame_hashes(frames):
    """FNV-1a 64 (hex) of Y | Cr | Cb of each picture, the hash bench.py's checker uses."""
    import bench
    return [format(bench.fnv1a64_planes(*(np.ascontiguousarray(p) for p in f)), "016x") for f in frames]


def streaming_decode(lib, packets, buffer_size=64 * 1024):
    """EVICT mode with a small buffer, write-a-packet / decode-what-is-there, like the reference player's
    streaming loop (src/player.js:222-229).  Returns (frames, bit index after every decode)."""
    d = decoder.MPEG1Video({"streaming": True, "videoBufferSize": buffer_size, "decodeFirstFrame": False}, lib=lib)
    rec = decoder.PlaneRecorder()
    d.connect(rec)
    trace = []
    for pts, payload in packets:
        d.write(pts, [payload])
        while d.decode():
            trace.append(d.bufferGetIndex())
    d.destroy()
    return rec.frames, trace


_STORE = os.path.join(REFERENCE_DATA, "decodes.json")
_store = None


def reference_decode(packets, mode="whole"):
    """What the compiled reference gave for these packets, stored in tests/golden/reference/decodes.json
    under the SHA-1 of the elementary stream: {"bit_index_after": [...], "fnv1a64": [...]} (one entry per
    decode() == true).  mode "whole": decode_all; "evict_streaming": streaming_decode; "picture_hashes": the
    harness's ref_picture_hashes (one decoder sized for the whole stream; hashes only, as bench.py's checker)."""
    global _store
    if _store is None:
        _store = json.load(open(_STORE)) if os.path.exists(_STORE) else {}
    key = f"{mode}:{hashlib.sha1(b''.join(p for _, p in packets)).hexdigest()}"
    if RECORD and ref_lib() is not None:
        if mode == "picture_hashes":
            import bench
            es = b"".join(p for _, p in packets)
            buf = (ctypes.c_uint64 * 4096)()
            n = bench.ref_library().ref_picture_hashes(es, len(es), buf, 4096)
            _store[key] = {"bit_index_after": None, "fnv1a64": [format(buf[k], "016x") for k in range(min(n, 4096))]}
        else:
            if mode == "whole":
                frames, idx, d = decode_all(ref_lib(), packets)
                d.destroy()
            else:
                frames, idx = streaming_decode(ref_lib(), packets)
            _store[key] = {"bit_index_after": idx, "fnv1a64": frame_hashes(frames)}
        with open(_STORE, "w") as f:
            json.dump(_store, f, indent=0, sort_keys=True)
            f.write("\n")
    assert key in _store, f"no stored reference decode {key}: the stream differs from the one recorded (tools/make_golden.py)"
    return _store[key]


def assert_frames_match_reference(frames, idx, packets, what, mode="whole", first=0):
    """Pictures (from `first` on) and bit indices equal to the stored reference decode of the same packets."""
    want = reference_decode(packets, mode)
    assert idx == want["bit_index_after"], f"{what}: bit indices differ from the reference"
    got = frame_hashes(frames)
    assert len(got) == len(want["fnv1a64"]), f"{what}: {len(got)} vs {len(want['fnv1a64'])} pictures"
    bad = [k for k in range(first, len(got)) if got[k] != want["fnv1a64"][k]]
    assert not bad, f"{what}: pictures {bad[:8]} differ from the reference"
