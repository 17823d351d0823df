#!/usr/bin/env python
"""Generate tests/golden/: small elementary streams plus the outputs of the REFERENCE itself on them.

Run where the reference's source tree is present (needs oracle/_ref/libjsmpeg_ref.so, built by oracle/Makefile):

    python tools/make_golden.py

For every case it writes
    tests/golden/<name>.es     the elementary stream (synthetic syntax-corner streams of
                               tools/synth_es.py, and two small cv2/FFmpeg-encoded clips)
    tests/golden/<name>.json   per decode() call: the bit index afterwards and the sha256 of the
                               Y / Cr / Cb planes the reference exposes through get_{y,cr,cb}_ptr,
                               plus width/height/coded size/frame rate
all produced by the unmodified reference C (src/wasm/mpeg1.c + buffer.c compiled by
oracle/Makefile) driven through its 15-function ABI.  The reference ships no golden vectors of
its own (SURVEY.md section 4); these are the vectors that pin the oracle and the CUDA path.

    JSMPEG_REFERENCE_TREE=<reference checkout> python tools/make_golden.py --reference-data

records instead what the tests that compare with the compiled reference read, so that they run where the
reference is absent: tests/golden/reference/decodes.json (picture hashes and bit indices per stream),
idct.npz, tables.json (the reference's constant arrays) and bitbuffer.npy beside it.
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import gen_streams  # noqa: E402
import helpers  # noqa: E402
import synth_es  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")

FFMPEG_CASES = {
    "ffmpeg_320x240_ip": dict(width=320, height=240, frames=14, seed=1234, noise=9),
    "ffmpeg_176x144_ip": dict(width=176, height=144, frames=26, seed=7, noise=4),
}


def sha(a):
    return hashlib.sha256(a.tobytes()).hexdigest()


def describe(lib, es):
    frames, idx, d = helpers.decode_all(lib, [(0.0, es)])
    out = {"width": d.width, "height": d.height, "coded_size": d.codedSize, "frame_rate": round(float(d.frameRate), 3),
           "es_sha256": hashlib.sha256(es).hexdigest(),
           "pictures": [{"index": i, "y": sha(y), "cr": sha(cr), "cb": sha(cb)} for i, (y, cr, cb) in zip(idx, frames)]}
    d.destroy()
    return out


# the CPU tests that compare with the reference record their own streams when run with JSMPEG_RECORD_REFERENCE=1
RECORDING_TESTS = ["test_oracle_vs_reference.py", "test_unit_parity.py", "test_vlc_tables.py", "test_rgba_cases.py",
                   "test_bench_contract.py", "test_b_pictures.py::test_extension_off_b_pictures_are_consumed_and_not_decoded"]


def gpu_test_streams():
    """The streams only GPU tests compare with the reference (test_gpu_parity, test_gpu_bench_config)."""
    import bench
    from test_gpu_parity import SIZES
    for w, h, n in SIZES + [(1920, 1080, 5)]:
        yield helpers.clip_packets(w, h, n), "whole"
    old, bench.PICTURES = bench.PICTURES, 25
    try:
        clips = bench.load_streams([1234 + i for i in range(64)], 1920, 1080)
    finally:
        bench.PICTURES = old
    for es in clips:
        yield [(0, es)], "picture_hashes"


def record_reference_data():
    if helpers.ref_lib() is None or not helpers.REFERENCE_TREE:
        raise SystemExit("needs oracle/_ref/libjsmpeg_ref.so (`make -C oracle REF=<reference checkout>`) and JSMPEG_REFERENCE_TREE")
    env = dict(os.environ, JSMPEG_RECORD_REFERENCE="1")
    tests = os.path.join(ROOT, "tests")
    subprocess.check_call([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider",
                           *(os.path.join(tests, t) for t in RECORDING_TESTS)], env=env, cwd=ROOT)
    with tempfile.TemporaryDirectory() as tmp:
        lib = os.path.join(tmp, "libbitbuffer_test.so")
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", lib, os.path.join(tests, "emu", "bitbuffer_test.cpp")])
        subprocess.check_call([sys.executable, os.path.join(tests, "emu", "bitbuffer_check.py"), lib,
                               os.path.join(GOLDEN, "reference", "bitbuffer.npy"), "--record", helpers.REF_LIB])
    helpers.RECORD = True
    for packets, mode in gpu_test_streams():
        helpers.reference_decode(packets, mode)


def main():
    if "--reference-data" in sys.argv:
        return record_reference_data()
    ref = helpers.ref_lib()
    if ref is None:
        raise SystemExit("oracle/_ref/libjsmpeg_ref.so missing: run `make -C oracle` where the reference tree is present")
    os.makedirs(GOLDEN, exist_ok=True)
    cases = {name: synth_es.make_case(name) for name in synth_es.CASES}
    for name, kw in FFMPEG_CASES.items():
        packets = gen_streams.make_clip_es(kw["width"], kw["height"], kw["frames"], kw["seed"], kw["noise"])
        cases[name] = b"".join(p for _, p in packets)
    for name, es in cases.items():
        with open(os.path.join(GOLDEN, name + ".es"), "wb") as f:
            f.write(es)
        info = describe(ref, es)
        info["generator"] = "tools/synth_es.py" if name in synth_es.CASES else "tools/gen_streams.py (cv2/FFmpeg mpeg1video)"
        info["produced_by"] = "reference src/wasm/mpeg1.c + buffer.c (unmodified), oracle/_ref build"
        with open(os.path.join(GOLDEN, name + ".json"), "w") as f:
            json.dump(info, f, indent=1)
        print(f"{name}: {len(es)} bytes, {len(info['pictures'])} pictures")


if __name__ == "__main__":
    main()
