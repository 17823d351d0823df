"""Host-side logic that stays outside the kernels: the MPEG-TS demuxer mirror, the decoder surface
(PTS table, seek, decodeFirstFrame, callbacks), the C-ABI library's exports.  No GPU needed: the
decoder surface is exercised over the oracle library, which exports the same 15-function ABI."""
import ctypes
import os
import re

import numpy as np
import pytest

import helpers
from jsmpeg_b200 import batch, capi, decoder, ts
from jsmpeg_b200.shard import assign_streams


def mux_ts(packets, pid=0x100, stream_id=0xE0, pad_last=True):
    """A minimal MPEG-TS muxer: one PES per payload (length 0, PTS only), 188-byte packets, the last
    packet of a PES padded with an adaptation field -- the shape FFmpeg produces (SURVEY app. B)."""
    out = bytearray()
    cc = 0
    for pts, payload in packets:
        p = int(round(pts * 90000))
        pts_bytes = bytes([0x21 | ((p >> 29) & 0x0E), (p >> 22) & 0xFF, 0x01 | ((p >> 14) & 0xFE), (p >> 7) & 0xFF, 0x01 | ((p << 1) & 0xFE)])
        pes = b"\x00\x00\x01" + bytes([stream_id]) + b"\x00\x00" + b"\x80\x80\x05" + pts_bytes + payload
        first = True
        pos = 0
        while pos < len(pes):
            room = 184
            chunk = pes[pos:pos + room]
            header = bytearray([0x47, (0x40 if first else 0x00) | (pid >> 8), pid & 0xFF, 0x10 | cc])
            if len(chunk) < room:  # pad with an adaptation field
                pad = room - len(chunk)
                header[3] = 0x30 | cc
                af = bytearray([pad - 1]) + (bytearray([0x00]) + bytearray([0xFF] * (pad - 2)) if pad > 1 else bytearray())
                out += header + af + chunk
            else:
                out += header + chunk
            pos += len(chunk)
            cc = (cc + 1) & 15
            first = False
    return bytes(out)


def test_ts_demux_round_trip():
    rng = np.random.default_rng(0)
    packets = [(1.0 + i / 30.0, bytes(rng.integers(0, 256, int(rng.integers(50, 3000)), dtype=np.uint8))) for i in range(20)]
    stream = mux_ts(packets)
    assert len(stream) % 188 == 0
    got = ts.demux_video_es(stream)
    assert len(got) == len(packets)
    for (pts_a, a), (pts_b, b) in zip(got, packets):
        assert a == b
        assert abs(pts_a - pts_b) < 1e-4


def test_ts_demux_chunked_writes_and_resync():
    rng = np.random.default_rng(1)
    packets = [(i / 25.0, bytes(rng.integers(0, 256, 1000, dtype=np.uint8))) for i in range(12)]
    stream = b"\x12\x34\x56" + mux_ts(packets)  # leading garbage: the demuxer must resync (ts.js:155-189)
    demux = ts.TS()
    col = ts.ESCollector()
    demux.connect(ts.TS.STREAM_VIDEO_1, col)
    for o in range(0, len(stream), 1000):
        demux.write(stream[o:o + 1000])
    demux.flush()
    assert b"".join(p for _, p in col.packets) == b"".join(p for _, p in packets)


def test_ts_demux_of_ffmpeg_clip_feeds_decoder():
    import gen_streams
    data = gen_streams.make_clip_ts(176, 144, 10, seed=3, noise=4)
    packets = ts.demux_video_es(data)
    assert len(packets) == 10  # one PES per picture
    frames, idx, d = helpers.decode_all(helpers.oracle_lib(), packets)
    assert len(frames) == 10 and (d.width, d.height) == (176, 144)
    assert d.startTime == packets[0][0]
    d.destroy()


def test_decoder_surface_seek_and_timestamps():
    packets = helpers.clip_packets(176, 144, 12, seed=5, noise=4)
    frames, idx, d = helpers.decode_all(helpers.oracle_lib(), packets)
    assert abs(d.currentTime - (packets[-1][0] + 1 / 30.0)) < 0.05
    # seek to the 5th packet: decoding resumes there (src/decoder.js:49-71); picture 4 is a P picture
    # of the same GOP so the planes differ from a clean decode, but the bookkeeping must hold
    d.seek(packets[4][0] + 1e-6)
    assert d.decodedTime == packets[4][0]
    assert d.bufferGetIndex() == sum(len(p) for _, p in packets[:4]) << 3
    assert d.decode()
    d.destroy()


def test_decode_first_frame_and_callbacks():
    packets = helpers.clip_packets(176, 144, 6, seed=5, noise=4)
    calls = []
    d = decoder.MPEG1Video({"onVideoDecode": lambda dec, ms: calls.append(ms)}, lib=helpers.oracle_lib())
    rec = decoder.PlaneRecorder()
    d.connect(rec)
    d.write(packets[0][0], [packets[0][1]])  # contains the sequence header: decodes one picture at once
    assert rec.size == (176, 144) and rec.count == 1 and len(calls) == 1
    assert not d.decode()  # nothing else buffered
    d.destroy()


def test_product_library_exports_every_declared_symbol():
    """libjsmpeg_b200.so loads without a GPU and exports everything include/jsmpeg_b200.h declares."""
    if not os.path.exists(capi.PRODUCT_LIB):
        pytest.skip("libjsmpeg_b200.so not built (run __graft_entry__.build())")
    header = open(os.path.join(helpers.ROOT, "include", "jsmpeg_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b((?:mpeg1_decoder|jsmpeg_b200)_\w+)\s*\(", header))
    assert set(capi.MPEG1_ABI) <= declared and len(declared) >= 30
    lib = ctypes.CDLL(capi.PRODUCT_LIB)
    missing = [name for name in sorted(declared) if not hasattr(lib, name)]
    assert not missing, missing
    # the Python binding tables name real symbols too
    for name in list(capi.MPEG1_ABI) + list(batch._BATCH_ABI):
        assert hasattr(lib, name), name


def test_product_has_no_cpu_fallback():
    """The product package never references the oracle; the C-ABI binding fails loudly when the
    library is missing."""
    pkg = os.path.join(helpers.ROOT, "jsmpeg_b200")
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                text = open(os.path.join(root, f), errors="ignore").read()
                # ("_ref" as a name of its own: oracle/_ref, libjsmpeg_ref -- not the "_ref" inside temporal_reference)
                assert "liboracle" not in text and "oracle/" not in text and not re.search(r"_ref(?![a-z])", text), f
    with pytest.raises(FileNotFoundError):
        capi.load_library(os.path.join(pkg, "does_not_exist.so"))


def test_stream_sharding_is_a_partition():
    for world in (1, 2, 4, 8):
        owned = [assign_streams(512, r, world) for r in range(world)]
        assert sorted(sum(owned, [])) == list(range(512))
        assert max(len(o) for o in owned) - min(len(o) for o in owned) <= 1


def test_without_a_cuda_device_the_c_abi_answers_false_and_the_python_host_raises():
    """Boundary behaviour of the reference ("create never fails, decode returns false", src/wasm/mpeg1.c:777-782,
    853-864) when there is no usable GPU: no abort(), a dead decoder that swallows writes and answers false, the
    reason available through jsmpeg_b200_decoder_last_error; the Python host classes raise instead.  (Round 1
    called abort() on any CUDA error.)  Skipped where a GPU is present: the same calls then simply work."""
    if not os.path.exists(capi.PRODUCT_LIB):
        pytest.skip("libjsmpeg_b200.so not built")
    lib = capi.product_library()
    d = lib.mpeg1_decoder_create(1000, capi.BIT_BUFFER_MODE_EXPAND)
    err = lib.jsmpeg_b200_decoder_last_error(d)
    if not err:
        lib.mpeg1_decoder_destroy(d)
        pytest.skip("a CUDA device is present")
    assert b"CUDA error" in err
    p = lib.mpeg1_decoder_get_write_ptr(d, 5000)  # more than the buffer: the caller's memcpy must still be safe
    assert p
    ctypes.memset(p, 0xB3, 5000)
    lib.mpeg1_decoder_did_write(d, 5000)
    assert lib.mpeg1_decoder_decode(d) is False
    assert lib.mpeg1_decoder_has_sequence_header(d) == 0
    assert lib.mpeg1_decoder_get_y_ptr(d) is None
    assert lib.mpeg1_decoder_get_index(d) == 0
    lib.mpeg1_decoder_destroy(d)
    with pytest.raises(RuntimeError):
        batch.BatchDecoder(2)
    with pytest.raises(RuntimeError):
        decoder.MPEG1Video({})


def test_napi_addon_source_parses():
    """addon/jsmpeg_b200_napi.c has never met a Node toolchain (none in this image): at least prove that it
    is C that parses and type-checks against the N-API calls it uses (tests/stubs/node_api.h declares
    exactly those, with the signatures of Node's js_native_api.h)."""
    import subprocess
    src = os.path.join(helpers.ROOT, "addon", "jsmpeg_b200_napi.c")
    r = subprocess.run(["gcc", "-fsyntax-only", "-Wall", "-Werror=implicit-function-declaration", "-Werror=incompatible-pointer-types",
                        "-I", os.path.join(helpers.ROOT, "tests", "stubs"), "-I", os.path.join(helpers.ROOT, "include"), src],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]


def test_kernels_are_the_measured_ones():
    """profiles/sass_hashes_sm90a.txt lists an md5 of every kernel's SASS on the build the H100 numbers were taken with
    (tools/sass_hash.py).  Recompiling the tree must give the same machine code: nobody edits a kernel after it was
    measured without this test saying so."""
    import shutil
    import sys
    if not (shutil.which("nvcc") and shutil.which("cuobjdump")):
        pytest.skip("nvcc / cuobjdump not available")
    sys.path.insert(0, os.path.join(helpers.ROOT, "tools"))
    import sass_hash
    recorded = {}
    for line in open(os.path.join(helpers.ROOT, "profiles", "sass_hashes_sm90a.txt")):
        parts = line.split()
        if len(parts) >= 3 and parts[0].endswith(".cu") and parts[1].endswith("_kernel"):
            recorded[parts[1]] = next(p for p in parts[2:] if len(p) == 32)
    assert {"walk_pictures_lanes_kernel", "expand_blocks_kernel", "reconstruct_kernel", "reconstruct_b_kernel",
            "walk_pictures_b_kernel", "walk_pictures_slices_kernel", "scan_start_codes_kernel"} <= set(recorded)
    now = {}
    for cu in ("parse.cu", "recon.cu", "scan.cu"):
        for name, (md5, _) in sass_hash.kernel_hashes(cu).items():
            now[sass_hash.demangle(name)] = md5
    changed = {k: (recorded[k], now.get(k)) for k in recorded if k in now and now[k] != recorded[k]}
    assert not changed, changed
    assert all(k in now for k in recorded if not k.startswith("ts_"))
