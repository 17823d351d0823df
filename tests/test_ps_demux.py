"""MPEG program stream demux, CPU side: the serial model (tools/mini_ps.py) against FFmpeg's muxers, the
writer and hand-written streams; the device's per-item header (psdemux.cuh) built with g++ against the model;
write_ps through the C ABI on a batch without a device."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import helpers
import mini_ps
import ps_cases


@pytest.mark.parametrize("size", [(320, 240, 24), (1280, 720, 30)])
@pytest.mark.parametrize("form", ["mpg", "vob"])
def test_model_es_of_ffmpeg_program_streams_equals_m1v_and_ts(size, form):
    import gen_streams
    from jsmpeg_b200.ts import demux_video_es
    w, h, n = size
    m1v = gen_streams.make_clip_m1v(w, h, n)
    ts_es = b"".join(p for _, p in demux_video_es(gen_streams.make_clip_ts(w, h, n)))
    data = gen_streams.make_clip_ps(w, h, n, form=form)
    es, pes, consumed, in_sync = mini_ps.demux(data)
    assert es == m1v == ts_es
    assert consumed == len(data) and in_sync
    assert 0 < len(pes) <= n
    assert all(a[0] < b[0] and a[1] < b[1] for a, b in zip(pes, pes[1:]))


@pytest.mark.parametrize("name", sorted(ps_cases.WRITER))
def test_model_round_trips_the_writer(name):
    data, table = ps_cases.writer_case(name)
    es, pes, consumed, in_sync = mini_ps.demux(data)
    assert es == ps_cases.video_es()
    assert pes == table
    assert consumed == len(data) and in_sync


@pytest.mark.parametrize("name", sorted(ps_cases.TINY))
def test_model_on_hand_written_streams(name):
    data, want_es, want_pes = ps_cases.TINY[name]
    es, pes, _, _ = mini_ps.demux(data)
    assert es == want_es
    assert pes == want_pes


def test_model_keeps_an_incomplete_packet_for_the_next_call():
    data, _, _ = ps_cases.TINY["incomplete_trailing_packet"]
    _, _, consumed, in_sync = mini_ps.demux(data)
    assert data[consumed:] == bytes.fromhex("000001E000100F44") and in_sync
    d = mini_ps.Demuxer()
    d.write(data)
    n, pes = d.write(b"\x55" * 14 + bytes.fromhex("000001B9"))  # the packet's 14 missing body bytes, then an end code
    assert n == 15 and bytes(d.es) == bytes.fromhex("3344") + b"\x55" * 14 and d.in_sync and d.leftover == b""


def _corpus():
    out = [(f"tiny_{k}", v[0]) for k, v in sorted(ps_cases.TINY.items())]
    for name in sorted(ps_cases.WRITER):
        data, _ = ps_cases.writer_case(name)
        out.append((name, data))
        for kind in ("flips", "lengths", "garbage"):
            out.append((f"{name}_{kind}", ps_cases.damaged(data, kind, 11)))
    return out


def test_model_is_independent_of_the_chunking():
    for name, data in _corpus():
        whole = mini_ps.demux_chunked(data, [])
        for seed in range(3):
            assert mini_ps.demux_chunked(data, ps_cases.random_cuts(len(data), seed, mean=300)) == whole, (name, seed)
        if len(data) < 200:
            assert mini_ps.demux_chunked(data, range(1, len(data))) == whole, name  # 1-byte writes
            for c in range(1, len(data)):
                assert mini_ps.demux_chunked(data, [c]) == whole, (name, c)


def _model_row(data, p):
    kind, ln = mini_ps.item_at(data, p)
    start, plen, pts = 0, 0, None
    if kind == mini_ps.ITEM and data[p + 3] > 0xBB:
        start, plen, pts = mini_ps.payload(data[p:p + ln])
    return (kind, ln, start, plen, int(pts is not None), pts or 0, int(mini_ps.is_pack(data, p)))


def test_item_header_compiled_for_the_host_equals_the_model(tmp_path):
    """psdemux.cuh is the device's per-item arithmetic; built with g++ it must give the model's answer at every
    start-code prefix of the corpus (true items, false ones in payloads, damaged ones) and at the buffer end."""
    if not shutil.which("g++"):
        pytest.skip("g++ not available")
    exe = tmp_path / "ps_item_check"
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", "-o", str(exe),
                        os.path.join(helpers.ROOT, "tests", "emu", "ps_item_check.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    checked = 0
    for name, data in _corpus():
        path = tmp_path / "buf.bin"
        path.write_bytes(data)
        positions = [i for i in range(len(data) - 2) if data[i:i + 3] == b"\x00\x00\x01"]
        positions += list(range(max(0, len(data) - 16), len(data)))  # prefixes cut by the buffer end
        out = subprocess.run([str(exe), str(path)], input="\n".join(map(str, positions)), capture_output=True,
                             text=True, check=True).stdout.split("\n")
        for p, line in zip(positions, out):
            assert tuple(int(x) for x in line.split()) == _model_row(data, p), (name, p)
        checked += len(positions)
    assert checked > 1000


def test_write_ps_on_a_batch_without_a_device_returns_minus_one():
    """Like every entry point of a dead batch: -1, no PES entries, and no abort().  Skipped where a device is
    present (the GPU tests cover the live batch)."""
    from jsmpeg_b200 import batch, capi
    if not os.path.exists(capi.PRODUCT_LIB):
        pytest.skip("libjsmpeg_b200.so not built")
    lib = batch.bind_batch_abi(capi.product_library())
    b = lib.jsmpeg_b200_batch_create(1, 0, 2)
    try:
        if not lib.jsmpeg_b200_batch_last_error(b):
            pytest.skip("a CUDA device is present")
        data, _, _ = ps_cases.TINY["false_pack_in_audio"]
        pts = np.zeros(8, np.uint64)
        off = np.zeros(8, np.uint32)
        n = ctypes.c_int(7)
        assert lib.jsmpeg_b200_batch_write_ps(b, 0, data, len(data), 0xE0, pts.ctypes.data, off.ctypes.data, 8,
                                              ctypes.byref(n)) == -1
        assert n.value == 0
        assert lib.jsmpeg_b200_debug_read_es(b, 0, None, 0) == -1
    finally:
        lib.jsmpeg_b200_batch_destroy(b)
