"""The many-request program stream pass of jsmpeg_b200_batch_write_ps_many, run on the host: tests/emu/ps_many_check.cpp
drives the device's step functions (jsmpeg_b200/csrc/psdemux.cuh) through the kernels' steps, many requests of
different chunkings per call over many calls, and every stream must come out as the serial model (tools/mini_ps.py)
fed that stream's bytes alone: ES, PES table, bytes left over and in-sync state.  The chain each request marks must be
exactly the items the model visits."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import helpers
import mini_ps
import ps_cases
from ps_many_cases import chunked, two_video_program_stream

EXE_SRC = os.path.join(helpers.ROOT, "tests", "emu", "ps_many_check.cpp")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if not shutil.which("g++"):
        pytest.skip("g++ not available")
    out = tmp_path_factory.mktemp("ps_many") / "ps_many_check"
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", "-o", str(out), EXE_SRC], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def run(exe, tmp_path, n_streams, calls):
    """calls: [[(stream, stream_id, bytes), ...], ...] -> (rows per request (appended, n_pes, leftover, in_sync, [item
    positions]), per stream (es, pes, leftover, in_sync))."""
    blob = bytearray(struct.pack("<II", n_streams, len(calls)))
    for c in calls:
        blob += struct.pack("<I", len(c))
        for s, sid, data in c:
            blob += struct.pack("<iiI", s, sid, len(data)) + data
    (tmp_path / "in.bin").write_bytes(bytes(blob))
    subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], check=True)
    out = (tmp_path / "out.bin").read_bytes()
    at = 0

    def take(fmt):
        nonlocal at
        v = struct.unpack_from(fmt, out, at)
        at += struct.calcsize(fmt)
        return v

    rows = []
    for c in calls:
        for _ in c:
            appended, n_pes, left, in_sync, k = take("<IIIII")
            rows.append((appended, n_pes, left, in_sync, list(take(f"<{k}I")) if k else []))
    streams = []
    for _ in range(n_streams):
        (n,) = take("<I")
        es = out[at:at + n]
        at += n
        (n,) = take("<I")
        pes = [take("<IQ") for _ in range(n)]
        (n,) = take("<I")
        left = out[at:at + n]
        at += n
        (in_sync,) = take("<I")
        streams.append((es, pes, left, bool(in_sync)))
    return rows, streams


def schedule(feeds, rng, lo=6, hi=8):
    """feeds: per stream (stream_id, [chunks]) -> calls, each naming a random subset of lo..hi of the streams that still
    have chunks (every stream at most once per call)."""
    pending = [list(ch) for _, ch in feeds]
    calls = []
    while any(pending):
        live = [s for s in range(len(feeds)) if pending[s]]
        k = min(len(live), int(rng.integers(lo, hi + 1)))
        c = [(int(s), feeds[s][0], pending[s].pop(0)) for s in rng.permutation(live)[:k]]
        calls.append(c)
    return calls


def check(exe, tmp_path, feeds, seed):
    rng = np.random.default_rng(seed)
    calls = schedule(feeds, rng)
    rows, got = run(exe, tmp_path, len(feeds), calls)
    models = [mini_ps.Demuxer(sid) for sid, _ in feeds]
    k = 0
    for c in calls:
        for s, sid, data in c:
            m = models[s]
            items = []
            mini_ps.demux(m.leftover + data, sid, m.in_sync, items=items)
            appended, new = m.write(data)
            assert rows[k][:4] == (appended, len(new), len(m.leftover), int(m.in_sync)), (k, s)
            assert rows[k][4] == [it[0] for it in items], (k, s, "marked chain")
            k += 1
    for s, (es, pes, left, in_sync) in enumerate(got):
        m = models[s]
        assert es == bytes(m.es), f"stream {s}: {len(es)} vs {len(m.es)} ES bytes"
        assert pes == m.pes, f"stream {s}: PES table"
        assert left == m.leftover, f"stream {s}: left-over bytes"
        assert in_sync == m.in_sync, f"stream {s}: in sync"
    return calls


def test_tiny_streams_in_one_byte_writes(exe, tmp_path):
    feeds = [(0xE0, chunked(data, 1)) for data, _, _ in ps_cases.TINY.values()]
    calls = check(exe, tmp_path, feeds, seed=1)
    assert max(len(c) for c in calls) >= 6
    _, got = run(exe, tmp_path, len(feeds), calls)
    for (es, pes, _, _), (_, want_es, want_pes) in zip(got, ps_cases.TINY.values()):
        assert es == want_es and pes == want_pes


def test_writer_cases_in_any_chunking(exe, tmp_path):
    rng = np.random.default_rng(2)
    sizes = [None, 1, 7, 333, 2048, "random"]
    feeds = []
    for k, name in enumerate(ps_cases.WRITER):
        data, _ = ps_cases.writer_case(name, n=12000)
        feeds.append((0xE0, chunked(data, sizes[k % len(sizes)] or len(data), rng)))
        feeds.append((0xE0, [data]))
    check(exe, tmp_path, feeds, seed=3)


@pytest.mark.parametrize("kind", ["flips", "lengths", "garbage"])
def test_damaged_streams_with_many_breaks(exe, tmp_path, kind):
    rng = np.random.default_rng(4)
    feeds = []
    for k, name in enumerate(ps_cases.WRITER):
        data = ps_cases.damaged(ps_cases.writer_case(name, n=16000)[0], kind, seed=10 + k)
        feeds.append((0xE0, [data]))
        feeds.append((0xE0, chunked(data, ["random", 100, 1999][k % 3], rng)))
    check(exe, tmp_path, feeds, seed=5)
    # a whole damaged buffer: its chain has breaks, and what it marks is what the model visits
    data = ps_cases.damaged(ps_cases.writer_case("mpg_all", n=16000)[0], kind, seed=99)
    items = []
    mini_ps.demux(data, items=items)
    rows, _ = run(exe, tmp_path, 1, [[(0, 0xE0, data)]])
    assert rows[0][4] == [it[0] for it in items] and len(items) > 20


def test_chunks_from_one_byte_to_whole_streams(exe, tmp_path):
    data, _ = ps_cases.writer_case("vob_all", n=8000)
    bad = ps_cases.damaged(data, "garbage", seed=7)
    feeds = [(0xE0, chunked(d, size)) for d in (data, bad) for size in (1, 2, 3, 5, 16, 17, 100, 1000, len(d))]
    check(exe, tmp_path, feeds, seed=6)


def test_two_video_streams_of_one_program_stream_in_one_call(exe, tmp_path):
    es_a, es_b = ps_cases.video_es(9000, seed=1), ps_cases.video_es(7000, seed=2)
    for form in ("mpg", "vob"):
        mux = two_video_program_stream(es_a, es_b, form)
        for size in (len(mux), 1024, 333):
            pieces = chunked(mux, size)
            rows, got = run(exe, tmp_path, 2, [[(0, 0xE0, p), (1, 0xE1, p)] for p in pieces])
            for s, (sid, es) in enumerate(((0xE0, es_a), (0xE1, es_b))):
                want_es, want_pes = mini_ps.demux_chunked(mux, [], sid)
                assert got[s][0] == want_es == es, (form, size, s)
                assert got[s][1] == want_pes and len(want_pes) >= 5, (form, size, s)
                assert got[s][2] == b"" and got[s][3]


def test_the_ps_kernels_are_the_measured_ones():
    """profiles/sass_hashes_sm90a.txt records the program stream demux kernels' SASS md5 (tools/sass_hash.py);
    recompiling psdemux.cu must give the kernels that were measured."""
    if not (shutil.which("nvcc") and shutil.which("cuobjdump")):
        pytest.skip("nvcc / cuobjdump not available")
    import sys
    sys.path.insert(0, os.path.join(helpers.ROOT, "tools"))
    import sass_hash
    recorded = {}
    for line in open(os.path.join(helpers.ROOT, "profiles", "sass_hashes_sm90a.txt")):
        parts = line.lstrip("# ").split()
        if len(parts) >= 3 and parts[0] == "psdemux.cu" and parts[1].endswith("_kernel"):
            recorded[parts[1]] = parts[2]
    assert set(recorded) == {"ps_candidates_kernel", "ps_pack_kernel", "ps_link_kernel", "ps_double_kernel", "ps_head_kernel",
                             "ps_mark_kernel", "ps_classify_kernel", "ps_totals_kernel", "ps_gather_kernel"}
    now = {sass_hash.demangle(k): md5 for k, (md5, _) in sass_hash.kernel_hashes("psdemux.cu").items()}
    assert {k: now.get(k) for k in recorded} == recorded
