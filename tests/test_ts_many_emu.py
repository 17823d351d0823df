"""The segmented MPEG-TS pass of jsmpeg_b200_batch_write_ts_many, run on the host: tests/emu/ts_many_check.cpp
drives the device's per-packet arithmetic (jsmpeg_b200/csrc/tsdemux.cuh) through the kernels' steps, many requests
of different chunkings per call over many calls, and every stream must come out as src/ts.js's host mirror
(jsmpeg_b200/ts.py) fed that stream's bytes alone: ES, PES table, bytes left over and PID bindings carried on."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import helpers
import ts_many_cases as cases

EXE_SRC = os.path.join(helpers.ROOT, "tests", "emu", "ts_many_check.cpp")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if not shutil.which("g++"):
        pytest.skip("g++ not available")
    out = tmp_path_factory.mktemp("ts_many") / "ts_many_check"
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", "-o", str(out), EXE_SRC], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def run(exe, tmp_path, n_streams, calls):
    """calls: [[(stream, stream_id, bytes), ...], ...] -> (rows per request, per stream (es, pes, leftover, bound))."""
    blob = bytearray(struct.pack("<II", n_streams, len(calls)))
    for c in calls:
        blob += struct.pack("<I", len(c))
        for s, sid, data in c:
            blob += struct.pack("<iiI", s, sid, len(data)) + data
    (tmp_path / "in.bin").write_bytes(bytes(blob))
    subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], check=True)
    out = (tmp_path / "out.bin").read_bytes()
    n_rows = sum(len(c) for c in calls)
    rows = [struct.unpack_from("<III", out, 12 * i) for i in range(n_rows)]
    at = 12 * n_rows
    streams = []

    def take(fmt):
        nonlocal at
        v = struct.unpack_from(fmt, out, at)
        at += struct.calcsize(fmt)
        return v

    for _ in range(n_streams):
        (n,) = take("<I")
        es = out[at:at + n]
        at += n
        (n,) = take("<I")
        pes = [take("<IQ") for _ in range(n)]
        (n,) = take("<I")
        left = out[at:at + n]
        at += n
        (n,) = take("<I")
        bound = dict(take("<Ii") for _ in range(n))
        streams.append((es, pes, left, bound))
    return rows, streams


def schedule(feeds, rng):
    """feeds: per stream (stream_id, [chunks]) -> calls, each naming a random subset of the streams that still have
    chunks (every stream at most once per call)."""
    pending = [list(ch) for _, ch in feeds]
    calls = []
    while any(pending):
        c = []
        for s in rng.permutation(len(feeds)):
            if pending[s] and rng.random() < 0.7:
                c.append((int(s), feeds[s][0], pending[s].pop(0)))
        if c:
            calls.append(c)
    return calls


def check(exe, tmp_path, feeds, seed):
    rng = np.random.default_rng(seed)
    calls = schedule(feeds, rng)
    rows, got = run(exe, tmp_path, len(feeds), calls)
    models = [cases.StreamModel(sid) for sid, _ in feeds]
    k = 0
    for c in calls:
        for s, _, data in c:
            appended, new = models[s].write(data)
            assert rows[k] == (appended, len(new), len(models[s].leftover)), (k, s)
            k += 1
    for s, (es, pes, left, bound) in enumerate(got):
        m = models[s]
        assert es == m.es(), f"stream {s}: {len(es)} vs {len(m.es())} ES bytes"
        assert pes == m.table, f"stream {s}: PES table"
        assert left == m.leftover, f"stream {s}: left-over bytes"
        assert bound == m.bound, f"stream {s}: PID bindings"
    return calls


def test_many_requests_of_any_chunking_equal_the_host_mirror_per_stream(exe, tmp_path):
    """Eight streams in calls that name random subsets: garbage between packets (resync), misaligned requests beside
    aligned ones, a PID re-bound mid-stream and back, chunks under 188 bytes, whole clips."""
    import gen_streams
    rng = np.random.default_rng(5)
    clips = [gen_streams.make_clip_ts(176, 144, 8, seed=20 + k, noise=4) for k in range(4)]
    feeds = [
        (0xE0, cases.chunked(clips[0], 188 * 7)),
        (0xE0, cases.chunked(cases.with_garbage(clips[1], 1), 1000)),
        (0xE0, cases.chunked(cases.rebound(clips[2], 2, 3), 333)),
        (0xE0, cases.chunked(cases.with_garbage(cases.rebound(clips[3], 1, 1), 2), "random", rng)),
        (0xE0, [clips[0]]),
        (0xE0, cases.chunked(clips[1], 100)),
        (0xE0, cases.chunked(clips[2][:188 * 9 + 77], 1)[:40] + [clips[2][40:188 * 9 + 77]]),
        (0xE1, cases.chunked(cases.rebound(clips[3], 0, 100), 188 * 3)),
    ]
    calls = check(exe, tmp_path, feeds, seed=1)
    assert max(len(c) for c in calls) >= 5


def test_one_multiplex_of_two_programs_in_two_requests(exe, tmp_path):
    """The same buffer in two requests of a call, stream id 0xE0 to one stream and 0xE1 to another; chunked and whole."""
    import gen_streams
    mux = cases.two_programs(gen_streams.make_clip_ts(176, 144, 6, seed=7, noise=4),
                             gen_streams.make_clip_ts(176, 144, 6, seed=8, noise=4))
    for chunk in (len(mux), 188 * 5, 777):
        pieces = cases.chunked(mux, chunk)
        calls = [[(0, 0xE0, p), (1, 0xE1, p)] for p in pieces]
        rows, got = run(exe, tmp_path, 2, calls)
        for s, sid in ((0, 0xE0), (1, 0xE1)):
            m = cases.StreamModel(sid)
            for p in pieces:
                m.write(p)
            es, pes, left, bound = got[s]
            assert es == m.es() and len(es) > 1000, (chunk, s)
            assert pes == m.table and len(pes) >= 6, (chunk, s)
            assert left == m.leftover and bound == m.bound == {0x100: 0xE0, 0x101: 0xE1}, (chunk, s)


def test_the_ts_kernels_are_the_measured_ones():
    """profiles/sass_hashes_sm90a.txt records the TS demux kernels' SASS md5 (tools/sass_hash.py); recompiling
    tsdemux.cu must give the kernels that were measured."""
    if not (shutil.which("nvcc") and shutil.which("cuobjdump")):
        pytest.skip("nvcc / cuobjdump not available")
    import sys
    sys.path.insert(0, os.path.join(helpers.ROOT, "tools"))
    import sass_hash
    recorded = {}
    for line in open(os.path.join(helpers.ROOT, "profiles", "sass_hashes_sm90a.txt")):
        parts = line.split()
        if len(parts) >= 3 and parts[0] == "tsdemux.cu" and parts[1].endswith("_kernel"):
            recorded[parts[1]] = parts[2]
    assert set(recorded) == {"ts_check_grid_kernel", "ts_walk_grid_kernel", "ts_classify_kernel", "ts_bind_kernel",
                             "ts_carry_kernel", "ts_totals_kernel", "ts_gather_kernel"}
    now = {sass_hash.demangle(k): md5 for k, (md5, _) in sass_hash.kernel_hashes("tsdemux.cu").items()}
    assert {k: now.get(k) for k in recorded} == recorded
