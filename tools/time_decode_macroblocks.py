#!/usr/bin/env python
"""Macroblock entries on the playback path: decode() with and without OUT_MACROBLOCKS, and against decode() followed
by decode_macroblocks of the same pictures (the second walk the flag saves).

    python tools/time_decode_macroblocks.py [--reps 7] [--out FILE]

decode(60) of the bench's 64 distinct 1080p x 60-picture clips (max_slots as bench.py: one round), three variants
alternated in every round of one process: "off" (OUT_DEVICE), "on" (OUT_MACROBLOCKS), "two_walks" (OUT_DEVICE, then
the C call decode_macroblocks of every listed picture into destinations allocated once).  Each variant rewinds first
and ends in a device synchronise, so a host clock around it measures it.  Best and median of `reps` after a warm-up
round.  Then, outside the timed rounds: the export kernel's device time in one "on" call under torch.profiler, and the
host's queueing time (JSMPEG_B200_HOST_TRACE) of "off" and "on".  The card's name and power limit are read in the same
process.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import re
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_intra import card  # noqa: E402


def host_trace(fn, calls):
    """Mean of the JSMPEG_B200_HOST_TRACE fields (ms) over `calls` calls of fn: the library prints them to stderr."""
    sums, n = {}, 0
    with tempfile.TemporaryFile(mode="w+b") as f:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            for _ in range(calls):
                fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        for line in f.read().decode(errors="replace").splitlines():
            if "host_ms:" in line:
                n += 1
                for key, value in re.findall(r"(\w+)=([\d.]+)", line):
                    sums[key] = sums.get(key, 0.0) + float(value)
    return {k: v / n for k, v in sums.items()} if n else {}


def export_ms(fn):
    """Device time (ms) of the export kernel in one call of fn, and its launches."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    ms, launches = 0.0, 0
    for e in prof.key_averages():
        if "export_macroblocks" in e.key:
            ms += e.device_time_total / 1000.0
            launches += e.count
    return {"export_ms": ms, "export_launches": launches}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    os.environ["JSMPEG_B200_HOST_TRACE"] = "1"  # read when a batch is made; prints only while traced below
    import bench
    from jsmpeg_b200.batch import OUT_DEVICE, OUT_MACROBLOCKS, BatchDecoder

    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips), max_slots=len(clips) * bench.PICTURES + 8)
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    reqs = [(s, e["picture"]) for s in range(len(clips)) for e in bd.macroblock_index(s)]
    n = len(reqs)
    keep = bd.decode_macroblocks(reqs)
    streams = (ctypes.c_int * n)(*[s for s, _ in reqs])
    pictures = (ctypes.c_uint32 * n)(*[p for _, p in reqs])
    dst = (ctypes.c_void_p * n)(*[t.data_ptr() for t in keep])
    want = len(clips) * bench.PICTURES

    def decode(flags):
        bd.rewind()
        assert bd.decode(bench.PICTURES, flags) == want

    def two_walks():
        decode(OUT_DEVICE)
        assert bd.lib.jsmpeg_b200_batch_decode_macroblocks(bd.handle, n, streams, pictures, dst, None, None) == n

    variants = {"off": lambda: decode(OUT_DEVICE), "on": lambda: decode(OUT_MACROBLOCKS), "two_walks": two_walks}
    quiet = open(os.devnull, "w")
    times = {k: [] for k in variants}
    saved = os.dup(2)
    os.dup2(quiet.fileno(), 2)  # (the host trace of the timed rounds)
    try:
        for rep in range(args.reps + 1):  # round 0 is the warm-up
            for name, fn in variants.items():
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                if rep:
                    times[name].append(dt)
    finally:
        os.dup2(saved, 2)
        os.close(saved)
    result = {"card": card(), "reps": args.reps, "streams": len(clips),
              "clip": f"{bench.WIDTH}x{bench.HEIGHT}x{bench.PICTURES}", "pictures": want, "listed": n}
    for name, ts in times.items():
        result[name] = {"best_s": min(ts), "median_s": statistics.median(ts), "all_s": ts}
    for name in ("on", "two_walks"):
        result[name]["over_off_best_ms"] = (result[name]["best_s"] - result["off"]["best_s"]) * 1e3
        result[name]["over_off_median_ms"] = (result[name]["median_s"] - result["off"]["median_s"]) * 1e3
    result["on"]["per_step_over_off_median_ms"] = result["on"]["over_off_median_ms"] / bench.PICTURES
    result["on"].update(export_ms(lambda: decode(OUT_MACROBLOCKS)))
    result["host_trace_off_ms"] = host_trace(lambda: decode(OUT_DEVICE), 3)
    result["host_trace_on_ms"] = host_trace(lambda: decode(OUT_MACROBLOCKS), 3)
    bd.close()

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
