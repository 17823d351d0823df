#!/usr/bin/env python
"""Input rate of the device program stream demux (jsmpeg_b200_batch_write_ps) next to the TS demux and a plain
write of the same content.

    python tools/time_ps.py [--streams 64] [--width 1920 --height 1080 --frames 60] [--reps 3] [--out FILE]

One batch of `streams` streams on cuda:0, each fed the same FFmpeg encode: as an .mpg program stream with
write_ps in one call and in 64 KB chunks, as MPEG-TS with write_ts in one call and in 64 KB chunks, and as the raw ES with a
plain write + upload (what makes it resident in HBM, as the demuxers leave it).  Every call returns after a
device synchronise, so a host clock around the calls measures them.  A warm-up round runs first; the batch
is reset between rounds.  Then one profiled round of write_ps (torch.profiler, CUDA activity) attributes
the device time to the demux's kernels.  Reads the card's name and power limit in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=64)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=65536)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import gen_streams
    from jsmpeg_b200.batch import BatchDecoder

    w, h, n = args.width, args.height, args.frames
    ps = gen_streams.make_clip_ps(w, h, n, form="mpg")
    ts = gen_streams.make_clip_ts(w, h, n)
    es = gen_streams.make_clip_m1v(w, h, n)
    ps_chunks = [ps[o:o + args.chunk] for o in range(0, len(ps), args.chunk)]
    ts_chunks = [ts[o:o + args.chunk] for o in range(0, len(ts), args.chunk)]
    bd = BatchDecoder(args.streams)

    def run_ps(s):
        assert bd.write_ps(s, ps)[0] == len(es)

    def run_ps_chunked(s):
        assert sum(bd.write_ps(s, c)[0] for c in ps_chunks) == len(es)

    def run_ts(s):
        assert bd.write_ts(s, ts)[0] == len(es)

    def run_ts_chunked(s):
        assert sum(bd.write_ts(s, c)[0] for c in ts_chunks) == len(es)

    def run_write(s):
        bd.write(s, es)

    methods = {"write_ps": (run_ps, len(ps)), "write_ps_64k": (run_ps_chunked, len(ps)), "write_ts": (run_ts, len(ts)),
               "write_ts_64k": (run_ts_chunked, len(ts)), "write_upload": (run_write, len(es))}
    times = {k: [] for k in methods}
    for rep in range(args.reps + 1):  # round 0 is the warm-up
        for name, (fn, _) in methods.items():
            bd.reset()
            t0 = time.perf_counter()
            for s in range(args.streams):
                fn(s)
            if name == "write_upload":
                bd.upload()
            dt = time.perf_counter() - t0
            if rep:
                times[name].append(dt)
    result = {"card": card(), "streams": args.streams, "clip": f"{w}x{h}x{n}", "ps_bytes": len(ps), "ts_bytes": len(ts),
              "es_bytes": len(es), "reps": args.reps, "chunk": args.chunk, "methods": {}}
    for name, (_, in_bytes) in methods.items():
        best = min(times[name])
        result["methods"][name] = {"input_bytes_per_stream": in_bytes, "best_s": best, "all_s": times[name],
                                   "ms_per_stream": 1e3 * best / args.streams,
                                   "input_GBps": in_bytes * args.streams / best / 1e9}

    # where write_ps's device time goes: kernel time by name over one round
    import torch
    from torch.profiler import ProfilerActivity, profile
    bd.reset()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(args.streams):
            run_ps(s)
    kernels = {}
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            kernels[ev.key] = {"calls": ev.count, "total_ms": ev.device_time_total / 1e3}
    result["write_ps_device_ms"] = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["total_ms"]))
    bd.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
