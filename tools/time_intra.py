#!/usr/bin/env python
"""Key-picture decoding (BatchDecoder.decode_intra) against the serial decode() path.

    python tools/time_intra.py [--reps 5] [--long-frames 600] [--out FILE]

(a) all I pictures of the bench's 64 distinct 1080p x 60-picture clips (FFmpeg GOP 12: 5 I pictures per stream,
    320 pictures) in one decode_intra call;
(b) one 1080p stream of `long_frames` pictures: decode_intra of all its listed I pictures in one call, against
    decode() with OUT_DEVICE of every picture up to the last of them (the only way to reach them without this call).
Every call returns after a device synchronise, so a host clock around it measures it (wall time, planes included:
decode_intra allocates its output tensors).  One warm-up round first.  The card's name and power limit are read in
the same process.
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


def best_of(fn, reps):
    times = []
    for rep in range(reps + 1):  # round 0 is the warm-up
        t0 = time.perf_counter()
        fn()
        dt = time.perf_counter() - t0
        if rep:
            times.append(dt)
    return min(times), times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--long-frames", type=int, default=600)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import bench
    import gen_streams
    from jsmpeg_b200.batch import OUT_DEVICE, BatchDecoder

    result = {"card": card(), "reps": args.reps}

    # (a) 64 streams x 5 I pictures, one call
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips))
    for s, es in enumerate(clips):
        bd.write(s, es)
    reqs = [(s, e["picture"]) for s in range(len(clips)) for e in bd.intra_index(s)]

    best, times = best_of(lambda: bd.decode_intra(reqs), args.reps)  # (outputs dropped: the next round reuses them)
    result["many_streams"] = {"streams": len(clips), "clip": f"{bench.WIDTH}x{bench.HEIGHT}x{bench.PICTURES}",
                              "pictures": len(reqs), "best_s": best, "all_s": times, "pictures_per_s": len(reqs) / best}
    bd.close()

    # (b) one long stream: decode_intra of its I pictures against decode() up to the last of them
    es = b"".join(p for _, p in gen_streams.make_clip_es(bench.WIDTH, bench.HEIGHT, args.long_frames, seed=1234, noise=bench.NOISE))
    bd = BatchDecoder(1)
    bd.write(0, es)
    entries = bd.intra_index(0)
    last = entries[-1]["picture"]
    best_i, times_i = best_of(lambda: bd.decode_intra([(0, e["picture"]) for e in entries]), args.reps)

    def serial():
        bd.rewind()
        assert bd.decode(last + 1, OUT_DEVICE) == last + 1

    best_s, times_s = best_of(serial, args.reps)
    bd.close()
    per_picture_a = result["many_streams"]["pictures_per_s"]
    result["one_stream"] = {
        "clip": f"{bench.WIDTH}x{bench.HEIGHT}x{args.long_frames}", "i_pictures": len(entries), "last_i_picture": last,
        "decode_intra": {"best_s": best_i, "all_s": times_i, "pictures_per_s": len(entries) / best_i},
        "serial_decode": {"pictures": last + 1, "best_s": best_s, "all_s": times_s, "pictures_per_s": (last + 1) / best_s,
                          "i_pictures_per_s": len(entries) / best_s},
        "speedup_vs_serial": best_s / best_i,
        "rate_vs_many_streams": (len(entries) / best_i) / per_picture_a,
    }
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
