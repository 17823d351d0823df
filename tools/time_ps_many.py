#!/usr/bin/env python
"""Cost of feeding MPEG program streams to many streams: one jsmpeg_b200_batch_write_ps call per stream against one
jsmpeg_b200_batch_write_ps_many call for all of them.

    python tools/time_ps_many.py [--streams 64] [--width 1920 --height 1080 --frames 60] [--reps 3] [--out FILE]

`streams` streams on cuda:0, stream k fed gen_streams.make_clip_ps (.mpg) with seed k.  Legs: (a) whole clips; (b) 64
KB and (c) 16 KB per stream per round; (d) 64 KB per stream per round of a damaged copy, random bytes followed by a
false pack-header prefix inserted at 32 places of every clip (each a break in the item chain: one more
head/mark/end round and synchronisation per break in the per-break-round demuxer this pass replaced).  In each round
every stream gets its next piece, through `streams` write_ps calls in one batch and through one write_ps_many call in
another; both calls return after a device synchronise, so a host clock around a round measures it.  Reported per leg and path: ms per round (best of `reps` passes over the clip,
after a warm-up pass), input GB/s, the launches per call (stats.kernel_launches) and the nominal host synchronisations per call.
Every leg checks every stream's ES (read_es) and PES table against the per-stream path.  Then one profiled round of
the 64 KB leg per path (torch.profiler, CUDA activity) attributes the device time to copies and kernels.  Reads the
card's name and power limit in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from multiprocessing import Pool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

# host synchronisations per call of the PS path (csrc/engine.cu demux_many) by design, not counted: the candidate
# counts, the per-request results, then the copy back.  A stream whose HBM mirror or the per-candidate scratch grows
# adds one; the timed passes start from a reset batch whose mirrors and scratch mostly have room already.
SYNCS_PER_CALL_NOMINAL = 3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out


def _clip(args):
    import gen_streams
    w, h, n, seed = args
    return gen_streams.make_clip_ps(w, h, n, seed=seed, form="mpg")


def damaged(clip, seed, breaks=32):
    """`clip` with `breaks` runs of 1-299 random bytes and a false pack-header prefix inserted at random places."""
    import numpy as np
    rng = np.random.default_rng(seed)
    b = bytearray(clip)
    for at in sorted(rng.integers(0, len(b), breaks), reverse=True):
        b[at:at] = rng.integers(0, 256, int(rng.integers(1, 300)), dtype=np.uint8).tobytes() + b"\x00\x00\x01\xba"
    return bytes(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=64)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from jsmpeg_b200.batch import BatchDecoder

    S = args.streams
    with Pool(min(S, os.cpu_count() or 1)) as pool:
        clips = pool.map(_clip, [(args.width, args.height, args.frames, k) for k in range(S)])
    one, many = BatchDecoder(S), BatchDecoder(S)

    def pieces(chunk):
        return [[c[o:o + chunk] for o in range(0, len(c), chunk)] for c in clips]

    bad = [damaged(c, 1000 + k) for k, c in enumerate(clips)]
    legs = {"whole": [[c] for c in clips], "64k": pieces(65536), "16k": pieces(16384),
            "64k_damaged": [[c[o:o + 65536] for o in range(0, len(c), 65536)] for c in bad]}
    result = {"card": card(), "streams": S, "clip": f"{args.width}x{args.height}x{args.frames} .mpg",
              "ps_bytes_per_stream": sum(len(c) for c in clips) / S, "reps": args.reps, "legs": {}}

    def rounds(leg):
        chunks = legs[leg]
        return [[(s, chunks[s][j]) for s in range(S) if j < len(chunks[s])] for j in range(max(len(c) for c in chunks))]

    def run_one(rnd):
        return [one.write_ps(s, data) for s, data in rnd]

    def run_many(rnd):
        return many.write_ps_many(rnd)

    for leg in legs:
        rs = rounds(leg)
        total_in = sum(len(d) for r in rs for _, d in r)
        best = {"write_ps": float("inf"), "write_ps_many": float("inf")}
        stats = {}
        for rep in range(args.reps + 1):  # pass 0 is the warm-up
            for name, bd, fn in (("write_ps", one, run_one), ("write_ps_many", many, run_many)):
                bd.reset()
                bd.reset_stats()
                got = []
                t = 0.0
                for rnd in rs:
                    t0 = time.perf_counter()
                    got.append(fn(rnd))
                    t += time.perf_counter() - t0
                if rep:
                    best[name] = min(best[name], t)
                stats[name] = (bd.stats()["kernel_launches"], got)
        # the same bytes and PES tables, stream by stream
        assert stats["write_ps"][1] == stats["write_ps_many"][1], leg
        for s in range(S):
            assert one.read_es(s) == many.read_es(s), (leg, s)
        calls = {"write_ps": sum(len(r) for r in rs), "write_ps_many": len(rs)}
        result["legs"][leg] = {
            "rounds": len(rs), "input_bytes": total_in,
            **{name: {"ms_per_round": 1e3 * best[name] / len(rs), "total_ms": 1e3 * best[name],
                      "input_GBps": total_in / best[name] / 1e9,
                      "launches_per_call": stats[name][0] / calls[name], "syncs_per_call_nominal": SYNCS_PER_CALL_NOMINAL}
               for name in best},
            "speedup": best["write_ps"] / best["write_ps_many"],
        }
        print(leg, json.dumps(result["legs"][leg]), flush=True)

    # where the device time of one 64 KB round goes, per path
    import torch
    from torch.profiler import ProfilerActivity, profile
    rnd = rounds("64k")[1]
    result["profiled_round_64k"] = {}
    for name, bd, fn in (("write_ps", one, run_one), ("write_ps_many", many, run_many)):
        bd.reset()
        fn(rounds("64k")[0])
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn(rnd)
        device = {}
        for ev in prof.key_averages():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                key = ev.key.replace("(anonymous namespace)::", "")
                if key.startswith("void cub::"):  # e.g. "cub DeviceRadixSortOnesweepKernel"
                    key = "cub " + key.split("<")[0].split("::")[-1]
                elif not key.startswith(("Memcpy", "Memset")):
                    key = key.split("(")[0]
                d = device.setdefault(key, {"calls": 0, "total_ms": 0.0})
                d["calls"] += ev.count
                d["total_ms"] += ev.device_time_total / 1e3
        result["profiled_round_64k"][name] = dict(sorted(device.items(), key=lambda kv: -kv[1]["total_ms"]))
    one.close()
    many.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
