#!/usr/bin/env python
"""Macroblock data (BatchDecoder.decode_macroblocks) against decoding the pictures.

    python tools/time_macroblocks.py [--reps 5] [--long-frames 600] [--out FILE]

(a) every listed picture of the bench's 64 distinct 1080p x 60-picture clips in one call, against decode() with
    OUT_DEVICE of all 60 pictures of every clip and against decode_pictures of every listed picture;
(b) every listed picture of one 1080p stream of `long_frames` pictures (FFmpeg GOP 12) in one call, against decode()
    of every picture.
Every call returns after a device synchronise, so a host clock around it measures it (wall time, output tensors
included; "c_abi_preallocated": the C call alone into destinations allocated once).  Best of `reps` after a warm-up
round.  One more decode_macroblocks call per leg runs under torch.profiler, whose kernel times give the split: walk
kernels, the export kernel, copies and fills.  The card's name and power limit are read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_intra import best_of, card  # noqa: E402


def kernel_split(fn):
    """Device time (ms) of one call of `fn` by kind: walk kernels, export kernel, copies / fills, other kernels."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"walk_ms": 0.0, "export_ms": 0.0, "copy_fill_ms": 0.0, "other_ms": 0.0}
    for e in prof.key_averages():
        ms = e.device_time_total / 1000.0
        name = e.key.lower()
        if "export_macroblocks" in name:
            out["export_ms"] += ms
        elif "walk" in name:
            out["walk_ms"] += ms
        elif "memcpy" in name or "memset" in name:
            out["copy_fill_ms"] += ms
        elif ms > 0:
            out["other_ms"] += ms
    return out


def abi_call(bd, reqs):
    """The C ABI call alone, into destinations allocated once (what a caller that reuses its buffers pays)."""
    import ctypes
    n = len(reqs)
    keep = bd.decode_macroblocks(reqs)
    streams = (ctypes.c_int * n)(*[s for s, _ in reqs])
    pictures = (ctypes.c_uint32 * n)(*[p for _, p in reqs])
    dst = (ctypes.c_void_p * n)(*[t.data_ptr() for t in keep])

    def run(keep=keep):  # (the destinations live as long as the closure)
        assert bd.lib.jsmpeg_b200_batch_decode_macroblocks(bd.handle, n, streams, pictures, dst, None, None) == n
    return run


def timed(fn, reps):
    best, times = best_of(fn, reps)
    return {"best_s": best, "all_s": times}


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

    # (a) the bench's 64 clips, every listed picture
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips))
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    reqs = [(s, e["picture"]) for s in range(len(clips)) for e in bd.macroblock_index(s)]
    pics = [(s, e["picture"]) for s in range(len(clips)) for e in bd.picture_index(s)]

    def serial_all():
        bd.rewind()
        assert bd.decode(bench.PICTURES, OUT_DEVICE) == len(clips) * bench.PICTURES

    leg_a = {"streams": len(clips), "clip": f"{bench.WIDTH}x{bench.HEIGHT}x{bench.PICTURES}", "pictures": len(reqs),
             "decode_macroblocks": timed(lambda: bd.decode_macroblocks(reqs), args.reps),
             "serial_decode": dict(timed(serial_all, args.reps), pictures=len(clips) * bench.PICTURES),
             "decode_pictures": dict(timed(lambda: bd.decode_pictures(pics), args.reps), pictures=len(pics))}
    leg_a["c_abi_preallocated"] = timed(abi_call(bd, reqs), args.reps)
    leg_a["decode_macroblocks"]["split"] = kernel_split(lambda: bd.decode_macroblocks(reqs))
    leg_a["decode_macroblocks"]["pictures_per_s"] = len(reqs) / leg_a["decode_macroblocks"]["best_s"]
    leg_a["speedup_vs_serial"] = leg_a["serial_decode"]["best_s"] / leg_a["decode_macroblocks"]["best_s"]
    leg_a["speedup_vs_decode_pictures"] = leg_a["decode_pictures"]["best_s"] / leg_a["decode_macroblocks"]["best_s"]
    result["a_many_streams"] = leg_a
    bd.close()

    # (b) one long stream, every listed picture
    es = b"".join(p for _, p in gen_streams.make_clip_es(bench.WIDTH, bench.HEIGHT, args.long_frames, seed=1234, noise=bench.NOISE))
    bd = BatchDecoder(1)
    bd.write(0, es)
    every = [(0, e["picture"]) for e in bd.macroblock_index(0)]

    def serial():
        bd.rewind()
        assert bd.decode(args.long_frames, OUT_DEVICE) == args.long_frames

    leg_b = {"clip": f"{bench.WIDTH}x{bench.HEIGHT}x{args.long_frames}", "pictures": len(every),
             "decode_macroblocks": timed(lambda: bd.decode_macroblocks(every), args.reps),
             "serial_decode": dict(timed(serial, args.reps), pictures=args.long_frames)}
    leg_b["c_abi_preallocated"] = timed(abi_call(bd, every), args.reps)
    leg_b["decode_macroblocks"]["split"] = kernel_split(lambda: bd.decode_macroblocks(every))
    leg_b["speedup_vs_serial"] = leg_b["serial_decode"]["best_s"] / leg_b["decode_macroblocks"]["best_s"]
    result["b_one_stream"] = leg_b
    bd.close()

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
