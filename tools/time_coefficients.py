#!/usr/bin/env python
"""Coefficients (BatchDecoder.decode_coefficients) against macroblock data and against decoding the pictures.

    python tools/time_coefficients.py [--reps 5] [--per-clip 16] [--long-frames 600] [--out FILE]

(a) `per_clip` listed pictures (spread evenly) of each of the bench's 64 distinct 1080p x 60-picture clips in one call,
    against decode_macroblocks of the same requests and decode() with OUT_DEVICE of all 60 pictures of every clip;
(b) every listed picture of one 1080p stream of `long_frames` pictures (FFmpeg GOP 12) in one call, against decode()
    of every picture.
A 1080p picture's coefficients are 6.27 MB: `per_clip` keeps leg (a)'s destinations (and the slot pool beside them)
inside the card; it is printed.  Every call returns after a device synchronise, so a host clock around it measures it
(wall time, output tensors included; "c_abi_preallocated": the C call alone into destinations allocated once).  Best
of `reps` after a warm-up round.  One more call per leg runs under torch.profiler, whose kernel times give the split:
walk kernels, expand, the export kernel, copies and fills.  The export kernel's bytes -- 768 written and a 16-byte
record read per macroblock, 32 per coded block (its compact record) and 128 more per dense block -- over its kernel
time give its share of the H100 SXM data sheet's 3.35 TB/s.  Coded blocks are counted from the entries' cbp bits,
dense blocks as coded blocks with more than 12 nonzero values (a written value is never 0 except an intra DC of 0).
The card's name and power limit are read in the same process.
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

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def kernel_split(fn):
    """Device time (ms) of one call of `fn` by kind: walk kernels, expand, the two export kernels, copies / fills."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"walk_ms": 0.0, "expand_ms": 0.0, "export_coefficients_ms": 0.0, "export_macroblocks_ms": 0.0,
           "copy_fill_ms": 0.0, "other_ms": 0.0}
    for e in prof.key_averages():
        ms = e.device_time_total / 1000.0
        name = e.key.lower()
        if "export_coefficients" in name:
            out["export_coefficients_ms"] += ms
        elif "export_macroblocks" in name:
            out["export_macroblocks_ms"] += ms
        elif "expand" in name:
            out["expand_ms"] += ms
        elif "walk" in name:
            out["walk_ms"] += ms
        elif "memcpy" in name or "memset" in name:
            out["copy_fill_ms"] += ms
        elif ms > 0:
            out["other_ms"] += ms
    return out


def export_bytes(bd, reqs):
    """Bytes the export kernel moves for `reqs` (module docstring) and the block counts behind them."""
    import torch
    mbs = coded = dense = 0
    for c, m in bd.decode_coefficients(reqs, macroblocks=True):
        cbp = m[..., 9].to(torch.int32)
        bits = torch.stack([(cbp >> (5 - b)) & 1 for b in range(6)], dim=-1).bool()  # [h, w, 6]
        nonzero = (c != 0).flatten(-2).sum(-1)  # [h, w, 6]
        mbs += cbp.numel()
        coded += int(bits.sum())
        dense += int((bits & (nonzero > 12)).sum())
    return {"macroblocks": mbs, "coded_blocks": coded, "dense_blocks": dense,
            "bytes": mbs * (768 + 16) + coded * 32 + dense * 128}


def abi_call(bd, reqs):
    """The C ABI call alone, into destinations allocated once (what a caller that reuses its buffers pays)."""
    import ctypes
    n = len(reqs)
    keep = bd.decode_coefficients(reqs)
    streams = (ctypes.c_int * n)(*[s for s, _ in reqs])
    pictures = (ctypes.c_uint32 * n)(*[p for _, p in reqs])
    dst = (ctypes.c_void_p * n)(*[t.data_ptr() for t in keep])

    def run(keep=keep):  # (the destinations live as long as the closure)
        assert bd.lib.jsmpeg_b200_batch_decode_coefficients(bd.handle, n, streams, pictures, dst, None, None, None) == n
    return run


def timed(fn, reps):
    best, times = best_of(fn, reps)
    return {"best_s": best, "all_s": times}


def leg(bd, reqs, reps):
    """decode_coefficients of `reqs`: Python and C call times, the kernel split, the export kernel's bandwidth."""
    out = {"pictures": len(reqs), "decode_coefficients": timed(lambda: bd.decode_coefficients(reqs), reps)}
    out["c_abi_preallocated"] = timed(abi_call(bd, reqs), reps)
    split = kernel_split(lambda: bd.decode_coefficients(reqs))
    out["decode_coefficients"]["split"] = split
    out["decode_coefficients"]["pictures_per_s"] = len(reqs) / out["decode_coefficients"]["best_s"]
    moved = export_bytes(bd, reqs)
    moved["bytes_per_s"] = moved["bytes"] / (split["export_coefficients_ms"] / 1000.0)
    moved["share_of_3_35_tb_s"] = moved["bytes_per_s"] / PEAK_BYTES_PER_S
    out["export_kernel"] = moved
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--per-clip", type=int, default=16)
    ap.add_argument("--long-frames", type=int, default=600)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import bench
    import gen_streams
    from jsmpeg_b200.batch import OUT_DEVICE, BatchDecoder

    result = {"card": card(), "reps": args.reps}

    # (a) the bench's 64 clips, per_clip listed pictures of each
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips))
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    reqs = []
    for s in range(len(clips)):
        listed = [e["picture"] for e in bd.macroblock_index(s)]
        reqs += [(s, listed[i * len(listed) // args.per_clip]) for i in range(args.per_clip)]
    print(f"(a) {args.per_clip} pictures per clip, {len(reqs)} in one call", file=sys.stderr)

    def serial_all():
        bd.rewind()
        assert bd.decode(bench.PICTURES, OUT_DEVICE) == len(clips) * bench.PICTURES

    leg_a = {"streams": len(clips), "clip": f"{bench.WIDTH}x{bench.HEIGHT}x{bench.PICTURES}", "per_clip": args.per_clip,
             **leg(bd, reqs, args.reps),
             "decode_macroblocks": timed(lambda: bd.decode_macroblocks(reqs), args.reps),
             "serial_decode": dict(timed(serial_all, args.reps), pictures=len(clips) * bench.PICTURES)}
    leg_a["ratio_to_decode_macroblocks"] = leg_a["decode_coefficients"]["best_s"] / leg_a["decode_macroblocks"]["best_s"]
    leg_a["ratio_to_serial_decode"] = leg_a["decode_coefficients"]["best_s"] / leg_a["serial_decode"]["best_s"]
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

    leg_b = {"clip": f"{bench.WIDTH}x{bench.HEIGHT}x{args.long_frames}", **leg(bd, every, args.reps),
             "serial_decode": dict(timed(serial, args.reps), pictures=args.long_frames)}
    leg_b["ratio_to_serial_decode"] = leg_b["decode_coefficients"]["best_s"] / leg_b["serial_decode"]["best_s"]
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
