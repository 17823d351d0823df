#!/usr/bin/env python
"""Residuals (BatchDecoder.decode_residuals) against coefficients and against decoding the pictures.

    python tools/time_residuals.py [--reps 5] [--per-clip 16] [--long-frames 600] [--out FILE]

(a) `per_clip` listed pictures (spread evenly) of each of the bench's 64 distinct 1080p x 60-picture clips in one call;
(b) every listed picture of one 1080p stream of `long_frames` pictures (FFmpeg GOP 12) in one call.
Each leg against decode_coefficients and decode_pictures of the same requests.  Every call returns after a device
synchronise, so a host clock around it measures it (wall time, output tensors included; "c_abi_preallocated": the C
call alone into destinations allocated once).  Best of `reps` after a warm-up round.  One more call per leg runs under
torch.profiler, whose kernel times give the split: walk kernels, expand, the export kernel, copies and fills.

The export kernel's bytes: 768 written and the 4-byte flags word read per macroblock, 32 per coded block (its compact
record) and 128 more per dense block; over its kernel time, its share of the H100 SXM data sheet's 3.35 TB/s.  Its
instructions: a warp with a block that needs the transform runs the whole block path, at most the kernel's static
SASS length (straight-line code but for the request search and the record scatter, every branch of which is in that
count); the other warps a fraction of it.  `full_warps` x that length over the kernel time, against the issue rate of
132 SMs x 4 warp instructions per clock at the card's maximum SM clock, bounds its share of the instruction rate from
above.  Coded blocks are counted from the entries' cbp bits, dense blocks as coded blocks with more than 12 nonzero
values, blocks that need the transform as coded blocks with a nonzero value past the DC (a written value is never 0
except an intra DC of 0).  The card's name, power limit and maximum SM clock are read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_coefficients import timed  # noqa: E402
from time_intra import card  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
SMS, ISSUE_PER_SM = 132, 4   # H100 SXM: SMs, warp instructions issued per SM per clock


def kernel_split(fn):
    """Device time (ms) of one call of `fn` by kind: walk kernels, expand, the export kernels, copies / fills."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"walk_ms": 0.0, "expand_ms": 0.0, "export_residuals_ms": 0.0, "export_other_ms": 0.0, "copy_fill_ms": 0.0,
           "other_ms": 0.0}
    for e in prof.key_averages():
        ms = e.device_time_total / 1000.0
        name = e.key.lower()
        if "export_residuals" in name:
            out["export_residuals_ms"] += ms
        elif "export" in name:
            out["export_other_ms"] += ms
        elif "expand" in name:
            out["expand_ms"] += ms
        elif "walk" in name or "reconstruct" in name:
            out["walk_ms" if "walk" in name else "other_ms"] += ms
        elif "memcpy" in name or "memset" in name:
            out["copy_fill_ms"] += ms
        elif ms > 0:
            out["other_ms"] += ms
    return out


def export_work(bd, reqs):
    """Bytes the export kernel moves for `reqs`, the block counts behind them, and its warps (module docstring)."""
    import torch
    mbs = coded = dense = full_blocks = warps = full_warps = 0
    for c, m in bd.decode_coefficients(reqs, macroblocks=True):
        cbp = m[..., 9].to(torch.int32)
        bits = torch.stack([(cbp >> (5 - b)) & 1 for b in range(6)], dim=-1).bool()  # [h, w, 6]
        flat = c.flatten(-2)
        nonzero = (flat != 0).sum(-1)  # [h, w, 6]
        full = bits & (flat[..., 1:] != 0).any(-1)
        mbs += cbp.numel()
        coded += int(bits.sum())
        dense += int((bits & (nonzero > 12)).sum())
        full_blocks += int(full.sum())
        # the kernel's slots: per macroblock row [luma top 2W | luma bottom 2W | Cb W | Cr W], 32 per warp
        h, w = cbp.shape
        slots = torch.cat([full[:, :, 0:2].reshape(h, 2 * w), full[:, :, 2:4].reshape(h, 2 * w), full[:, :, 4], full[:, :, 5]], 1)
        slots = slots.reshape(-1)
        pad = (-slots.numel()) % 32
        slots = torch.cat([slots, slots.new_zeros(pad)]).reshape(-1, 32)
        warps += slots.shape[0]
        full_warps += int(slots.any(1).sum())
    return {"macroblocks": mbs, "coded_blocks": coded, "dense_blocks": dense, "transform_blocks": full_blocks,
            "warps": warps, "full_warps": full_warps, "bytes": mbs * (768 + 4) + coded * 32 + dense * 128}


def abi_call(bd, reqs):
    """The C ABI call alone, into destinations allocated once (what a caller that reuses its buffers pays)."""
    import ctypes
    n = len(reqs)
    keep = bd.decode_residuals(reqs)
    streams = (ctypes.c_int * n)(*[s for s, _ in reqs])
    pictures = (ctypes.c_uint32 * n)(*[p for _, p in reqs])
    dst = (ctypes.c_void_p * n)(*[t.data_ptr() for t in keep])

    def run(keep=keep):  # (the destinations live as long as the closure)
        assert bd.lib.jsmpeg_b200_batch_decode_residuals(bd.handle, n, streams, pictures, dst, None, None, None) == n
    return run


def static_instructions():
    import sass_hash
    return next(n for k, (_, n) in sass_hash.kernel_hashes("residuals.cu").items())


def leg(bd, reqs, reps, max_sm_hz, sass_len):
    """decode_residuals of `reqs` against decode_coefficients and decode_pictures: call times, the kernel split, the
    export kernel's bandwidth and instruction-rate shares."""
    import gc
    import torch
    out = {"pictures": len(reqs), "decode_residuals": timed(lambda: bd.decode_residuals(reqs), reps)}
    out["c_abi_preallocated"] = timed(abi_call(bd, reqs), reps)
    gc.collect()
    torch.cuda.empty_cache()
    out["decode_coefficients"] = timed(lambda: bd.decode_coefficients(reqs), reps)
    gc.collect()
    torch.cuda.empty_cache()
    out["decode_pictures"] = timed(lambda: bd.decode_pictures(reqs), reps)
    gc.collect()
    torch.cuda.empty_cache()
    split = kernel_split(lambda: bd.decode_residuals(reqs))
    out["decode_residuals"]["split"] = split
    out["decode_residuals"]["pictures_per_s"] = len(reqs) / out["decode_residuals"]["best_s"]
    out["ratio_to_decode_coefficients"] = out["decode_residuals"]["best_s"] / out["decode_coefficients"]["best_s"]
    out["ratio_to_decode_pictures"] = out["decode_residuals"]["best_s"] / out["decode_pictures"]["best_s"]
    work = export_work(bd, reqs)
    secs = split["export_residuals_ms"] / 1000.0
    work["bytes_per_s"] = work["bytes"] / secs
    work["share_of_3_35_tb_s"] = work["bytes_per_s"] / PEAK_BYTES_PER_S
    work["static_sass_instructions"] = sass_len
    if max_sm_hz:
        issue = SMS * ISSUE_PER_SM * max_sm_hz
        work["issue_rate_warp_instr_per_s"] = issue
        work["full_warp_instructions_upper"] = work["full_warps"] * sass_len
        work["share_of_issue_rate_upper"] = work["full_warps"] * sass_len / secs / issue
    out["export_kernel"] = work
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
    from jsmpeg_b200.batch import BatchDecoder

    c = card()
    m = re.search(r"(\d+)\s*MHz\s*$", c)
    max_sm_hz = int(m.group(1)) * 1e6 if m else None
    result = {"card": c, "reps": args.reps}
    sass_len = static_instructions()

    # (a) the bench's 64 clips, per_clip listed pictures of each
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips), decode_b=True)
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    reqs = []
    for s in range(len(clips)):
        listed = [e["picture"] for e in bd.macroblock_index(s)]
        reqs += [(s, listed[i * len(listed) // args.per_clip]) for i in range(args.per_clip)]
    print(f"(a) {args.per_clip} pictures per clip, {len(reqs)} in one call", file=sys.stderr)
    result["a_many_streams"] = {"streams": len(clips), "clip": f"{bench.WIDTH}x{bench.HEIGHT}x{bench.PICTURES}",
                                "per_clip": args.per_clip, **leg(bd, reqs, args.reps, max_sm_hz, sass_len)}
    bd.close()

    # (b) one long stream, every listed picture
    es = b"".join(p for _, p in gen_streams.make_clip_es(bench.WIDTH, bench.HEIGHT, args.long_frames, seed=1234, noise=bench.NOISE))
    bd = BatchDecoder(1, decode_b=True)
    bd.write(0, es)
    every = [(0, e["picture"]) for e in bd.macroblock_index(0)]
    result["b_one_stream"] = {"clip": f"{bench.WIDTH}x{bench.HEIGHT}x{args.long_frames}",
                              **leg(bd, every, args.reps, max_sm_hz, sass_len)}
    bd.close()

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
