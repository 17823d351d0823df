#!/usr/bin/env python
"""Accumulated maps (BatchDecoder.decode_accumulated) against decoding the pictures and against what a user writes
without it.

    python tools/time_accumulated.py [--reps 3] [--per-clip 16] [--long-frames 600] [--out FILE]

(a) the first `per_clip` I/P pictures of each of the bench's 64 distinct 1080p x 60-picture clips in one call;
(b) every I/P picture of one 1080p stream of `long_frames` pictures (FFmpeg GOP 12) in one call.
Each leg against decode_pictures of the same requests, and against the loop a user writes today: decode_macroblocks
and decode_residuals of every reference picture of the requests' chains, then per picture one torch gather step
(torch_step, the rule of include/jsmpeg_b200.h on the device with torch ops), chain by chain.  Every call returns
after a device synchronise, so a host clock around it measures it.  Best of `reps` after a warm-up round.  One more
call of decode_accumulated runs under torch.profiler: its accumulate kernel time, and the kernel's bytes (per sample
and depth a map record read and one written, 16 bytes -- 8 for a chain's first picture, which reads none -- plus the
8-byte record word per macroblock) over it, against the H100 SXM data sheet's 3.35 TB/s.  The card's name and power limit are read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_coefficients import timed  # noqa: E402
from time_intra import card  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def torch_step(prev, ent, res, mbw, mbh):
    """One depth of the accumulated map with torch ops: prev int32 [n, 4] or None, ent the picture's
    decode_macroblocks entries [mbh, mbw, 16], res its decode_residuals residual [n].  int32 [n, 4]."""
    import torch
    e16 = ent.view(torch.int16)
    fx, fy, flags = e16[..., 0].int(), e16[..., 1].int(), ent[..., 8].int()
    n = mbw * mbh * 256
    out = []
    for k, (off, size) in enumerate(((0, n), (n, n // 4), (n + n // 4, n // 4))):
        px = 16 if k == 0 else 8
        vx, vy = (fx, fy) if k == 0 else (torch.div(fx, 2, rounding_mode="trunc"), torch.div(fy, 2, rounding_mode="trunc"))
        stride = mbw * px
        rows = torch.arange(mbh * px, device=ent.device)
        cols = torch.arange(stride, device=ent.device)

        def per_sample(x):
            return x.repeat_interleave(px, 0).repeat_interleave(px, 1).reshape(-1)
        sx, sy, sf = per_sample(vx), per_sample(vy), per_sample(flags)
        origin = ((rows // 8 * 8)[:, None] * stride + (cols // 8 * 8)[None, :]).reshape(-1)
        src = origin + (sy >> 1) * stride + (sx >> 1)
        inside = (src >= 0) & (src + 7 * stride + 7 + (sy & 1) * stride + (sx & 1) < size)
        present = (sf & 1) != 0
        predicted = present & ((sf & 2) == 0) & inside
        m = torch.zeros((size, 4), dtype=torch.int32, device=ent.device)
        m[:, 3] = torch.where(present & ~predicted, 0, -1)
        if prev is not None:
            i = torch.arange(size, device=ent.device)
            at = torch.where(predicted, i + (sy >> 1) * stride + (sx >> 1), 0)
            p = prev[off:off + size][at]
            ok = predicted & (p[:, 3] >= 0)
            new = torch.stack([p[:, 0] + sx, p[:, 1] + sy, p[:, 2] + res[off:off + size].int(), p[:, 3] + 1], 1)
            m = torch.where(ok[:, None], new.clamp(-32768, 32767), m)
        out.append(m)
    return torch.cat(out)


def user_loop(bd, reqs, chains):
    """What a user writes today: the chains' reference pictures exported, then a gather step per picture"""
    import torch
    pics = [(s, k) for s, ks in chains for k in ks]
    ents = bd.decode_macroblocks(pics)
    res = bd.decode_residuals(pics)
    wanted = set(reqs)
    at = {}
    j = 0
    for s, ks in chains:
        mbh, mbw = ents[j].shape[:2]
        prev = None
        for k in ks:
            prev = torch_step(prev, ents[j], res[j], mbw, mbh)
            if (s, k) in wanted:
                at[(s, k)] = prev.to(torch.int16)
            j += 1
    out = [at[r] for r in reqs]
    torch.cuda.synchronize()
    return out


def chains_of(bd, reqs):
    """[(stream, [reference pictures from the chain start to the last request])] of the requests"""
    last = {}
    for s, k in reqs:
        e = next(x for x in bd.picture_index(s) if x["picture"] == k)
        key = (s, e["chain_start"])
        last[key] = max(last.get(key, k), k)
    out = []
    for (s, start), k in sorted(last.items()):
        out.append((s, [e["picture"] for e in bd.picture_index(s) if e["type"] in (1, 2) and start <= e["picture"] <= k
                        and e["chain_start"] == start]))
    return out


def kernel_ms(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    total = {"accumulate_ms": 0.0, "other_kernels_and_copies_ms": 0.0}
    for e in prof.key_averages():
        ms = e.device_time_total / 1000.0
        total["accumulate_ms" if "accumulate_kernel" in e.key else "other_kernels_and_copies_ms"] += ms
    return total


def leg(bd, reqs, reps):
    import gc
    import torch
    chains = chains_of(bd, reqs)
    depths = sum(len(ks) for _, ks in chains)
    out = {"pictures": len(reqs), "chain_pictures": depths,
           "decode_accumulated": timed(lambda: bd.decode_accumulated(reqs), reps)}
    gc.collect()
    torch.cuda.empty_cache()
    out["decode_pictures"] = timed(lambda: bd.decode_pictures(reqs), reps)
    gc.collect()
    torch.cuda.empty_cache()
    few = reqs[:64]  # (the two results of every request at once would not fit the device)
    got = bd.decode_accumulated(few)
    mine = user_loop(bd, few, chains_of(bd, few))
    out["user_loop_equal_first_64"] = all(bool(torch.equal(a, b)) for a, b in zip(got, mine))
    del got, mine
    gc.collect()
    torch.cuda.empty_cache()
    out["user_loop"] = timed(lambda: user_loop(bd, reqs, chains), max(1, reps // 2))
    gc.collect()
    torch.cuda.empty_cache()
    split = kernel_ms(lambda: bd.decode_accumulated(reqs))
    info = bd.stream_info(reqs[0][0])
    samples = info["coded_size"] * 3 // 2
    nbytes = (depths * 16 - len(chains) * 8) * samples + depths * (info["coded_size"] // 256) * 8
    out["split"] = split
    out["accumulate_bytes"] = nbytes
    out["accumulate_bytes_per_s"] = nbytes / (split["accumulate_ms"] / 1000.0)
    out["share_of_3_35_tb_s"] = out["accumulate_bytes_per_s"] / PEAK_BYTES_PER_S
    out["ratio_to_decode_pictures"] = out["decode_accumulated"]["best_s"] / out["decode_pictures"]["best_s"]
    out["speedup_over_user_loop"] = out["user_loop"]["best_s"] / out["decode_accumulated"]["best_s"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--per-clip", type=int, default=16)
    ap.add_argument("--long-frames", type=int, default=600)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import bench
    import gen_streams
    from jsmpeg_b200.batch import BatchDecoder

    result = {"card": card(), "reps": args.reps}
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips))
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    reqs = [(s, e["picture"]) for s in range(len(clips)) for e in
            [x for x in bd.picture_index(s) if x["type"] in (1, 2)][:args.per_clip]]
    print(f"(a) {args.per_clip} I/P pictures per clip, {len(reqs)} in one call", file=sys.stderr)
    result["a_many_streams"] = {"streams": len(clips), "clip": f"{bench.WIDTH}x{bench.HEIGHT}x{bench.PICTURES}",
                                "per_clip": args.per_clip, **leg(bd, reqs, args.reps)}
    bd.close()

    es = b"".join(p for _, p in gen_streams.make_clip_es(bench.WIDTH, bench.HEIGHT, args.long_frames, seed=1234, noise=bench.NOISE))
    bd = BatchDecoder(1)
    bd.write(0, es)
    every = [(0, e["picture"]) for e in bd.picture_index(0) if e["type"] in (1, 2)]
    print(f"(b) {len(every)} I/P pictures of one stream", file=sys.stderr)
    result["b_one_stream"] = {"clip": f"{bench.WIDTH}x{bench.HEIGHT}x{args.long_frames}", **leg(bd, every, args.reps)}
    bd.close()

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
