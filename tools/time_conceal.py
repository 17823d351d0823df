#!/usr/bin/env python
"""What the conceal option costs: decode(60) of the bench's 64 streams of 1080p with about one picture in six damaged
by a lost transport packet, with and without conceal.

    python tools/time_conceal.py [--reps 5] [--every 6] [--out FILE]

Each stream of the bench's workload (bench.load_streams) loses one 184-byte run from inside every `--every`-th picture
(conceal_model.lost_packets), so its walk stops early or skips slices there.  One batch per variant; each
rewinds and decodes 60 pictures into device planes, ending in a device synchronise.  The variants alternate in every
round after a warm-up round; medians reported.  In runs of their own under torch.profiler: conceal_kernel's device time
and launches, and the reconstruct kernels' for comparison.  Also: the pictures with an error and every picture's
n_present other than the picture's size (from decode_frames' infos), and how many pictures the two variants give
differently.  The card's name and power limit are read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_frames import timed  # noqa: E402
from time_intra import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--every", type=int, default=6)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from jsmpeg_b200.batch import OUT_DEVICE, BatchDecoder
    from conceal_model import lost_packets

    clips = [lost_packets(es, args.every, seed=i) for i, es in enumerate(bench.load_streams(bench.rank_seeds(0)))]
    S, P = len(clips), bench.PICTURES
    batches = {}
    for name, on in (("off", 0), ("on", 1)):
        bd = BatchDecoder(S, max_slots=S * P + 8, conceal=on)
        for s, es in enumerate(clips):
            bd.write(s, es)
        batches[name] = bd

    consumed = {}

    def run(name):
        bd = batches[name]
        bd.rewind()
        consumed[name] = bd.decode(P, OUT_DEVICE)
        torch.cuda.synchronize()

    result = {"card": card(), "reps": args.reps, "streams": S, "pictures": P, "damaged_every": args.every}
    result.update(timed({"off": lambda: run("off"), "on": lambda: run("on")}, args.reps))
    result["pictures_consumed"] = consumed
    result["on_over_off_median_ms"] = (result["on"]["median_s"] - result["off"]["median_s"]) * 1e3

    for name in ("off", "on"):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(name)
        ev = {e.key: {"ms": e.device_time_total / 1000.0, "count": e.count} for e in prof.key_averages()
              if e.device_time_total > 0 and ("conceal" in e.key or "reconstruct" in e.key)}
        result[f"kernels_{name}"] = ev
    for bd in batches.values():
        bd.close()
    batches.clear()
    torch.cuda.empty_cache()

    # the damage, from decode_frames' infos, and how many pictures differ: a batch of its own per variant (the frames
    # do not fit beside the timed batches' record slots), each frame reduced to a fingerprint
    def frames_of(on):
        bd = BatchDecoder(S, conceal=on)
        for s, es in enumerate(clips):
            bd.write(s, es)
        frames = bd.decode_frames(P, planes=True)
        w = torch.arange(1, frames[0]["planes"].shape[1] + 1, device=frames[0]["planes"].device, dtype=torch.int64)
        prints = [[int((f["planes"][j].to(torch.int64) * w).sum()) for j in range(f["n_frames"])] for f in frames]
        infos = [f["info"] for f in frames]
        bd.close()
        del frames, bd
        torch.cuda.empty_cache()
        return prints, infos

    on_prints, infos = frames_of(1)
    off_prints, _ = frames_of(0)
    mb_size = ((bench.WIDTH + 15) // 16) * ((bench.HEIGHT + 15) // 16)
    result.update(pictures_total=sum(len(i) for i in infos),
                  pictures_with_error=sum(r["error"] != 0 for i in infos for r in i),
                  pictures_short_of_mb_size=sum(r["n_present"] != mb_size for i in infos for r in i),
                  pictures_that_differ=sum(a != b for x, y in zip(on_prints, off_prints) for a, b in zip(x, y)))

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
