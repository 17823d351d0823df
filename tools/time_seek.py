#!/usr/bin/env python
"""Seeking decode() (BatchDecoder.seek_pictures) against the other ways to reach the same pictures.

    python tools/time_seek.py [--reps 5] [--long-frames 600] [--seeks 50] [--flags 0] [--out FILE]

(a) the bench's 64 distinct 1080p x 60-picture clips: every stream seeks to a seeded random listed P picture k (with
    16 listed pictures after it) in one call, then decode(16).  Timed: the seek alone; the seek + decode(16);
    decode_pictures of the same 64 pictures (the same chain work, into destinations); decode_pictures of the same
    1,024 pictures k + 1 .. k + 16; and the same states reached without the call: one single-stream batch per stream,
    set_index to the chain start j, then decode() k - j + 1 times (all 64 one after the other).
(b) one 1080p stream of `long_frames` pictures: `seeks` seeded seeks to listed pictures, one call each, against
    set_index to the chain start and sequential decode() up to the picture, for each of them.
Every seek passes `flags` (jsmpeg_b200.batch's OUT_* bits; default 0, OUT_DEVICE).  Every call returns after a device
synchronise, so a host clock around it measures it.  Best of `reps` after a warm-up round.  One more seek of (a) runs
under torch.profiler for the stage split (tools/time_pictures.py).  The card's name and power limit are read in the
same process.
"""
from __future__ import annotations

import argparse
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_intra import card  # noqa: E402
from time_pictures import stage_split, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--long-frames", type=int, default=600)
    ap.add_argument("--seeks", type=int, default=50)
    ap.add_argument("--flags", type=int, default=0, help="OUT_* bits of every seek, e.g. 5 = OUT_HOST | OUT_MACROBLOCKS")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import bench
    import gen_streams
    from jsmpeg_b200.batch import OUT_DEVICE, BatchDecoder

    result = {"card": card(), "reps": args.reps, "flags": args.flags}
    rng = random.Random(2026)

    # (a) 64 clips, one seek each, then 16 pictures
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips))
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    targets = []  # per stream: (k, its chain start, the 16 listed pictures after k)
    for s in range(len(clips)):
        listed = bd.picture_index(s)
        at = rng.choice([i for i, e in enumerate(listed) if e["type"] == 2 and i + 16 < len(listed)])
        targets.append((listed[at]["picture"], listed[at]["chain_start"], [e["picture"] for e in listed[at + 1:at + 17]]))
    seeks = [(s, k) for s, (k, _, _) in enumerate(targets)]
    following = [(s, p) for s, (_, _, after) in enumerate(targets) for p in after]

    def seek_and_play():
        assert bd.seek_pictures(seeks, args.flags) == len(seeks)
        assert bd.decode(16, OUT_DEVICE) == 16 * len(seeks)

    singles = []
    for clip in clips:
        one = BatchDecoder(1, max_slots=32)
        one.write(0, clip)
        singles.append((one, one.picture_index(0)))

    def without_the_call():
        for (one, listed), (k, j, _) in zip(singles, targets):
            one.set_index(0, listed[[e["picture"] for e in listed].index(j)]["byte_pos"] * 8)
            assert one.decode(k - j + 1, OUT_DEVICE) == k - j + 1

    leg_a = {"streams": len(clips), "clip": f"{bench.WIDTH}x{bench.HEIGHT}x{bench.PICTURES}",
             "chain_pictures": sum(k - j + 1 for k, j, _ in targets),
             "seek": timed(lambda: bd.seek_pictures(seeks, args.flags), args.reps),
             "seek_then_decode_16": timed(seek_and_play, args.reps),
             "decode_pictures_same_64": timed(lambda: bd.decode_pictures(seeks), args.reps),
             "decode_pictures_same_1024": dict(timed(lambda: bd.decode_pictures(following), args.reps), pictures=len(following)),
             "set_index_and_decode_per_stream": timed(without_the_call, args.reps)}
    leg_a["seek"]["split"] = stage_split(lambda: bd.seek_pictures(seeks, args.flags))
    for one, _ in singles:
        one.close()
    bd.close()
    result["a_64_streams"] = leg_a

    # (b) one long stream, one seek per call
    es = b"".join(p for _, p in gen_streams.make_clip_es(bench.WIDTH, bench.HEIGHT, args.long_frames, seed=1234, noise=bench.NOISE))
    bd = BatchDecoder(1)
    bd.write(0, es)
    listed = bd.picture_index(0)
    pos = {e["picture"]: e["byte_pos"] for e in listed}
    picks = [rng.choice(listed) for _ in range(args.seeks)]

    def seek_each():
        for e in picks:
            assert bd.seek_pictures([(0, e["picture"])], args.flags) == 1

    def sequential_each():
        for e in picks:
            bd.set_index(0, pos[e["chain_start"]] * 8)
            assert bd.decode(e["picture"] - e["chain_start"] + 1, OUT_DEVICE) == e["picture"] - e["chain_start"] + 1

    leg_b = {"clip": f"{bench.WIDTH}x{bench.HEIGHT}x{args.long_frames}", "seeks": len(picks),
             "chain_pictures": sum(e["picture"] - e["chain_start"] + 1 for e in picks),
             "seek_pictures": timed(seek_each, args.reps), "set_index_and_decode": timed(sequential_each, args.reps)}
    leg_b["speedup"] = leg_b["set_index_and_decode"]["best_s"] / leg_b["seek_pictures"]["best_s"]
    bd.close()
    result["b_one_stream"] = leg_b

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
