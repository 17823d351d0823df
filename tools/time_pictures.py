#!/usr/bin/env python
"""Random access (BatchDecoder.decode_pictures) against the serial decode() path.

    python tools/time_pictures.py [--reps 5] [--long-frames 600] [--compare-tree DIR] [--out FILE]

(a) every listed picture of one 1080p stream of `long_frames` pictures (FFmpeg GOP 12) in one call, against decode()
    with OUT_DEVICE of every picture;
(b) 8 evenly spaced listed pictures from each of the bench's 64 distinct 1080p x 60-picture clips in one call, against
    decode() of all 60 pictures of every clip;
(c) one seek: the last P picture before the final I picture of the long stream, against decode() from picture 0 up
    to it;
(d) with --compare-tree: tools/time_intra.py of DIR (a checkout of an earlier version, its library built) and of
    this tree, alternated three times in one job.
Every call returns after a device synchronise, so a host clock around it measures it (wall time, output tensors
included).  Best of `reps` after a warm-up round.  For (a) to (c) one more call runs under torch.profiler, whose
kernel times give the stage split: stage 1 (walk + expand kernels), stage 2 (reconstruct kernels), copies and fills.
The card's name and power limit are read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_intra import best_of, card  # noqa: E402


def stage_split(fn):
    """Device time (ms) of one call of `fn` by kind: stage 1, stage 2, copies / fills, other kernels."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"stage1_ms": 0.0, "stage2_ms": 0.0, "copy_fill_ms": 0.0, "other_ms": 0.0}
    for e in prof.key_averages():
        ms = e.device_time_total / 1000.0
        name = e.key.lower()
        if "reconstruct" in name:
            out["stage2_ms"] += ms
        elif "walk" in name or "expand" in name or "parse" in name:
            out["stage1_ms"] += ms
        elif "memcpy" in name or "memset" in name:
            out["copy_fill_ms"] += ms
        elif ms > 0:
            out["other_ms"] += ms
    return out


def timed(fn, reps):
    best, times = best_of(fn, reps)
    return {"best_s": best, "all_s": times}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--long-frames", type=int, default=600)
    ap.add_argument("--compare-tree", default=None, help="a built checkout of an earlier version, for leg (d)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import bench
    import gen_streams
    import numpy as np
    from jsmpeg_b200.batch import OUT_DEVICE, BatchDecoder

    result = {"card": card(), "reps": args.reps}

    # (a) + (c): one long stream
    es = b"".join(p for _, p in gen_streams.make_clip_es(bench.WIDTH, bench.HEIGHT, args.long_frames, seed=1234, noise=bench.NOISE))
    bd = BatchDecoder(1)
    bd.write(0, es)
    entries = bd.picture_index(0)
    every = [(0, e["picture"]) for e in entries]

    def serial(n):
        def run():
            bd.rewind()
            assert bd.decode(n, OUT_DEVICE) == n
        return run

    leg_a = {"clip": f"{bench.WIDTH}x{bench.HEIGHT}x{args.long_frames}", "pictures": len(every),
             "decode_pictures": timed(lambda: bd.decode_pictures(every), args.reps),
             "serial_decode": dict(timed(serial(args.long_frames), args.reps), pictures=args.long_frames)}
    leg_a["decode_pictures"]["split"] = stage_split(lambda: bd.decode_pictures(every))
    leg_a["speedup_vs_serial"] = leg_a["serial_decode"]["best_s"] / leg_a["decode_pictures"]["best_s"]
    result["a_every_picture"] = leg_a

    last_i = max(e["picture"] for e in entries if e["type"] == 1)
    seek = max(e["picture"] for e in entries if e["type"] == 2 and e["picture"] < last_i)
    leg_c = {"picture": seek, "decode_pictures": timed(lambda: bd.decode_pictures([(0, seek)]), args.reps),
             "serial_decode": dict(timed(serial(seek + 1), args.reps), pictures=seek + 1)}
    leg_c["decode_pictures"]["split"] = stage_split(lambda: bd.decode_pictures([(0, seek)]))
    leg_c["speedup_vs_serial"] = leg_c["serial_decode"]["best_s"] / leg_c["decode_pictures"]["best_s"]
    result["c_seek"] = leg_c
    bd.close()

    # (b) 64 clips x 8 evenly spaced pictures
    clips = bench.load_streams(bench.rank_seeds(0))
    bd = BatchDecoder(len(clips))
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    reqs = []
    for s in range(len(clips)):
        listed = [e["picture"] for e in bd.picture_index(s)]
        reqs += [(s, listed[int(i)]) for i in np.linspace(0, len(listed) - 1, 8).round()]

    def serial_all():
        bd.rewind()
        assert bd.decode(bench.PICTURES, OUT_DEVICE) == len(clips) * bench.PICTURES

    leg_b = {"streams": len(clips), "clip": f"{bench.WIDTH}x{bench.HEIGHT}x{bench.PICTURES}", "pictures": len(reqs),
             "decode_pictures": timed(lambda: bd.decode_pictures(reqs), args.reps),
             "serial_decode": dict(timed(serial_all, args.reps), pictures=len(clips) * bench.PICTURES)}
    leg_b["decode_pictures"]["split"] = stage_split(lambda: bd.decode_pictures(reqs))
    leg_b["decode_pictures"]["pictures_per_s"] = len(reqs) / leg_b["decode_pictures"]["best_s"]
    leg_b["speedup_vs_serial"] = leg_b["serial_decode"]["best_s"] / leg_b["decode_pictures"]["best_s"]
    result["b_sampled_frames"] = leg_b
    bd.close()

    # (d) decode_intra, an earlier version against this one, alternated
    if args.compare_tree:
        runs = {"compare": [], "this": []}
        env = {k: v for k, v in os.environ.items() if k != "JSMPEG_B200_LIB"}
        for _ in range(3):
            for which, tree in (("compare", os.path.abspath(args.compare_tree)), ("this", ROOT)):
                out = subprocess.run([sys.executable, os.path.join(tree, "tools", "time_intra.py"), "--reps", str(args.reps)],
                                     env=env, capture_output=True, text=True, check=True, cwd=tree).stdout
                r = json.loads(out.strip().splitlines()[-1])
                runs[which].append({"many_streams_s": r["many_streams"]["best_s"],
                                    "one_stream_s": r["one_stream"]["decode_intra"]["best_s"]})
        result["d_decode_intra_ab"] = {
            "runs": runs,
            "best": {w: {k: min(r[k] for r in v) for k in ("many_streams_s", "one_stream_s")} for w, v in runs.items()}}

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
