#!/usr/bin/env python
"""Accumulated maps on the playback path: decode() with and without OUT_ACCUMULATED, and against the way without the
flag -- decode(1) and then decode_accumulated of the step's pictures, one step at a time.

    python tools/time_decode_accumulated.py [--reps 7] [--out FILE]

The bench's 64 distinct 1080p x 60-picture clips (I and P pictures only, each followed by a sequence end code so that
decode_accumulated can take its last picture; max_slots as bench.py), three variants
alternated in every round of one process: "off" (decode(60)), "on" (decode(60, OUT_ACCUMULATED)) and "per_step" (60 x
decode(1) followed by the C call decode_accumulated of the 64 pictures that step consumed, into destinations allocated
once: every call re-walks and re-accumulates each picture's chain from its I picture).  Each variant rewinds first and
ends in a device synchronise, so a host clock around it measures it.  Best and median of `reps` after a warm-up round.
Outside the timed rounds: the maps of the last step of "per_step" are checked against those of "on", and the accumulate
kernel's device time in one "on" and one "per_step" run is read under torch.profiler.  The card's name and power limit
are read in the same process.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_intra import card  # noqa: E402


def accumulate_ms(fn):
    """Device time (ms) of the accumulate kernel in one call of fn, and its launches."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    ms, launches = 0.0, 0
    for e in prof.key_averages():
        if "accumulate_kernel" in e.key:
            ms += e.device_time_total / 1000.0
            launches += e.count
    return {"accumulate_ms": ms, "accumulate_launches": launches}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import bench
    from jsmpeg_b200.batch import OUT_ACCUMULATED, OUT_DEVICE, BatchDecoder

    clips = bench.load_streams(bench.rank_seeds(0))
    S, P = len(clips), bench.PICTURES
    bd = BatchDecoder(S, max_slots=S * P + 8)
    for s, clip in enumerate(clips):
        bd.write(s, clip + b"\x00\x00\x01\xb7")  # (a sequence end code closes picture 59: the index lists it)
    assert all([e["picture"] for e in bd.picture_index(s)][:P] == list(range(P)) for s in range(S))
    maps = bd.decode_accumulated([(s, 0) for s in range(S)])  # the destinations, reused by every step
    streams = (ctypes.c_int * S)(*range(S))
    dst = (ctypes.c_void_p * S)(*[t.data_ptr() for t in maps])
    status = (ctypes.c_int32 * S)()

    def decode(flags):
        bd.rewind()
        assert bd.decode(P, flags) == S * P

    def per_step():
        bd.rewind()
        for k in range(P):
            assert bd.decode(1, OUT_DEVICE) == S
            pictures = (ctypes.c_uint32 * S)(*([k] * S))
            assert bd.lib.jsmpeg_b200_batch_decode_accumulated(bd.handle, S, streams, pictures, dst, status, None, None) == S

    variants = {"off": lambda: decode(OUT_DEVICE), "on": lambda: decode(OUT_ACCUMULATED), "per_step": per_step}
    times = {k: [] for k in variants}
    for rep in range(args.reps + 1):  # round 0 is the warm-up
        for name, fn in variants.items():
            t0 = time.perf_counter()
            fn()
            dt = time.perf_counter() - t0
            if rep:
                times[name].append(dt)

    decode(OUT_ACCUMULATED)
    flag_maps = [bd.device_accumulated(s).clone() for s in range(S)]
    per_step()
    same = all(status[s] == 1 and torch.equal(maps[s], flag_maps[s]) for s in range(S))
    del flag_maps

    result = {"card": card(), "reps": args.reps, "streams": S, "clip": f"{bench.WIDTH}x{bench.HEIGHT}x{P}",
              "pictures": S * P, "last_step_maps_equal": same}
    for name, ts in times.items():
        result[name] = {"best_s": min(ts), "median_s": statistics.median(ts), "all_s": ts}
    for name in ("on", "per_step"):
        result[name]["over_off_best_ms"] = (result[name]["best_s"] - result["off"]["best_s"]) * 1e3
        result[name]["over_off_median_ms"] = (result[name]["median_s"] - result["off"]["median_s"]) * 1e3
    result["on"].update(accumulate_ms(lambda: decode(OUT_ACCUMULATED)))
    result["on"]["accumulate_ms_per_step"] = result["on"]["accumulate_ms"] / P
    result["per_step"].update(accumulate_ms(per_step))
    bd.close()

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    assert same, "per_step's maps of the last step differ from OUT_ACCUMULATED's"


if __name__ == "__main__":
    main()
