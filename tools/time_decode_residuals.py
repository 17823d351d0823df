#!/usr/bin/env python
"""The residual on the playback path: decode() with and without OUT_RESIDUALS, and against the way without the flag --
decode(1) and then decode_residuals of the step's pictures, one step at a time.

    python tools/time_decode_residuals.py [--reps 7] [--out FILE]

The bench's 64 distinct 1080p x 60-picture clips (I and P pictures only, each followed by a sequence end code so that
decode_residuals can take its last picture; max_slots as bench.py), five variants alternated in every round of one
process:
  (a) "off" (decode(60)) and "on" (decode(60, OUT_RESIDUALS): the last step stores the 64 residuals);
  (b) the live loop, 60 x decode(1): "live_off", "live_on" (every step with the flag) and "live_export" (each
      decode(1) followed by the C call decode_residuals of the 64 pictures it consumed, into destinations allocated
      once: a second walk, expand and transform).
Each variant rewinds first and ends in a device synchronise, so a host clock around it measures it.  Best and median of
`reps` after a warm-up round.  Outside the timed rounds:
  * the residuals after "on" are checked against decode_residuals of picture 59;
  (c) one "live_off", one "live_on" and one "live_export" run under torch.profiler: the device time per step of
      reconstruct_kernel (live_off) and reconstruct_res_kernel (live_on) on the same steps, and that of
      export_residuals_kernel for the same 64 pictures per step (live_export) -- the fused store's cost against the
      unfused alternative's.
The card's name and power limit are read in the same process.
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

KERNELS = ("reconstruct_kernel", "reconstruct_res_kernel", "export_residuals_kernel")


def kernel_ms(fn):
    """{kernel: {"ms": device time, "launches": n}} of the KERNELS in one call of fn"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k + "(" in e.key or e.key.endswith(k):
                d = out.setdefault(k, {"ms": 0.0, "launches": 0})
                d["ms"] += e.device_time_total / 1000.0
                d["launches"] += e.count
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import bench
    from jsmpeg_b200.batch import OUT_DEVICE, OUT_RESIDUALS, BatchDecoder

    clips = bench.load_streams(bench.rank_seeds(0))
    S, P = len(clips), bench.PICTURES
    bd = BatchDecoder(S, max_slots=S * P + 8)
    for s, clip in enumerate(clips):
        bd.write(s, clip + b"\x00\x00\x01\xb7")  # (a sequence end code closes picture 59: the index lists it)
    assert all([e["picture"] for e in bd.macroblock_index(s)][:P] == list(range(P)) for s in range(S))
    res = bd.decode_residuals([(s, 0) for s in range(S)])  # the destinations, reused by every step
    streams = (ctypes.c_int * S)(*range(S))
    dst = (ctypes.c_void_p * S)(*[t.data_ptr() for t in res])

    def decode(flags):
        bd.rewind()
        assert bd.decode(P, flags) == S * P

    def live(flags, export=False):
        bd.rewind()
        for k in range(P):
            assert bd.decode(1, flags) == S
            if export:
                pictures = (ctypes.c_uint32 * S)(*([k] * S))
                assert bd.lib.jsmpeg_b200_batch_decode_residuals(bd.handle, S, streams, pictures, dst, None, None, None) == S

    variants = {"off": lambda: decode(OUT_DEVICE), "on": lambda: decode(OUT_RESIDUALS),
                "live_off": lambda: live(OUT_DEVICE), "live_on": lambda: live(OUT_RESIDUALS),
                "live_export": lambda: live(OUT_DEVICE, export=True)}
    times = {k: [] for k in variants}
    for rep in range(args.reps + 1):  # round 0 is the warm-up
        for name, fn in variants.items():
            t0 = time.perf_counter()
            fn()
            dt = time.perf_counter() - t0
            if rep:
                times[name].append(dt)

    decode(OUT_RESIDUALS)
    flag_res = [bd.device_residuals(s).clone() for s in range(S)]
    want = bd.decode_residuals([(s, P - 1) for s in range(S)])
    same = all(torch.equal(flag_res[s], want[s]) for s in range(S))
    del flag_res, want

    result = {"card": card(), "reps": args.reps, "streams": S, "clip": f"{bench.WIDTH}x{bench.HEIGHT}x{P}",
              "pictures": S * P, "last_residuals_equal": same}
    for name, ts in times.items():
        result[name] = {"best_s": min(ts), "median_s": statistics.median(ts), "all_s": ts}
    for name, base in (("on", "off"), ("live_on", "live_off"), ("live_export", "live_off")):
        result[name]["over_" + base + "_best_ms"] = (result[name]["best_s"] - result[base]["best_s"]) * 1e3
        result[name]["over_" + base + "_median_ms"] = (result[name]["median_s"] - result[base]["median_s"]) * 1e3
    prof = {"live_off": kernel_ms(lambda: live(OUT_DEVICE)), "live_on": kernel_ms(lambda: live(OUT_RESIDUALS)),
            "live_export": kernel_ms(lambda: live(OUT_DEVICE, export=True))}
    plain = prof["live_off"]["reconstruct_kernel"]
    fused = prof["live_on"]["reconstruct_res_kernel"]
    export = prof["live_export"]["export_residuals_kernel"]
    result["kernels"] = {
        "per_step_reconstruct_kernel_ms": plain["ms"] / plain["launches"],
        "per_step_reconstruct_res_kernel_ms": fused["ms"] / fused["launches"],
        "per_step_export_residuals_kernel_ms": export["ms"] / export["launches"],
        "launches": {"reconstruct_kernel": plain["launches"], "reconstruct_res_kernel": fused["launches"],
                     "export_residuals_kernel": export["launches"]},
    }
    kk = result["kernels"]
    kk["per_step_fused_store_ms"] = kk["per_step_reconstruct_res_kernel_ms"] - kk["per_step_reconstruct_kernel_ms"]
    kk["fused_store_cheaper_than_export"] = kk["per_step_fused_store_ms"] < kk["per_step_export_residuals_kernel_ms"]
    bd.close()

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    assert same, "the residuals after decode(60, OUT_RESIDUALS) differ from decode_residuals of picture 59"


if __name__ == "__main__":
    main()
