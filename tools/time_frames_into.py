#!/usr/bin/env python
"""Coefficient and map frames of decode(n) on the device: decode_frames_into against decode(n) and against the way
without it -- decode(1) per picture and a copy (maps) or a decode_coefficients (coefficients) of what it leaves.

    python tools/time_frames_into.py [--reps 5] [--pictures 8] [--out FILE]

The bench's 64 distinct 1080p clips (I and P pictures only; max_slots as bench.py), the first --pictures of each (8: 64 x
8 map frames are 12.8 GB beside the record slots).  Two phases, each with its own destinations (allocated once, with
torch, after the record slots), its variants alternated in every round after a warm-up round; each variant rewinds
first and ends in a device synchronise:
  (a) maps: "decode_acc" (decode(n, OUT_ACCUMULATED)), "into_acc" (decode_frames_into(n, OUT_ACCUMULATED) with map
      frames) and "live_acc" (n x decode(1, OUT_ACCUMULATED), each followed by a torch copy of every stream's
      device_accumulated into its frame);
  (b) coefficients: "decode" (decode(n)), "into_coef" (decode_frames_into(n) with coefficient frames) and "live_coef"
      (n x decode(1), each followed by one decode_coefficients call for the step's 64 pictures, into their frames).
Then, under torch.profiler in runs of their own, the device time per 64-picture step of accumulate_kernel in
"decode_acc" and "into_acc" and of export_coefficients_kernel in "into_coef", and the device events "into_acc" has and
"decode_acc" has not (the end-of-call map copies, whatever the profiler calls a batched copy).  Sampled frames of
"into_*" are checked against "live_*".  The card's name and power limit are read in the same process.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_frames import timed, view  # noqa: E402
from time_intra import card  # noqa: E402

KERNELS = ("accumulate_kernel", "export_coefficients_kernel", "Memcpy DtoD")


def kernel_ms(fn):
    """{kernel or copy kind: {"ms": device time, "count": n}} of KERNELS in one call of fn, and under "all" every
    device event's {"ms", "count"} by its name"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    out = {k: {"ms": 0.0, "count": 0} for k in KERNELS}
    out["all"] = {e.key: {"ms": e.device_time_total / 1000.0, "count": e.count} for e in prof.key_averages()
                  if e.device_time_total > 0}
    for e in prof.key_averages():
        for k in KERNELS:
            if k + "(" in e.key or e.key.endswith(k) or (k.startswith("Memcpy") and e.key.startswith(k)):
                out[k]["ms"] += e.device_time_total / 1000.0
                out[k]["count"] += e.count
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pictures", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import bench
    from jsmpeg_b200.batch import OUT_ACCUMULATED, OUT_DEVICE, BatchDecoder, FrameDst

    clips = bench.load_streams(bench.rank_seeds(0))
    S, P, N = len(clips), bench.PICTURES, args.pictures
    bd = BatchDecoder(S, max_slots=S * P + 8)
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    assert bd.decode(P) == S * P  # (the record slots exist before the destinations are allocated)
    info = bd.stream_info(0)
    cs, W, H = info["coded_size"], info["width"], info["height"]
    mb_h, mb_w = (H + 15) // 16, (W + 15) // 16
    VP = ctypes.c_void_p * S
    n_frames = (ctypes.c_int32 * S)()

    def into(n, flags, coef=None, acc=None):
        bd.rewind()
        arrs = [None if t is None else VP(*[t[s].data_ptr() for s in range(S)]) for t in (coef, acc)]
        dst = FrameDst(None, None, None, None, *[None if a is None else ctypes.addressof(a) for a in arrs])
        assert bd.lib.jsmpeg_b200_batch_decode_frames_into(bd.handle, n, flags, ctypes.byref(dst), None, n_frames) == S * n
        assert list(n_frames) == [n] * S

    def decode(n, flags=OUT_DEVICE):
        bd.rewind()
        assert bd.decode(n, flags) == S * n

    def live(n, flags, after):
        bd.rewind()
        for j in range(n):
            assert bd.decode(1, flags) == S
            after(j)
            torch.cuda.synchronize()  # (the map a copy reads is rewritten two decode() calls later)

    result = {"card": card(), "reps": args.reps, "streams": S, "clip": f"{bench.WIDTH}x{bench.HEIGHT}", "pictures_per_stream": N,
              "pictures": S * N, "bytes_per_frame": {"coefficients": mb_h * mb_w * 768, "accumulated": cs * 12}}
    sample = [(s, j) for s in range(0, S, 9) for j in sorted({0, 1, N // 2, N - 1})]
    ok = True

    # (a) map frames
    maps = torch.empty((S, N, cs * 3 // 2, 4), dtype=torch.int16, device="cuda")

    def copy_maps(j):
        for s in range(S):
            maps[s, j].copy_(bd.device_accumulated(s), non_blocking=True)

    va = {"decode_acc": lambda: decode(N, OUT_ACCUMULATED), "into_acc": lambda: into(N, OUT_ACCUMULATED, acc=maps),
          "live_acc": lambda: live(N, OUT_ACCUMULATED, copy_maps)}
    result.update(timed(va, args.reps))
    into(N, OUT_ACCUMULATED, acc=maps)
    got = [maps[s, j].clone() for s, j in sample]
    live(N, OUT_ACCUMULATED, copy_maps)
    ok = ok and all(torch.equal(g, maps[s, j]) for g, (s, j) in zip(got, sample))
    prof = {"decode_acc": kernel_ms(va["decode_acc"]), "into_acc": kernel_ms(va["into_acc"])}
    del maps, got
    torch.cuda.empty_cache()

    # (b) coefficient frames
    coefs = torch.empty((S, N, mb_h, mb_w, 6, 8, 8), dtype=torch.int16, device="cuda")
    streams = (ctypes.c_int * S)(*range(S))

    def export_step(j):  # picture j of every stream (rewound: picture j is the j-th decode(1) reconstructs)
        pictures = (ctypes.c_uint32 * S)(*[j] * S)
        dst = VP(*[coefs[s, j].data_ptr() for s in range(S)])
        assert bd.lib.jsmpeg_b200_batch_decode_coefficients(bd.handle, S, streams, pictures, dst, None, None, None) == S

    vb = {"decode": lambda: decode(N), "into_coef": lambda: into(N, OUT_DEVICE, coef=coefs),
          "live_coef": lambda: live(N, OUT_DEVICE, export_step)}
    result.update(timed(vb, args.reps))
    into(N, OUT_DEVICE, coef=coefs)
    got = [coefs[s, j].clone() for s, j in sample]
    live(N, OUT_DEVICE, export_step)
    ok = ok and all(torch.equal(g, coefs[s, j]) for g, (s, j) in zip(got, sample))
    prof["into_coef"] = kernel_ms(vb["into_coef"])
    del coefs, got
    bd.close()
    result["sampled_frames_equal"] = ok

    for name, base in (("into_acc", "decode_acc"), ("live_acc", "decode_acc"), ("live_acc", "into_acc"),
                       ("into_coef", "decode"), ("live_coef", "decode"), ("live_coef", "into_coef")):
        result[name]["over_" + base + "_median_ms"] = (result[name]["median_s"] - result[base]["median_s"]) * 1e3
    result["kernels"] = {
        "per_step_accumulate_kernel_ms": {k: prof[k]["accumulate_kernel"]["ms"] / N for k in ("decode_acc", "into_acc")},
        "per_step_export_coefficients_kernel_ms": prof["into_coef"]["export_coefficients_kernel"]["ms"] / N,
        "into_acc_only_events": {k: v for k, v in prof["into_acc"]["all"].items() if k not in prof["decode_acc"]["all"]},
        "counts": {k: {kk: v["count"] for kk, v in p.items() if kk != "all"} for k, p in prof.items()},
        "coefficient_bytes_per_step": S * mb_h * mb_w * 768,
    }

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    assert ok, "sampled frames of decode_frames_into differ from the per-picture way's"


if __name__ == "__main__":
    main()
