#!/usr/bin/env python
"""Every picture of decode(n) on the device: decode_frames against decode(n) and against the way without it -- decode(1)
per picture and a copy of what it leaves.

    python tools/time_frames.py [--reps 5] [--out FILE]

The bench's 64 distinct 1080p x 60-picture clips (I and P pictures only; max_slots as bench.py, so a call is one round).
Three phases, each with its own destinations (allocated once per phase, with torch, after the record slots), its
variants alternated in every round after a warm-up round; each variant rewinds first and ends in a device synchronise:
  (a) "decode" (decode(60)), "frames" (decode_frames(60), planar frames) and "live_copy" (60 x decode(1), each followed by
      a torch copy of every stream's device_planes into its frame);
  (b) "frames_res_mb" (decode_frames(60) with residual and macroblock frames) and "live_res_mb" (60 x decode(1,
      OUT_RESIDUALS | OUT_MACROBLOCKS), each followed by copies of device_residuals and device_macroblocks);
  (c) at 30 pictures (RGBA frames of 60 do not fit beside the slots): "decode_rgba" (decode(30, OUT_RGBA)), "frames_rgba"
      (decode_frames(30) with RGBA frames) and "live_rgba" (30 x decode(1, OUT_RGBA) + a copy of each read_rgba view).
Then, under torch.profiler in runs of their own, the decision rule of DESIGN 3.16: the device time per step of
reconstruct_frame_kernel in "frames" against reconstruct_kernel in "decode" (the fused planar store's cost), and that of
the 64 device-to-device copies of one step in "live_copy" (the copy-out's).  The frames are checked against decode(1)'s
planes on sampled pictures.  The card's name and power limit are read in the same process.
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

KERNELS = ("reconstruct_kernel", "reconstruct_frame_kernel", "Memcpy DtoD")


def kernel_ms(fn):
    """{kernel or copy kind: {"ms": device time, "count": n}} of KERNELS in one call of fn"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k + "(" in e.key or e.key.endswith(k) or (k.startswith("Memcpy") and e.key.startswith(k)):
                d = out.setdefault(k, {"ms": 0.0, "count": 0})
                d["ms"] += e.device_time_total / 1000.0
                d["count"] += e.count
    return out


def view(ptr, shape, typestr):
    import torch

    class _V:
        __cuda_array_interface__ = {"data": (ptr, False), "shape": shape, "typestr": typestr, "version": 2}

    return torch.as_tensor(_V(), device="cuda")


def timed(variants, reps):
    times = {k: [] for k in variants}
    for rep in range(reps + 1):  # round 0 is the warm-up
        for name, fn in variants.items():
            t0 = time.perf_counter()
            fn()
            dt = time.perf_counter() - t0
            if rep:
                times[name].append(dt)
    return {k: {"best_s": min(v), "median_s": statistics.median(v), "all_s": v} for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import bench
    from jsmpeg_b200.batch import OUT_DEVICE, OUT_MACROBLOCKS, OUT_RESIDUALS, OUT_RGBA, BatchDecoder

    clips = bench.load_streams(bench.rank_seeds(0))
    S, P = len(clips), bench.PICTURES
    bd = BatchDecoder(S, max_slots=S * P + 8)
    for s, clip in enumerate(clips):
        bd.write(s, clip)
    assert bd.decode(P) == S * P  # (the record slots exist before the destinations are allocated)
    info = bd.stream_info(0)
    cs, W, H = info["coded_size"], info["width"], info["height"]
    mb_bytes = (W + 15) // 16 * ((H + 15) // 16) * 16
    VP = ctypes.c_void_p * S
    n_frames = (ctypes.c_int32 * S)()

    def frames(n, flags=OUT_DEVICE, planes=None, rgba=None, res=None, mb=None):
        bd.rewind()
        arrs = [None if t is None else VP(*[t[s].data_ptr() for s in range(S)]) for t in (planes, rgba, res, mb)]
        assert bd.lib.jsmpeg_b200_batch_decode_frames(bd.handle, n, flags, *arrs, None, n_frames) == S * n
        assert list(n_frames) == [n] * S

    def decode(n, flags=OUT_DEVICE):
        bd.rewind()
        assert bd.decode(n, flags) == S * n

    def live(n, flags, copy):
        bd.rewind()
        for j in range(n):
            assert bd.decode(1, flags) == S
            for s in range(S):
                copy(s, j)
            torch.cuda.synchronize()  # (the set a copy reads is rewritten two decode() calls later)

    result = {"card": card(), "reps": args.reps, "streams": S, "clip": f"{bench.WIDTH}x{bench.HEIGHT}x{P}",
              "pictures": S * P, "bytes_per_frame": {"planes": cs * 3 // 2, "rgba": W * H * 4, "residuals": cs * 3,
                                                     "macroblocks": mb_bytes}}

    # (a) planar frames
    planes = torch.empty((S, P, cs * 3 // 2), dtype=torch.uint8, device="cuda")

    def copy_planes(s, j):
        planes[s, j].copy_(view(bd.device_planes(s)[0], (cs * 3 // 2,), "|u1"), non_blocking=True)

    va = {"decode": lambda: decode(P), "frames": lambda: frames(P, planes=planes),
          "live_copy": lambda: live(P, OUT_DEVICE, copy_planes)}
    result.update(timed(va, args.reps))
    frames(P, planes=planes)
    ok = True
    bd.rewind()
    for j in range(P):
        bd.decode(1)
        if j in (0, 1, P // 2, P - 1):
            for s in range(0, S, 5):
                ok = ok and torch.equal(planes[s, j], view(bd.device_planes(s)[0], (cs * 3 // 2,), "|u1"))
    result["sampled_frames_equal"] = ok
    prof = {"decode": kernel_ms(va["decode"]), "frames": kernel_ms(va["frames"]), "live_copy": kernel_ms(va["live_copy"])}
    del planes
    torch.cuda.empty_cache()

    # (b) residual and macroblock frames
    res = torch.empty((S, P, cs * 3 // 2), dtype=torch.int16, device="cuda")
    mb = torch.empty((S, P, mb_bytes), dtype=torch.uint8, device="cuda")

    def copy_res_mb(s, j):
        res[s, j].copy_(bd.device_residuals(s), non_blocking=True)
        mb[s, j].copy_(bd.device_macroblocks(s).view(-1), non_blocking=True)

    vb = {"frames_res_mb": lambda: frames(P, res=res, mb=mb),
          "live_res_mb": lambda: live(P, OUT_RESIDUALS | OUT_MACROBLOCKS, copy_res_mb)}
    result.update(timed(vb, args.reps))
    del res, mb
    torch.cuda.empty_cache()

    # (c) RGBA frames, 30 pictures
    R = P // 2
    rgba = torch.empty((S, R, H, W, 4), dtype=torch.uint8, device="cuda")
    rgba_ptr = [None] * S

    def copy_rgba(s, j):
        if rgba_ptr[s] is None:
            p = ctypes.c_void_p()
            assert bd.lib.jsmpeg_b200_batch_get_rgba(bd.handle, s, ctypes.byref(p)) == 0
            rgba_ptr[s] = view(p.value, (H, W, 4), "|u1")
        rgba[s, j].copy_(rgba_ptr[s], non_blocking=True)

    vc = {"decode_rgba": lambda: decode(R, OUT_RGBA), "frames_rgba": lambda: frames(R, rgba=rgba),
          "live_rgba": lambda: live(R, OUT_RGBA, copy_rgba)}
    result.update(timed(vc, args.reps))
    del rgba
    bd.close()

    for name, base in (("frames", "decode"), ("live_copy", "decode"), ("live_copy", "frames"),
                       ("live_res_mb", "frames_res_mb"), ("frames_rgba", "decode_rgba"), ("live_rgba", "frames_rgba")):
        result[name]["over_" + base + "_median_ms"] = (result[name]["median_s"] - result[base]["median_s"]) * 1e3
    plain = prof["decode"]["reconstruct_kernel"]
    fused = prof["frames"]["reconstruct_frame_kernel"]
    copies = prof["live_copy"]["Memcpy DtoD"]
    kk = {"per_step_reconstruct_kernel_ms": plain["ms"] / P, "per_step_reconstruct_frame_kernel_ms": fused["ms"] / P,
          "per_step_d2d_copy_of_64_pictures_ms": copies["ms"] / P,
          "launches": {"reconstruct_kernel": plain["count"], "reconstruct_frame_kernel": fused["count"],
                       "d2d_copies": copies["count"]}}
    kk["per_step_fused_store_ms"] = kk["per_step_reconstruct_frame_kernel_ms"] - kk["per_step_reconstruct_kernel_ms"]
    kk["fused_store_cheaper_than_copy"] = kk["per_step_fused_store_ms"] < kk["per_step_d2d_copy_of_64_pictures_ms"]
    result["kernels"] = kk

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    assert ok, "sampled frames of decode_frames(60) differ from decode(1)'s planes"


if __name__ == "__main__":
    main()
