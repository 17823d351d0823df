#!/usr/bin/env python
"""Frames of decode(n) in display order: decode_frames_display against decode_frames_into in coded order, and against
the way without it -- coded frames, then a torch gather into display order plus the I/P frame carried into the next call.

    python tools/time_frames_display.py [--reps 5] [--streams 64] [--calls 6,6] [--out FILE]

64 streams of the 720p I/P/B fixture (tests/fixtures/b_clip_1280x720.m1v: I P B B P B B ..., 13 pictures), decode_b on.
Each variant rewinds, then makes the calls (--calls: pictures per call) and ends in a device synchronise; the variants
are alternated in every round after a warm-up round, medians reported.  Two sets of kinds: planes alone, and planes +
residual + macroblock entries.  Variants per set: "coded" (decode_frames_into), "display" (decode_frames_display) and
"gather" (decode_frames_into into a scratch, then per call one index_select of every kind into display order, the
carried frame written first, and the call's last I/P frame copied out as the next call's carry).  The display frames are
checked against the gather's.  Under torch.profiler, in runs of their own, the device events "display" has and "coded"
has not (the store copies of held pictures).  The card's name and power limit are read in the same process.
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

from display_model import DisplayModel  # noqa: E402
from time_frames import timed  # noqa: E402
from time_frames_into import kernel_ms  # noqa: E402
from time_intra import card  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "fixtures", "b_clip_1280x720.m1v")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--streams", type=int, default=64)
    ap.add_argument("--calls", default="6,6")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from jsmpeg_b200.batch import OUT_DEVICE, BatchDecoder, Frame, FrameDst

    S, calls = args.streams, [int(c) for c in args.calls.split(",")]
    es = open(FIXTURE, "rb").read()
    bd = BatchDecoder(S, decode_b=True)
    for s in range(S):
        bd.write(s, es)
    assert bd.decode(sum(calls)) == S * sum(calls)  # (the record slots exist before the destinations are allocated)
    info = bd.stream_info(0)
    cs, W, H = info["coded_size"], info["width"], info["height"]
    dev = torch.device("cuda", 0)
    N = max(calls)
    shapes = {"planes": ((cs * 3 // 2,), torch.uint8), "residuals": ((cs * 3 // 2,), torch.int16),
              "macroblocks": ((cs // 256, 16), torch.uint8)}
    field = {"planes": "planes", "residuals": "res", "macroblocks": "mb"}
    VP = ctypes.c_void_p * S
    n_frames = (ctypes.c_int32 * S)()
    info_out = (Frame * (S * (N + 1)))()

    def buffers(kinds, n):
        return {k: torch.empty((S, n, *shapes[k][0]), dtype=shapes[k][1], device=dev) for k in kinds}

    def frame_dst(bufs):
        arrs = {k: VP(*[t[s].data_ptr() for s in range(S)]) for k, t in bufs.items()}
        return FrameDst(**{field[k]: ctypes.addressof(a) for k, a in arrs.items()}), arrs

    def run(bufs, display, after=None):
        bd.rewind()
        dst, keep = frame_dst(bufs)
        for n in calls:
            fn = bd.lib.jsmpeg_b200_batch_decode_frames_display if display else bd.lib.jsmpeg_b200_batch_decode_frames_into
            assert fn(bd.handle, n, OUT_DEVICE, ctypes.byref(dst), info_out, n_frames) == S * n
            if after:
                after(n)
        torch.cuda.synchronize()
        return keep

    # the gather's order, from stream 0's frame infos (every stream is the same clip): per call, the coded frames'
    # presentation order, with -1 for the carried frame, and the frame it carries on
    bd.rewind()
    model, plans = DisplayModel(True), []
    for n in calls:
        assert bd.lib.jsmpeg_b200_batch_decode_frames_into(bd.handle, n, OUT_DEVICE, ctypes.byref(FrameDst()), info_out, n_frames) == S * n
        coded = [{"type": info_out[j].picture_type, "j": j} for j in range(n_frames[0])]
        carried = model.held
        shown = model.call(coded)
        plans.append(([-1 if f is carried else f["j"] for f in shown], model.held["j"] if model.held else None))
    torch.cuda.synchronize()

    result = {"card": card(), "reps": args.reps, "streams": S, "clip": f"{W}x{H} I/P/B (decode_b)", "calls": calls,
              "frames_per_call_display": [len(p) for p, _ in plans]}
    ok = True
    for label, kinds in (("planes", ("planes",)), ("planes_res_mb", ("planes", "residuals", "macroblocks"))):
        coded, shown = buffers(kinds, N), buffers(kinds, N + 1)
        carry = {k: torch.empty((S, *shapes[k][0]), dtype=shapes[k][1], device=dev) for k in kinds}
        gathered = buffers(kinds, N + 1)
        state = {"call": 0}

        def gather(n):
            order, held = plans[state["call"] % len(plans)]
            state["call"] += 1
            src = torch.tensor([j for j in order if j >= 0], dtype=torch.long, device=dev)
            to = torch.tensor([p for p, j in enumerate(order) if j >= 0], dtype=torch.long, device=dev)
            for k in kinds:
                if -1 in order:
                    gathered[k][:, order.index(-1)].copy_(carry[k])
                gathered[k].index_copy_(1, to, coded[k].index_select(1, src))
                if held is not None:
                    carry[k].copy_(coded[k][:, held])

        variants = {f"coded_{label}": lambda: run(coded, False), f"display_{label}": lambda: run(shown, True),
                    f"gather_{label}": lambda: run(coded, False, gather)}
        result.update(timed(variants, args.reps))
        run(shown, True)
        state["call"] = 0
        run(coded, False, gather)  # (the last call's frames, both ways)
        last = len(plans[-1][0])
        ok = ok and all(torch.equal(shown[k][:, :last], gathered[k][:, :last]) for k in kinds)
        pc, pd = kernel_ms(variants[f"coded_{label}"]), kernel_ms(variants[f"display_{label}"])
        result[f"display_only_events_{label}"] = {k: v for k, v in pd["all"].items() if k not in pc["all"]}
        result[f"device_ms_{label}"] = {"coded": sum(v["ms"] for v in pc["all"].values()),
                                        "display": sum(v["ms"] for v in pd["all"].values())}
        for name, base in (("display", "coded"), ("gather", "coded"), ("gather", "display")):
            a, b = f"{name}_{label}", f"{base}_{label}"
            result[a][f"over_{b}_median_ms"] = (result[a]["median_s"] - result[b]["median_s"]) * 1e3
        del coded, shown, carry, gathered
        torch.cuda.empty_cache()
    bd.close()
    result["display_frames_equal_gather"] = ok

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    assert ok, "decode_frames_display's frames differ from the gathered coded frames"


if __name__ == "__main__":
    main()
