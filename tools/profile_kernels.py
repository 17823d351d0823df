#!/usr/bin/env python
"""GPU helper: per-kernel device time of one decode step (bench-like workload) under torch.profiler.

    python tools/profile_kernels.py OUT.json [streams] [pictures]

The step is the one tools/time_stages.py times (64 x 1080p x 60 pictures by default, OUT_DEVICE); one untraced
step warms it up first.  OUT.json gets, per kernel name, the number of launches, the summed device time and the
first start and last end relative to the step's first kernel (which kernels ran side by side), plus the card's name
and power limit.
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402
from jsmpeg_b200.batch import OUT_DEVICE, BatchDecoder  # noqa: E402

out_path = sys.argv[1]
streams = int(sys.argv[2]) if len(sys.argv) > 2 else 64
pictures = int(sys.argv[3]) if len(sys.argv) > 3 else 60
bench.PICTURES = pictures
clips = bench.load_streams([1234 + i for i in range(8)])
bd = BatchDecoder(streams, max_slots=streams * pictures + 8)
for i in range(streams):
    bd.write(i, clips[i % len(clips)])
bd.upload()
torch.cuda.init()
bd.rewind()
bd.decode(pictures, OUT_DEVICE)  # warm-up
bd.rewind()
bd.reset_stats()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    n = bd.decode(pictures, OUT_DEVICE)
    torch.cuda.synchronize()
st = bd.stats()
kernels = {}
for e in prof.key_averages():
    t = getattr(e, "device_time_total", None)
    if t is None:
        t = getattr(e, "cuda_time_total", 0)
    if t > 0 and e.count > 0:
        kernels[e.key] = {"launches": e.count, "ms": t / 1e3}
spans = {}  # kernel name -> [first start, last end] in us
for ev in prof.events():
    if ev.device_type == torch.autograd.DeviceType.CUDA and ev.name in kernels:
        lo, hi = spans.setdefault(ev.name, [ev.time_range.start, ev.time_range.end])
        spans[ev.name] = [min(lo, ev.time_range.start), max(hi, ev.time_range.end)]
t0 = min(lo for lo, _ in spans.values()) if spans else 0
for k, (lo, hi) in spans.items():
    kernels[k]["first_start_ms"] = (lo - t0) / 1e3
    kernels[k]["last_end_ms"] = (hi - t0) / 1e3
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
res = {"card": card, "streams": streams, "pictures": n, "parse_ms": st["parse_ms"], "walk_ms": st["walk_ms"],
       "recon_ms": st["recon_ms"], "kernels": dict(sorted(kernels.items(), key=lambda kv: -kv[1]["ms"]))}
with open(out_path, "w") as f:
    json.dump(res, f, indent=1)
for k, v in res["kernels"].items():
    print(f"{v['ms']:9.2f} ms {v['launches']:5d} x  [{v.get('first_start_ms', 0):7.2f} .. {v.get('last_end_ms', 0):7.2f} ms]  {k[:90]}")
print(card)
