#!/usr/bin/env python
"""GPU helper: the B-picture extension on a wave of I/P/B streams -- device time per stage, frames/s, and a
check of every stream's last picture against the oracle.

    python tools/time_b.py [streams] [reps]        (tests/fixtures/b_clip_1280x720.m1v, tools/mini_enc.py)
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402

import helpers  # noqa: E402
from jsmpeg_b200.batch import OUT_DEVICE, BatchDecoder  # noqa: E402

streams = int(sys.argv[1]) if len(sys.argv) > 1 else 64
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 4
es = open(os.path.join(ROOT, "tests", "fixtures", "b_clip_1280x720.m1v"), "rb").read()
types = []
i = 0
while True:
    i = es.find(b"\x00\x00\x01\x00", i)
    if i < 0:
        break
    types.append((es[i + 5] >> 3) & 7)
    i += 4
pictures = len(types)

olib = helpers.oracle_lib()
olib.oracle_set_decode_b(1)
want, _, od = helpers.decode_all(olib, [(0, es)])
olib.oracle_set_decode_b(0)

out = {"workload": f"{streams} x 1280x720 I/P/B ({types.count(1)} I, {types.count(2)} P, {types.count(3)} B per stream), ES resident",
       "runs": []}
quick = os.environ.get("TIME_B_QUICK") == "1"  # under ncu: the extension's run only, one repetition, no file
if quick:
    reps = 1
for decode_b, slice_walk in (((1, 0),) if quick else ((1, 0), (0, 0), (1, 1))):  # (1, 1): I/P pictures on the slice walk
    bd = BatchDecoder(streams, max_slots=streams * pictures + 8, decode_b=decode_b, slice_walk=slice_walk)
    for s in range(streams):
        bd.write(s, es)
    bd.upload()
    for rep in range(reps):
        bd.rewind()
        bd.reset_stats()
        t0 = time.perf_counter()
        n = bd.decode(pictures, OUT_DEVICE)
        dt = time.perf_counter() - t0
        st = bd.stats()
        run = dict(decode_b=decode_b, slice_walk=slice_walk, rep=rep, pictures=n, decoded=st["pictures_decoded"], wall_ms=round(dt * 1e3, 3),
                   parse_ms=round(st["parse_ms"], 3), walk_ms=round(st["walk_ms"], 3), recon_ms=round(st["recon_ms"], 3),
                   frames_per_s=round(st["pictures_decoded"] / dt), launches=st["kernel_launches"],
                   recon_GBps=round(st["algorithmic_bytes"] / max(st["recon_ms"], 1e-9) / 1e6, 1), errors=st["parse_errors"])
        out["runs"].append(run)
        print(run, flush=True)
    if decode_b:
        ok = all(all(np.array_equal(a, b) for a, b in zip(bd.read_planes(s), want[-1])) for s in range(streams))
        key = "verified_last_picture_of_every_stream" + ("_slice_walk" if slice_walk else "")
        out[key] = bool(ok)
        print(key, ok, flush=True)
    bd.close()
if quick:
    sys.exit(0)
with open(os.environ.get("TIME_B_OUT", "time_b.json"), "w") as f:
    json.dump(out, f, indent=1)
sys.exit(0 if out.get("verified_last_picture_of_every_stream") and out.get("verified_last_picture_of_every_stream_slice_walk", True) else 1)
