#!/usr/bin/env python
"""GPU helper: per-stage device time of the batch decode on a bench-like workload.

    python tools/time_stages.py [streams] [pictures] [reps]

parse (the tasks' upload to the end of the last expand) and recon (around the reconstruct launches) overlap.  Before each
line the library prints where the host's time of the call went (JSMPEG_B200_HOST_TRACE: upload_all, planning, building
and queueing stage 1, the wait for the infos, their consumption, queueing stage 2, the closing synchronises) and
`device`, the span from the tasks' upload to the end of the later of expand and reconstruction; step - scan - device is
what no device event covers.
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
os.environ.setdefault("JSMPEG_B200_HOST_TRACE", "1")
import bench  # noqa: E402
from jsmpeg_b200.batch import OUT_DEVICE, BatchDecoder  # noqa: E402

streams = int(sys.argv[1]) if len(sys.argv) > 1 else 64
pictures = int(sys.argv[2]) if len(sys.argv) > 2 else 60
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
bench.PICTURES = pictures
distinct = int(os.environ.get("TIME_STAGES_DISTINCT", "8"))
clips = bench.load_streams([1234 + i for i in range(distinct)])
bd = BatchDecoder(streams, max_slots=streams * pictures + 8)
for i in range(streams):
    bd.write(i, clips[i % len(clips)])
bd.upload()
for rep in range(reps):
    bd.rewind()
    bd.reset_stats()
    t0 = time.perf_counter()
    n = bd.decode(pictures, OUT_DEVICE)
    dt = time.perf_counter() - t0
    st = bd.stats()
    print(f"streams={streams} pictures={n} step={dt * 1e3:8.2f} ms scan={st['scan_ms']:6.2f} parse={st['parse_ms']:8.2f} ms (walk {st['walk_ms']:.2f}) "
          f"recon={st['recon_ms']:7.2f} ms fps={n / dt:9.0f} coded_blocks/pic={st['coded_blocks'] / max(1, st['pictures_decoded']):.0f} "
          f"errors={st['parse_errors']} lane_walk={st['lane_walk_pictures']}", flush=True)
