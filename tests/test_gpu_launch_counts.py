"""How many kernels decode(), decode_pictures, decode_intra and decode_macroblocks launch on a fixed mixed workload.
The host routes each picture to a walk kernel and each reconstruct task to a kernel, and cuts each kernel's work into
launches; this pins the result, per call, both as the decoder's stats count it and per kernel as torch.profiler sees it.

The workload: one-slice 320x240 I/P clips and the row-sliced 1280x720 I/P/B clip, with decode_b and slice_walk on, so
that a wave holds lane-walk, slice-walk and B-walk pictures.  It has plain and RGBA outputs, steps of more tasks than
one reconstruct launch holds (80 plain, 60 RGBA), and waves of more than 64 x 8 lane-walk pictures, which stage 1 forks
into 8 size groups.  The expected numbers were taken on an H100 from the code as it was before stage 1 and stage 2
each got one host launcher."""
import os
import re
from collections import Counter

import pytest

import helpers
from jsmpeg_b200.batch import OUT_DEVICE, OUT_RGBA, BatchDecoder

pytestmark = pytest.mark.gpu

FIXTURE_720P = os.path.join(helpers.ROOT, "tests", "fixtures", "b_clip_1280x720.m1v")
N_SMALL, N_720P = 100, 4

EXPECTED = [
    ("decode plain", 36, 6, {"scan_start_codes_kernel": 1, "walk_pictures_lanes_kernel": 8, "walk_pictures_slices_kernel": 1,
                             "walk_pictures_b_kernel": 1, "expand_blocks_kernel": 10, "reconstruct_kernel": 12,
                             "reconstruct_b_kernel": 3}),
    ("decode rgba", 72, 12, {"walk_pictures_lanes_kernel": 8, "walk_pictures_slices_kernel": 1, "walk_pictures_b_kernel": 1,
                             "expand_blocks_kernel": 10, "reconstruct_rgba_kernel": 12, "reconstruct_rgba_b_kernel": 4}),
    # (decode_pictures, decode_intra and decode_macroblocks leave kernel_launches and recon_launches to decode())
    ("decode_pictures plain", 72, 12, {"walk_pictures_lanes_kernel": 8, "walk_pictures_slices_kernel": 1,
                                       "walk_pictures_b_kernel": 2, "expand_blocks_kernel": 11, "reconstruct_kernel": 22,
                                       "reconstruct_b_kernel": 8}),
    ("decode_pictures rgba", 72, 12, {"walk_pictures_lanes_kernel": 8, "walk_pictures_slices_kernel": 1,
                                      "walk_pictures_b_kernel": 2, "expand_blocks_kernel": 11, "reconstruct_kernel": 1,
                                      "reconstruct_rgba_kernel": 22, "reconstruct_rgba_b_kernel": 8}),
    ("decode_intra rgba", 72, 12, {"walk_pictures_lanes_kernel": 1, "walk_pictures_slices_kernel": 1,
                                   "expand_blocks_kernel": 2, "reconstruct_rgba_kernel": 2}),
    ("decode_macroblocks", 72, 12, {"walk_pictures_lanes_kernel": 1, "walk_pictures_slices_kernel": 1,
                                    "walk_pictures_b_kernel": 1, "export_macroblocks_kernel": 1}),
]


def workload():
    """[(call, kernel_launches, recon_launches, {kernel: launches in the call})] after each call of the workload, the
    stats counted from a reset after the writes."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    small = b"".join(p for _, p in helpers.clip_packets(320, 240, 12))
    big = open(FIXTURE_720P, "rb").read()
    bd = BatchDecoder(N_SMALL + N_720P, max_slots=1200, decode_b=1, slice_walk=1)
    seen = []

    def call(name, fn, *args, **kw):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn(*args, **kw)
            torch.cuda.synchronize()
        kernels = Counter()
        for ev in prof.events():
            m = re.search(r"(\w+_kernel)\(", ev.name)
            if ev.device_type == torch.autograd.DeviceType.CUDA and m:
                kernels[m.group(1)] += 1
        st = bd.stats()
        seen.append((name, st["kernel_launches"], st["recon_launches"], dict(kernels)))

    try:
        for s in range(N_SMALL):
            bd.write(s, small)
        for s in range(N_720P):
            bd.write(N_SMALL + s, big)
        bd.reset_stats()
        call("decode plain", bd.decode, 6, OUT_DEVICE)
        call("decode rgba", bd.decode, 6, OUT_RGBA)
        streams = range(N_SMALL + N_720P)
        pictures = [(s, e["picture"]) for s in streams for e in bd.picture_index(s)]
        call("decode_pictures plain", bd.decode_pictures, pictures)
        call("decode_pictures rgba", bd.decode_pictures, pictures, rgba=True)
        call("decode_intra rgba", bd.decode_intra, [(s, e["picture"]) for s in streams for e in bd.intra_index(s)], rgba=True)
        call("decode_macroblocks", bd.decode_macroblocks,
             [(s, e["picture"]) for s in streams for e in bd.macroblock_index(s)])
        return seen
    finally:
        bd.close()


def test_launch_counts_of_a_mixed_workload():
    assert workload() == EXPECTED
