"""The accumulated map of decode_accumulated WITHOUT a GPU: the serial model (tools/accumulate_model.py) tied to the
oracle's records, residuals and pixels -- key pictures, P pictures right after their key picture, and on full-sample
streams the traced samples reproduce the decoded pictures exactly wherever the trace meets no clamping; the kernel's
block code (accumulate_block, jsmpeg_b200/csrc/accumulate.cuh) built with g++, plain and under AddressSanitizer,
against the model on random records and maps; and the kernel's recorded SASS hash."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import accumulate_model
import helpers
import macroblock_model
from test_macroblock_index import GOLDEN, MINI_ENC, corpus_stream
from test_residual_export import sample_mask

MBF_PRESENT, MBF_INTRA, MBF_SKIPPED = macroblock_model.MBF_PRESENT, macroblock_model.MBF_INTRA, macroblock_model.MBF_SKIPPED


def sequential_maps(es):
    """[(info, records, coefficient plane, planes, map, map of the previous reference picture or None, type of that
    picture)] of every I and P picture the oracle (B pictures off) decodes from `es`, the maps folded along the way.
    (A key picture's map depends on nothing before it, so this fold gives every chain's maps.)"""
    got, mbw, mbh = accumulate_model.oracle_decode(helpers.oracle_lib(), es)
    out, prev, prev_type = [], None, None
    for _, info, rec, coef, planes in got:
        if info.status != 1 or info.picture_type not in (1, 2):
            continue
        m = accumulate_model.depth(prev, rec, coef, mbw, mbh)
        out.append((info, rec, coef, planes, m, prev, prev_type))
        prev, prev_type = m, info.picture_type
    return out, mbw, mbh


def plane_geometry(mbw, mbh):
    """per plane (offset, stride, size)"""
    n = mbw * mbh * 256
    return [(0, mbw * 16, n), (n, mbw * 8, n // 4), (n + n // 4, mbw * 8, n // 4)]


@pytest.mark.parametrize("name", GOLDEN + ["ffmpeg_320x240", "ffmpeg_1280x720"] + sorted(MINI_ENC))
def test_key_pictures_and_first_p_pictures_follow_the_records(name):
    """A key picture's map is back 0 with zero motion and residual wherever its macroblocks are PRESENT, untraced
    elsewhere.  A P picture right after its key picture: back 1 and the exported vector (halved, truncated, for chroma)
    with the picture's own residual where it is predicted from inside the plane, back 0 where intra."""
    seen = set()
    maps, mbw, mbh = sequential_maps(corpus_stream(name))
    for info, rec, coef, _, m, _, prev_type in maps:
        r = np.frombuffer(rec.tobytes(), macroblock_model.RECORD)
        present = sample_mask((r["flags"] & MBF_PRESENT) != 0, mbw, mbh)
        intra = sample_mask((r["flags"] & (MBF_PRESENT | MBF_INTRA)) == (MBF_PRESENT | MBF_INTRA), mbw, mbh)
        if info.picture_type == 1:
            assert (m[present, 3] == 0).all() and (m[~present, 3] == -1).all() and not m[:, :3].any(), name
            seen.add(1)
            continue
        if prev_type != 1:
            continue
        assert (m[intra] == 0).all() and (m[~present, 3] == -1).all()
        res = macroblock_model.residuals(rec, coef, mbw, mbh)
        ent = np.frombuffer(macroblock_model.export(rec, 2).tobytes(), macroblock_model.ENTRY)
        for k, (off, stride, size) in enumerate(plane_geometry(mbw, mbh)):
            fx, fy = ent["fwd_x"].astype(np.int64), ent["fwd_y"].astype(np.int64)
            if k:
                fx, fy = np.fix(fx / 2).astype(np.int64), np.fix(fy / 2).astype(np.int64)
            vx = np.repeat(np.repeat(fx.reshape(mbh, mbw), 16 >> (k > 0), 0), 16 >> (k > 0), 1).reshape(-1)
            vy = np.repeat(np.repeat(fy.reshape(mbh, mbw), 16 >> (k > 0), 0), 16 >> (k > 0), 1).reshape(-1)
            pm = m[off:off + size]
            one = pm[:, 3] == 1
            assert np.array_equal(pm[one, 0], vx[one]) and np.array_equal(pm[one, 1], vy[one]), (name, k)
            assert np.array_equal(pm[one, 2], res[off:off + size][one]), (name, k)
            assert set(np.unique(pm[:, 3])) <= {-1, 0, 1}
        assert (m[:, 3] == 1).sum() > 0 or not (present & ~intra).any()
        seen.add(2)
    assert 1 in seen, name


FULL_SAMPLE = ["fcodes_fullpel", "mini_enc_fcodes_4_2_fullpel_fwd"]


@pytest.mark.parametrize("name", FULL_SAMPLE)
def test_full_sample_traces_give_the_decoded_samples(name):
    """Every sample with back >= 1 whose trace takes full-sample steps and meets no clamping on its way (checked by
    walking the trace through the oracle's own pictures): picture k's sample = the sample of the picture `back`
    references earlier at x + d / 2, plus the accumulated residual -- exactly."""
    maps, mbw, mbh = sequential_maps(corpus_stream(name))
    checked = 0
    for n, (info, _, _, planes, m, _, _) in enumerate(maps):
        if info.picture_type != 2:
            continue
        for off, stride, size in plane_geometry(mbw, mbh):
            pm = m[off:off + size].astype(np.int64)
            idx = np.nonzero(pm[:, 3] >= 1)[0]
            back = pm[idx, 3]
            ok = np.ones(len(idx), bool)
            at = idx.copy()
            depth = np.zeros(len(idx), np.int64)
            for _ in range(int(back.max()) if len(idx) else 0):  # walk every trace one reference back at a time
                live = depth < back
                j = n - depth  # the picture whose sample `at` the trace is on
                nxt = at.copy()
                for pic in np.unique(j[live]):
                    sel = live & (j == pic)
                    cur_map = maps[pic][4][off:off + size].astype(np.int64)
                    prev_map = maps[pic - 1][4][off:off + size].astype(np.int64)
                    # one step: the sample's own vector in picture `pic`, its tap in the picture before
                    a = at[sel]
                    rec = maps[pic][1]
                    r = np.frombuffer(rec.tobytes(), macroblock_model.RECORD)
                    px = 16 if stride == mbw * 16 else 8
                    mb = (a // stride) // px * mbw + (a % stride) // px
                    vx, vy = r["mv_h"][mb].astype(np.int64), r["mv_v"][mb].astype(np.int64)
                    if px == 8:
                        vx, vy = np.fix(vx / 2).astype(np.int64), np.fix(vy / 2).astype(np.int64)
                    even = ((vx & 1) == 0) & ((vy & 1) == 0)
                    t = a + (vy >> 1) * stride + (vx >> 1)
                    t = np.clip(t, 0, size - 1)
                    res = macroblock_model.residuals(rec, maps[pic][2], mbw, mbh)[off:off + size].astype(np.int64)
                    here = maps[pic][3][off:off + size].astype(np.int64)
                    before = maps[pic - 1][3][off:off + size].astype(np.int64)
                    unclamped = here[a] == before[t] + res[a]
                    assert (prev_map[t, 3] == cur_map[a, 3] - 1).all()
                    ok[sel] &= even & unclamped
                    nxt[sel] = t
                at = np.where(live, nxt, at)
                depth += live
            k_samples = planes[off:off + size].astype(np.int64)[idx]
            src_pic = n - back
            end = np.clip(idx + (pm[idx, 1] // 2) * stride + pm[idx, 0] // 2, 0, size - 1)
            got = np.array([maps[p][3][off:off + size][i] for p, i in zip(src_pic, end)], np.int64)
            want = np.clip(got + pm[idx, 2], 0, 255)
            assert np.array_equal(k_samples[ok], want[ok]), (name, n)
            assert np.array_equal(at[ok], end[ok])
            checked += int(ok.sum())
    assert checked > 20000, (name, checked)


# ---- the kernel's block code compiled for the host ----------------------------------------------------------------

def host_build(tmp_path, asan):
    if not shutil.which("g++"):
        pytest.skip("g++ not available")
    inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(inc, "cuda_runtime.h")):
        pytest.skip("CUDA headers not available")
    exe = tmp_path / ("accumulate_check_asan" if asan else "accumulate_check")
    flags = ["-g", "-fsanitize=address", "-fno-omit-frame-pointer"] if asan else []
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", "-Wno-unknown-pragmas", *flags, "-I", inc, "-o",
                        str(exe), os.path.join(helpers.ROOT, "tests", "emu", "accumulate_check.cpp")],
                       capture_output=True, text=True)
    if asan and r.returncode != 0 and "asan" in r.stderr.lower():
        pytest.skip("AddressSanitizer not available")
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def random_case(rng, mbw, mbh, with_prev):
    """Records with absent, intra, skipped (zero and nonzero vector) and predicted macroblocks; vectors from small
    half-sample ones to ones far outside the plane (row-end wrap of the flat index included); a residual and a previous
    map of any int16 values, traced and untraced (back up to 32,766), so that sums saturate"""
    mb = mbw * mbh
    rec = np.zeros(mb, macroblock_model.RECORD)
    kind = rng.integers(0, 6, mb)
    rec["flags"] = np.choose(kind, [0, MBF_PRESENT | MBF_INTRA, MBF_PRESENT | MBF_SKIPPED, MBF_PRESENT, MBF_PRESENT,
                                    MBF_PRESENT | MBF_SKIPPED])
    small = rng.integers(-9, 10, (mb, 2))
    wide = rng.integers(-mbw * 40, mbw * 40, (mb, 2))
    huge = rng.integers(-32768, 32768, (mb, 2))
    pick = rng.integers(0, 10, mb)
    v = np.where((pick < 6)[:, None], small, np.where((pick < 9)[:, None], wide, huge))
    v[kind == 5] = 0  # skipped with a zero vector
    rec["mv_h"], rec["mv_v"] = v[:, 0], v[:, 1]
    rec["cbp"] = rng.integers(0, 64, mb)
    n = mb * 384
    res = rng.integers(-32768, 32768, n).astype(np.int16)
    res[rng.random(n) < 0.5] = rng.integers(-300, 300, 1)[0]
    prev = None
    if with_prev:
        prev = rng.integers(-32768, 32768, (n, 4)).astype(np.int16)
        prev[:, 3] = rng.integers(-1, 32767, n)
        prev[rng.random(n) < 0.3, 3] = -1
    return rec, res, prev


def run_host(exe, tmp_path, rec, res, prev, mbw, mbh):
    path = tmp_path / "case.bin"
    head = np.array([mbw, mbh, prev is not None], np.int32)
    path.write_bytes(head.tobytes() + rec.tobytes() + res.tobytes() + (prev.tobytes() if prev is not None else b""))
    out = subprocess.run([str(exe), str(path)], capture_output=True)
    assert out.returncode == 0, out.stderr.decode(errors="replace")[-3000:]
    return np.frombuffer(out.stdout, np.int16).reshape(-1, 4)


@pytest.mark.parametrize("asan", [False, True])
def test_the_block_code_compiled_for_the_host_equals_the_model(tmp_path, asan):
    exe = host_build(tmp_path, asan)
    rng = np.random.default_rng(21 + asan)
    kinds = set()
    for trial, (mbw, mbh) in enumerate([(1, 1), (2, 3), (5, 4), (11, 7), (3, 9)] * 2):
        rec, res, prev = random_case(rng, mbw, mbh, trial % 5 != 0)
        got = run_host(exe, tmp_path, rec, res, prev, mbw, mbh)
        want = accumulate_model.step(prev, rec, res, mbw, mbh)
        assert np.array_equal(got, want), (mbw, mbh, trial)
        kinds |= set(np.unique(want[:, 3] >= 1).tolist())
        if prev is not None:
            assert ((want[:, :3] == 32767) | (want[:, :3] == -32768)).any()  # some sums saturate
    assert kinds == {False, True}


def test_the_accumulate_kernel_is_the_measured_one():
    """profiles/sass_hashes_sm90a.txt records the accumulate kernel's SASS md5 (tools/sass_hash.py); recompiling
    accumulate.cu must give the same machine code."""
    if not (shutil.which("nvcc") and shutil.which("cuobjdump")):
        pytest.skip("nvcc / cuobjdump not available")
    sys.path.insert(0, os.path.join(helpers.ROOT, "tools"))
    import sass_hash
    line = next(x for x in open(os.path.join(helpers.ROOT, "profiles", "sass_hashes_sm90a.txt"))
                if "accumulate.cu" in x and "accumulate_kernel" in x)
    recorded = next(p for p in line.split() if len(p) == 32)
    now = {sass_hash.demangle(k): md5 for k, (md5, _) in sass_hash.kernel_hashes("accumulate.cu").items()}
    assert now == {"accumulate_kernel": recorded}
