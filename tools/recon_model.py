"""Plain model of stage 2 (jsmpeg_b200/csrc/recon.cuh): the planes a picture's macroblock records and coefficient blocks
make from its reference planes, stated from the rules of SURVEY Q9 / Q11 and DESIGN 3.2 / 3.4 over the whole
motion-vector domain.

Planes are flat uint8 arrays Y | Cr | Cb (coded_size * 3 // 2), records mb_record_t (macroblock_model.RECORD, or any
16-byte-per-record buffer), coefficients int16 [mb_size * 6 * 64], each block in raster order.
  * a macroblock that is not PRESENT keeps what the written plane set held;
  * an intra block is its residual, saturated;
  * a predicted block is its prediction plus its residual, saturated;
  * the residual of a coded block is the reference's integer inverse transform of the premultiplied block, or for a
    dc_only block (c0 * 32 + 128) >> 8 in every sample; an intra block's c0 is its dc (the records' clamped one,
    jsmpeg_b200/csrc/records.h) and is premultiplied by 256 instead, so its dc_only block is c0 itself; an uncoded
    block's residual is 0;
  * prediction addresses by flat index: the block's first tap is origin + (v >> 1) * stride + (h >> 1), so a tap past a
    row's end is the next row's first sample; the half-sample flags h & 1, v & 1 choose the copy, (a + b + 1) >> 1
    horizontally or vertically, or (a + b + c + d + 2) >> 2;
  * chroma vectors are the luma ones divided by 2, truncated toward zero;
  * any tap outside its plane zeroes that sample of that direction's prediction (the JS rule: the tap reads
    `undefined`, the sum becomes NaN, the stored sample 0; the residual is added to that 0);
  * B pictures: the forward and the backward prediction each on its own, then (f + b + 1) >> 1 where both are used;
    a record with neither direction predicts forward.
"""
from __future__ import annotations

from collections import Counter

import numpy as np

import macroblock_model as mm
from accumulate_model import inside  # stage 2's choice of path: PREDICTION_INSIDE

MBF_PRESENT, MBF_INTRA, MBF_MOTION_BWD, MBF_MOTION_FWD = mm.MBF_PRESENT, mm.MBF_INTRA, mm.MBF_MOTION_BWD, mm.MBF_MOTION_FWD


def halve(v):
    """A chroma vector component: the luma one divided by 2, truncated toward zero (not v >> 1)"""
    v = np.asarray(v, np.int64)
    return np.where(v < 0, -((-v) // 2), v // 2)


def idct(blocks):
    """The reference's 2-D inverse transform of premultiplied blocks (int [..., 64], raster order), in int64"""
    return mm.idct(np.asarray(blocks, np.int64))


def planes_layout(mb_width, mb_height):
    """[(name, offset, stride, rows, px)] of Y, Cr, Cb in the flat layout; px = samples per macroblock side"""
    ysize = mb_width * mb_height * 256
    return [("Y", 0, mb_width * 16, mb_height * 16, 16), ("Cr", ysize, mb_width * 8, mb_height * 8, 8),
            ("Cb", ysize + ysize // 4, mb_width * 8, mb_height * 8, 8)]


def _records(records):
    return np.frombuffer(np.ascontiguousarray(records).tobytes(), mm.RECORD)


def _per_sample(x, px):
    """per-macroblock values [mb_height, mb_width] -> per-sample [rows, stride] of a plane of px x px macroblocks"""
    return np.repeat(np.repeat(x, px, 0), px, 1)


def predict(ref, stride, rows, h, v):
    """One direction's prediction of a whole plane of `rows` x `stride` samples from `ref` (flat, that plane alone), with
    per-sample vector components h, v (half-pel units of this plane): int64 per sample, 0 where a tap is outside."""
    size = stride * rows
    y, x = np.mgrid[0:rows, 0:stride]
    oh, ov = (h & 1).astype(bool), (v & 1).astype(bool)
    a = y * stride + x + (v >> 1) * stride + (h >> 1)
    taps = [(a, np.ones_like(oh)), (a + 1, oh), (a + stride, ov), (a + stride + 1, oh & ov)]
    out = np.zeros(a.shape, bool)
    val = []
    for t, used in taps:
        outside = (t < 0) | (t >= size)
        out |= used & outside
        val.append(ref[np.clip(t, 0, size - 1)].astype(np.int64))
    A, B, C, D = val
    p = np.where(oh & ov, (A + B + C + D + 2) >> 2, np.where(oh, (A + B + 1) >> 1, np.where(ov, (A + C + 1) >> 1, A)))
    return np.where(out, 0, p)


def residual_planes(records, coef, mb_width, mb_height):
    """int64 residual of every sample (flat Y | Cr | Cb): coded blocks only, dc_only blocks by the shortcut"""
    r = _records(records)
    c = np.asarray(coef, np.int64).reshape(len(r), 6, 64)
    bits = 0x20 >> np.arange(6)
    coded = (((r["flags"] & MBF_PRESENT) != 0)[:, None] & ((r["cbp"][:, None] & bits) != 0))
    dc_only = coded & ((r["dc_only"][:, None] & bits) != 0)
    pc = c * mm.PREMULTIPLIER
    pc[:, :, 0] = np.where(((r["flags"] & MBF_INTRA) != 0)[:, None], c[:, :, 0] * 256, pc[:, :, 0])
    px = idct(pc)
    px = np.where(dc_only[:, :, None], ((pc[:, :, :1] + 128) >> 8), px)
    px = np.where(coded[:, :, None], px, 0).reshape(mb_height, mb_width, 6, 8, 8)
    y = px[:, :, :4].reshape(mb_height, mb_width, 2, 2, 8, 8).transpose(0, 2, 4, 1, 3, 5).reshape(-1)
    cb = px[:, :, 4].transpose(0, 2, 1, 3).reshape(-1)  # block 4 -> Cb, the third plane
    cr = px[:, :, 5].transpose(0, 2, 1, 3).reshape(-1)  # block 5 -> Cr, the second
    return np.concatenate([y, cr, cb])


def reconstruct(records, coef, fwd, cur, mb_width, mb_height, bwd=None):
    """The planes stage 2 writes (flat uint8 Y | Cr | Cb): `cur` is what the written set held, `fwd` the forward
    reference, `bwd` the backward one of a B picture (None: an I or P picture)"""
    r = _records(records)
    shape = (mb_height, mb_width)
    flags = r["flags"].astype(np.int64).reshape(shape)
    fh, fv = r["mv_h"].astype(np.int64).reshape(shape), r["mv_v"].astype(np.int64).reshape(shape)
    bh, bv = r["bwd_x"].astype(np.int64).reshape(shape), r["bwd_y"].astype(np.int64).reshape(shape)
    present = (flags & MBF_PRESENT) != 0
    intra = (flags & MBF_INTRA) != 0
    use_b = (flags & MBF_MOTION_BWD) != 0 if bwd is not None else np.zeros(shape, bool)
    use_f = ~use_b | ((flags & MBF_MOTION_FWD) != 0)
    res = residual_planes(records, coef, mb_width, mb_height)
    fwd, cur = np.asarray(fwd), np.asarray(cur)
    out = np.array(cur, np.uint8, copy=True)
    for _, off, stride, rows, px in planes_layout(mb_width, mb_height):
        size = stride * rows
        sl = slice(off, off + size)
        h, v = (fh, fv) if px == 16 else (halve(fh), halve(fv))
        pred = predict(fwd[sl], stride, rows, _per_sample(h, px), _per_sample(v, px))
        if bwd is not None:
            h2, v2 = (bh, bv) if px == 16 else (halve(bh), halve(bv))
            pb = predict(np.asarray(bwd)[sl], stride, rows, _per_sample(h2, px), _per_sample(v2, px))
            f_s, b_s = _per_sample(use_f, px), _per_sample(use_b, px)
            pred = np.where(f_s & b_s, (pred + pb + 1) >> 1, np.where(b_s, pb, pred))
        s_intra = _per_sample(intra, px).reshape(-1)
        s_present = _per_sample(present, px).reshape(-1)
        val = np.where(s_intra, 0, pred.reshape(-1)) + res[sl]
        out[sl] = np.where(s_present, np.clip(val, 0, 255), cur[sl]).astype(np.uint8)
    return out


def categories(records, mb_width, mb_height, picture_type):
    """Counter of the vector-domain categories the predicted blocks of a picture's records fall in (one count per
    block and direction): "wrap" (the 2-D footprint crosses the left or right edge, every flat-index tap inside),
    "one_row_out" (some sample zeroed, at most one row or column of them: a near miss), "far_out" (all 64 samples
    zeroed), "partly_out" (the rest that leave the plane), "chroma_only_out" (per macroblock and direction: the four luma
    blocks inside, a chroma block not), "large" (a component of more than 64 samples), "parity_hv" (the luma half-sample
    flags), "neg_odd" (a negative odd component) and "neg_odd_edge" (a chroma block that is inside by the truncating
    halving and would not be by v >> 1, or the other way round)."""
    r = _records(records)
    flags = r["flags"].astype(np.int64)
    predicted = ((flags & MBF_PRESENT) != 0) & ((flags & MBF_INTRA) == 0)
    dirs = [("f", r["mv_h"], r["mv_v"], predicted & ((picture_type != 3) | ((flags & MBF_MOTION_FWD) != 0) |
                                                     ((flags & MBF_MOTION_BWD) == 0)))]
    if picture_type == 3:
        dirs.append(("b", r["bwd_x"], r["bwd_y"], predicted & ((flags & MBF_MOTION_BWD) != 0)))
    cw, ch = mb_width * 16, mb_height * 16
    out = Counter()
    for _, vh, vv, used in dirs:
        for mb in np.nonzero(used)[0]:
            row, col = divmod(int(mb), mb_width)
            h, v = int(vh[mb]), int(vv[mb])
            out["large"] += max(abs(h), abs(v)) > 128
            out[f"parity_{h & 1}{v & 1}"] += 1
            out["neg_odd"] += (h < 0 and h & 1) or (v < 0 and v & 1)
            luma_in, chroma_in = True, True
            for b in range(6):
                if b < 4:
                    stride, size, px, bh, bv = cw, cw * ch, 16, h, v
                    oy, ox = row * 16 + (b >> 1) * 8, col * 16 + (b & 1) * 8
                else:
                    stride, size, px, bh, bv = cw // 2, cw * ch // 4, 8, int(halve(h)), int(halve(v))
                    oy, ox = row * 8, col * 8
                    floor_in = inside(oy * stride + ox + ((v >> 1) >> 1) * stride + ((h >> 1) >> 1), stride, size,
                                      (h >> 1) & 1, (v >> 1) & 1)
                src = oy * stride + ox + (bv >> 1) * stride + (bh >> 1)
                ok = bool(inside(src, stride, size, bh & 1, bv & 1))
                if b >= 4 and ((h < 0 and h & 1) or (v < 0 and v & 1)) and bool(floor_in) != ok:
                    out["neg_odd_edge"] += 1
                x0, x1 = ox + (bh >> 1), ox + (bh >> 1) + 8 + (bh & 1)
                if ok:
                    out["wrap"] += x0 < 0 or x1 > stride
                    continue
                luma_in &= b >= 4
                chroma_in &= b < 4
                y, x = np.mgrid[0:8, 0:8]
                a = src + y * stride + x
                taps = [a, a + (bh & 1), a + (bv & 1) * stride, a + (bh & 1) + (bv & 1) * stride]
                zeroed = np.zeros((8, 8), bool)
                for t in taps:
                    zeroed |= (t < 0) | (t >= size)
                n = int(zeroed.sum())
                one_line = zeroed.any(1).sum() <= 1 or zeroed.any(0).sum() <= 1
                out["far_out" if n == 64 else ("one_row_out" if one_line else "partly_out")] += 1
            out["chroma_only_out"] += luma_in and not chroma_in
    return out
