"""Serial model of the macroblock index (jsmpeg_b200_batch_macroblock_index) and of what decode_macroblocks must give.

Picture k of a stream is the k-th picture start code (00 00 01 00) in its buffer.  The index lists picture k when
  1. it starts at or after the end of the stream's first sequence header,
  2. it is closed (tools/intra_model.py), and
  3. the walks decode it with B pictures on: picture_coding_type 1; 2 with forward_f_code != 0; 3 with both f_codes
     != 0 (tools/chain_model.py: is_decoded) -- whatever the decode_b option says, and with no chain start.
A listed picture's entries are export() of the records a fresh decoder with B pictures on gives for fresh_bytes(): the
first sequence header, the picture's bytes up to its closing code, and the closing code itself.  decode_coefficients
lists the same pictures; its coefficients are coefficients() of the same decoder's records and coefficient plane, and
decode_residuals' residuals are residuals() of them.
"""
from __future__ import annotations

import numpy as np

import chain_model
import intra_model

# jsmpeg_b200_macroblock_t flags (include/jsmpeg_b200.h) and mb_record_t flags (jsmpeg_b200/csrc/records.h)
MB_PRESENT, MB_INTRA, MB_SKIPPED, MB_BACKWARD, MB_FORWARD = 0x01, 0x02, 0x04, 0x08, 0x10
MBF_PRESENT, MBF_INTRA, MBF_SKIPPED, MBF_MOTION_BWD, MBF_MOTION_FWD = 0x01, 0x02, 0x04, 0x08, 0x10

RECORD = np.dtype([("mv_h", "<i2"), ("mv_v", "<i2"), ("flags", "u1"), ("cbp", "u1"), ("dc_only", "u1"), ("qscale", "u1"),
                   ("bit_pos", "<u4"), ("bwd_x", "<i2"), ("bwd_y", "<i2")])  # mb_record_t, mv_bwd split into its halves
ENTRY = np.dtype([("fwd_x", "<i2"), ("fwd_y", "<i2"), ("bwd_x", "<i2"), ("bwd_y", "<i2"), ("flags", "u1"), ("cbp", "u1"),
                  ("qscale", "u1"), ("reserved", "u1", 5)])  # jsmpeg_b200_macroblock_t
assert RECORD.itemsize == ENTRY.itemsize == 16


def macroblock_index(es):
    """[{"picture", "byte_pos", "type", "temporal_reference", "close"}] of the pictures the index lists for `es`."""
    seq = intra_model.first_sequence_header(es)
    if seq is None:
        return []
    floor = (seq[1] + 7) >> 3
    codes = [p for p in intra_model.prefixes(es) if p + 3 < len(es)]
    out, k = [], -1
    for j, p in enumerate(codes):
        if es[p + 3] != 0:
            continue
        k += 1
        if p < floor or not chain_model.is_decoded(es, p, True):
            continue
        close = next((q for q in codes[j + 1:] if intra_model._closes(es[q + 3])), None)
        if close is not None:
            out.append({"picture": k, "byte_pos": p, "type": chain_model.picture_type(es, p),
                        "temporal_reference": chain_model.header_bits(es, p, 0, 10), "close": close})
    return out


def fresh_bytes(es, entry):
    """What a fresh decoder is fed for a listed picture: first sequence header + the picture + its closing code."""
    return intra_model.fresh_bytes(es, entry)


def export(records, picture_type):
    """The public entries (uint8 [n, 16]) of n mb_record_t (any 16-byte-per-record buffer) of a picture of
    picture_coding_type `picture_type` -- the rule of jsmpeg_b200/csrc/macroblocks.cuh."""
    r = np.frombuffer(np.ascontiguousarray(records).tobytes(), RECORD)
    present = (r["flags"] & MBF_PRESENT) != 0
    intra = (r["flags"] & MBF_INTRA) != 0
    if picture_type == 3:
        fwd = present & ~intra & ((r["flags"] & MBF_MOTION_FWD) != 0)
        bwd = present & ~intra & ((r["flags"] & MBF_MOTION_BWD) != 0)
    else:
        fwd = present & ~intra
        bwd = np.zeros_like(present)
    e = np.zeros(len(r), ENTRY)
    e["flags"] = np.where(present, MB_PRESENT, 0) | np.where(present & intra, MB_INTRA, 0) | \
        np.where(present & ((r["flags"] & MBF_SKIPPED) != 0), MB_SKIPPED, 0) | \
        np.where(fwd, MB_FORWARD, 0) | np.where(bwd, MB_BACKWARD, 0)
    e["fwd_x"] = np.where(fwd, r["mv_h"], 0)
    e["fwd_y"] = np.where(fwd, r["mv_v"], 0)
    e["bwd_x"] = np.where(bwd, r["bwd_x"], 0)
    e["bwd_y"] = np.where(bwd, r["bwd_y"], 0)
    e["cbp"] = np.where(present, r["cbp"], 0)
    e["qscale"] = np.where(present, r["qscale"], 0)
    return e.view(np.uint8).reshape(len(r), 16)


def coefficients(records, coef):
    """What decode_coefficients gives (int16 [n, 6, 64], each block in raster order) for n mb_record_t (any 16-byte-
    per-record buffer) and the int16 coefficient plane of the same picture ([n * 6 * 64] values in the oracle's layout,
    which is the public one): the plane, with every value 0 where the macroblock is not PRESENT or the block's cbp bit
    (bit 5 - block) is clear."""
    r = np.frombuffer(np.ascontiguousarray(records).tobytes(), RECORD)
    c = np.frombuffer(np.ascontiguousarray(coef).tobytes(), np.int16).reshape(len(r), 6, 64)
    coded = ((r["flags"] & MBF_PRESENT) != 0)[:, None] & ((r["cbp"][:, None] >> (5 - np.arange(6))) & 1).astype(bool)
    return np.where(coded[:, :, None], c, np.int16(0)).astype(np.int16)


# PREMULTIPLIER_MATRIX (src/mpeg1.js:1026-1035), raster order
PREMULTIPLIER = np.array([
    32, 44, 42, 38, 32, 25, 17, 9, 44, 62, 58, 52, 44, 35, 24, 12, 42, 58, 55, 49, 42, 33, 23, 12,
    38, 52, 49, 44, 38, 30, 20, 10, 32, 44, 42, 38, 32, 25, 17, 9, 25, 35, 33, 30, 25, 20, 14, 7,
    17, 24, 23, 20, 17, 14, 9, 5, 9, 12, 12, 10, 9, 7, 5, 2], np.int64)


def round8(z):
    """(z + 128) >> 8, the transform's one rounding step (an arithmetic shift: floor).  Anything with a `round8`
    method (tests/test_residual_export.py's bound arithmetic) brings its own."""
    return z.round8() if hasattr(z, "round8") else (z + 128) >> 8


def idct8(x, row):
    """One 8-point pass of the reference IDCT (src/mpeg1.js:916-983, oracle/mpeg1_oracle.c idct_pass) on the eight
    sequences x[0..7] (numpy arrays or anything with + - * and round8): the eight outputs, each rounded with round8 in
    the row pass."""
    b1 = x[4]
    b3 = x[2] + x[6]
    b4 = x[5] - x[3]
    t1 = x[1] + x[7]
    t2 = x[3] + x[5]
    b6 = x[1] - x[7]
    b7 = t1 + t2
    m0 = x[0]
    x4 = round8(b6 * 473 - b4 * 196) - b7
    x0 = x4 - round8((t1 - t2) * 362)
    x1 = m0 - b1
    x2 = round8((x[2] - x[6]) * 362) - b3
    x3 = m0 + b1
    y3, y4, y5, y6 = x1 + x2, x3 + b3, x1 - x2, x3 - b3
    y7 = -x0 - round8(b4 * 473 + b6 * 196)
    o = [b7 + y4, x4 + y3, y5 - x0, y6 - y7, y6 + y7, x0 + y5, y3 - x4, y4 - b7]
    return [round8(v) for v in o] if row else o


def idct(blocks):
    """The reference's 2-D transform (oracle_idct) of premultiplied blocks, int [..., 64] in raster order, all at once:
    the column passes, then the row passes.  int64 [..., 64]."""
    v = np.asarray(blocks, np.int64).reshape(-1, 8, 8)
    cols = idct8([v[:, k, :] for k in range(8)], False)  # element k of every column: raster row k
    v = np.stack(cols, axis=1)
    rows = idct8([v[:, :, k] for k in range(8)], True)
    return np.stack(rows, axis=2).reshape(np.shape(blocks))


def residuals(records, coef, mb_width, mb_height):
    """What decode_residuals gives (int16 [coded_size * 3 // 2]: Y | Cr | Cb) for the records and coefficient plane of
    a picture of mb_width x mb_height macroblocks: residual_planes() of its coefficients()."""
    return residual_planes(coefficients(records, coef), mb_width, mb_height)


def residual_planes(blocks, mb_width, mb_height):
    """The residual of a picture from what decode_coefficients gives for it (int16 [mb_size, 6, 64] or any shape of as
    many values): every block premultiplied and transformed (idct), placed where stage 2 writes it -- blocks 0-3 the
    luma quadrants, 4 Cb (the third plane), 5 Cr (the second).  int16 [coded_size * 3 // 2]: Y | Cr | Cb."""
    c = np.asarray(blocks).reshape(-1, 64).astype(np.int64)
    px = idct(c * PREMULTIPLIER).astype(np.int16).reshape(mb_height, mb_width, 6, 8, 8)
    y = px[:, :, :4].reshape(mb_height, mb_width, 2, 2, 8, 8).transpose(0, 2, 4, 1, 3, 5)
    cb = px[:, :, 4].transpose(0, 2, 1, 3)
    cr = px[:, :, 5].transpose(0, 2, 1, 3)
    return np.concatenate([y.reshape(-1), cr.reshape(-1), cb.reshape(-1)])
