"""Serial model of what decode_accumulated must give (include/jsmpeg_b200.h, DESIGN 3.11).

A map is int16 [coded_size * 3 // 2, 4] in the planes' layout (Y | Cr | Cb): per sample (dx, dy, residual, back), back
-1 for an untraced sample.  step() is one depth: the map of reference picture p_m from that of p_(m-1), p_m's records
and residual; oracle_chain() folds it over a chain.  The chain's pictures are those the oracle's decode() reconstructs,
with B pictures off, when fed chain_model.fresh_bytes() of the requested picture (oracle_chain).  sequential() is the
map decode() keeps under OUT_ACCUMULATED: the same step, folded over the I/P pictures decode() reconstructs.
"""
from __future__ import annotations

import ctypes

import numpy as np

import chain_model
import macroblock_model

UNTRACED = -1


def inside(src, stride, plane_size, oh, ov):
    """Stage 2's flat-index rule (PREDICTION_INSIDE, jsmpeg_b200/csrc/common.cuh): every tap of a block's prediction,
    whose first tap is at flat index `src`, lies inside the plane"""
    return (src >= 0) & (src + 7 * stride + 7 + np.where(ov, stride, 0) + np.where(oh, 1, 0) < plane_size)


def _halve(v):
    """a chroma vector component: the luma one divided by 2, truncated toward zero"""
    return np.where(v < 0, -((-v) // 2), v // 2)


def _plane(prev, flags, mh, mv, res, mb_width, mb_height, chroma):
    """The map [size, 4] of one plane: flags / mh / mv per macroblock [mb_height, mb_width], res [size]"""
    px = 8 if chroma else 16
    stride, rows = mb_width * px, mb_height * px
    size = stride * rows
    if chroma:
        mh, mv = _halve(mh), _halve(mv)
    by, bx = np.mgrid[0:rows // 8, 0:stride // 8]
    mby, mbx = by * 8 // px, bx * 8 // px
    bh, bv, bf = mh[mby, mbx], mv[mby, mbx], flags[mby, mbx]
    src = by * 8 * stride + bx * 8 + (bv >> 1) * stride + (bh >> 1)
    present = (bf & macroblock_model.MBF_PRESENT) != 0
    predicted = present & ((bf & macroblock_model.MBF_INTRA) == 0) & inside(src, stride, size, bh & 1, bv & 1)

    def samples(x):
        return np.repeat(np.repeat(x, 8, 0), 8, 1).reshape(-1)

    out = np.zeros((size, 4), np.int64)
    out[:, 3] = np.where(samples(present & ~predicted), 0, UNTRACED)
    if prev is not None:
        sh, sv, traced = samples(bh), samples(bv), samples(predicted)
        at = np.where(traced, np.arange(size) + (sv >> 1) * stride + (sh >> 1), 0)
        p = prev[at].astype(np.int64)
        ok = traced & (p[:, 3] >= 0)
        out[ok, 0] = p[ok, 0] + sh[ok]
        out[ok, 1] = p[ok, 1] + sv[ok]
        out[ok, 2] = p[ok, 2] + res.astype(np.int64)[ok]
        out[ok, 3] = p[ok, 3] + 1
    return np.clip(out, -32768, 32767)


def step(prev, records, residual, mb_width, mb_height):
    """The map of a reference picture from `prev` (the previous reference picture's map, or None for the chain's first
    picture), its mb_record_t records (any 16-byte-per-record buffer) and its residual (int16 [coded_size * 3 // 2],
    macroblock_model.residuals)"""
    r = np.frombuffer(np.ascontiguousarray(records).tobytes(), macroblock_model.RECORD)
    flags = r["flags"].astype(np.int64).reshape(mb_height, mb_width)
    mh = r["mv_h"].astype(np.int64).reshape(mb_height, mb_width)
    mv = r["mv_v"].astype(np.int64).reshape(mb_height, mb_width)
    n = mb_width * mb_height * 256
    res = np.asarray(residual)
    prev = None if prev is None else np.asarray(prev)
    cut = [(0, n), (n, n + n // 4), (n + n // 4, n + n // 2)]  # Y, Cr, Cb
    return np.concatenate([_plane(None if prev is None else prev[a:z], flags, mh, mv, res[a:z], mb_width, mb_height, k > 0)
                           for k, (a, z) in enumerate(cut)]).astype(np.int16)


def depth(prev, records, coef, mb_width, mb_height):
    """step() with the residual of the picture's coefficient plane (macroblock_model.residual_planes of its
    coefficients)"""
    return step(prev, records, macroblock_model.residuals(records, coef, mb_width, mb_height), mb_width, mb_height)


def untraced(mb_width, mb_height):
    m = np.zeros((mb_width * mb_height * 384, 4), np.int16)
    m[:, 3] = UNTRACED
    return m


def oracle_decode(lib, es, stop=None, decode_b=False, index=None):
    """The oracle (B pictures off, or on with `decode_b`) fed `es`: [(start byte, picture_info, records, coefficient
    plane, planes)] of every picture its decode() consumes, up to the one whose header starts at byte `stop`; with
    `index`, from that bit index on (set_index right after the write)."""
    from jsmpeg_b200 import decoder

    import helpers
    lib.oracle_set_decode_b(int(decode_b))
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=lib)
    d.write(0.0, [es])
    if index is not None:
        d.bufferSetIndex(index)
    seq = lib.oracle_seq_params(d.decoder)
    mb, mbw = seq.contents.mb_size, seq.contents.mb_width
    cs = mb * 256
    out = []
    while d.decode():
        info = helpers.PictureInfo.from_buffer_copy(lib.oracle_last_picture_info(d.decoder).contents)
        rec = np.ctypeslib.as_array(ctypes.cast(lib.oracle_last_mb_records(d.decoder), ctypes.POINTER(ctypes.c_uint8)),
                                    shape=(mb * 16,)).reshape(mb, 16).copy()
        coef = np.ctypeslib.as_array(ctypes.cast(lib.oracle_last_coefficients(d.decoder), ctypes.POINTER(ctypes.c_int16)),
                                     shape=(mb * 6 * 64,)).copy()
        planes = np.concatenate([np.ctypeslib.as_array(ctypes.cast(p(d.decoder), ctypes.POINTER(ctypes.c_uint8)),
                                                       shape=(n,)).copy()
                                 for p, n in ((lib.mpeg1_decoder_get_y_ptr, cs), (lib.mpeg1_decoder_get_cr_ptr, cs // 4),
                                              (lib.mpeg1_decoder_get_cb_ptr, cs // 4))])
        out.append((info.start_byte, info, rec, coef, planes))
        if stop is not None and info.start_byte >= stop:
            break
    d.destroy()
    lib.oracle_set_decode_b(0)
    return out, mbw, mb // mbw


def oracle_chain(lib, es, entry, rest=False):
    """(status, n_present, error, map) that decode_accumulated must give for picture index entry `entry` of `es`: the
    fold over the pictures the oracle (B pictures off) reconstructs from chain_model.fresh_bytes(es, entry) -- with
    `rest`, from everything after the chain start instead, the bits a damaged picture's walk reads past its closing
    code; status 0 and an untraced map when it never consumes the picture."""
    target = chain_model.target_start_byte(es, entry)
    fed = chain_model.fresh_bytes(es, entry)
    if rest:
        fed = fed[:len(fed) - (entry["close"] + 4 - entry["chain_start_pos"])] + es[entry["chain_start_pos"]:]
    got, mbw, mbh = oracle_decode(lib, fed, stop=target)
    prev = None
    for start, info, rec, coef, _ in got:
        if info.status == 1 and info.picture_type in (1, 2):
            prev = depth(prev, rec, coef, mbw, mbh)
        if start == target:
            if info.status != 1:
                return info.status, info.n_present, info.error, untraced(mbw, mbh)
            return info.status, info.n_present, info.error, prev
    return 0, 0, 0, untraced(mbw, mbh)


def sequential(lib, es, decode_b=False, index=None):
    """The maps decode() with OUT_ACCUMULATED keeps for `es` (include/jsmpeg_b200.h): [(start byte, picture_info, map)]
    per I/P picture the oracle's decode() reconstructs (B pictures as `decode_b` says; from bit index `index` when
    given), each one step from the map of the I/P picture reconstructed before it -- none for the first, so a start on
    a P picture leaves its predicted samples untraced up to the next I picture.  B pictures get no map."""
    got, mbw, mbh = oracle_decode(lib, es, decode_b=decode_b, index=index)
    out, prev = [], None
    for start, info, rec, coef, _ in got:
        if info.status == 1 and info.picture_type in (1, 2):
            prev = depth(prev, rec, coef, mbw, mbh)
            out.append((start, info, prev))
    return out
