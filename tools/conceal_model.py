"""Serial model of the `conceal` option (include/jsmpeg_b200.h, DESIGN 3.19): the oracle's decode() with the rule.

The oracle (oracle/mpeg1_oracle.c) parses each picture; this model keeps its own plane sets with the oracle's rotation
(two I/P sets, `forward` and `current`, swapped after every I/P picture; two B-picture sets written in turn) and
reconstructs every PIC_DECODED picture with the oracle's own oracle_reconstruct / oracle_reconstruct_b.  With
conceal on, before that call every macroblock whose record lacks MBF_PRESENT gets the co-located samples of the
picture's forward set: for an I/P picture `forward` (the newest I/P picture before it), for a B picture `current`
(its past reference).  With conceal off the model is the oracle's decode() exactly.
"""
from __future__ import annotations

import ctypes
import random

import numpy as np

import intra_model
import macroblock_model

MBF_PRESENT = 0x01
MBF_INTRA = 0x02
PIC_DECODED = 1
TS_PAYLOAD = 184  # the payload of one MPEG-TS packet


class _Planes(ctypes.Structure):  # the oracle's planes_t
    _fields_ = [("y", ctypes.c_void_p), ("cr", ctypes.c_void_p), ("cb", ctypes.c_void_p)]


class PlaneSet:
    """Y | Cr | Cb of the coded size in one array (the product's plane-set layout)."""

    def __init__(self, coded_width, coded_height):
        self.ysize = coded_width * coded_height
        self.data = np.zeros(self.ysize * 3 // 2, dtype=np.uint8)

    def planes(self):
        base = self.data.ctypes.data
        return _Planes(base, base + self.ysize, base + self.ysize + self.ysize // 4)


def macroblock_views(data, mb_width, mb_height):
    """(luma [mb_h, mb_w, 16, 16], Cr, Cb [mb_h, mb_w, 8, 8]) views of one Y | Cr | Cb array."""
    ysize = mb_width * mb_height * 256
    y = data[:ysize].reshape(mb_height, 16, mb_width, 16).transpose(0, 2, 1, 3)
    cr = data[ysize:ysize * 5 // 4].reshape(mb_height, 8, mb_width, 8).transpose(0, 2, 1, 3)
    cb = data[ysize * 5 // 4:].reshape(mb_height, 8, mb_width, 8).transpose(0, 2, 1, 3)
    return y, cr, cb


def conceal(cur, fwd, absent, mb_width, mb_height):
    """The rule: the macroblocks `absent` (bool [mb_size]) of `cur` get `fwd`'s co-located samples (both Y | Cr | Cb)."""
    a = absent.reshape(mb_height, mb_width)
    for c, f in zip(macroblock_views(cur, mb_width, mb_height), macroblock_views(fwd, mb_width, mb_height)):
        c[a] = f[a]


def records(olib, d, mb_size):
    """uint8 [mb_size, 16]: the oracle's last picture's macroblock records (a copy)"""
    return np.ctypeslib.as_array(ctypes.cast(olib.oracle_last_mb_records(d), ctypes.POINTER(ctypes.c_uint8)),
                                 shape=(mb_size * 16,)).reshape(mb_size, 16).copy()


def present_mask(olib, d, mb_size):
    """bool [mb_size]: the oracle's last picture's macroblocks with MBF_PRESENT."""
    return (records(olib, d, mb_size)[:, 4] & MBF_PRESENT) != 0


def zero_unfinished_intra_blocks(cur, hdr, mb_width, mb_height):
    """Stage 2's rule for a PRESENT intra macroblock whose walk stopped inside it (DESIGN 3.9): the blocks it did not
    finish (cbp bit clear) come out 0, where the oracle leaves the plane's content.  In an undamaged stream every
    intra macroblock codes all six blocks, so this changes nothing there."""
    rec = hdr.reshape(mb_height, mb_width, 16)
    intra = (rec[..., 4] & (MBF_PRESENT | MBF_INTRA)) == (MBF_PRESENT | MBF_INTRA)
    y, cr, cb = macroblock_views(cur, mb_width, mb_height)
    for b in range(6):
        m = intra & ((rec[..., 5] & (0x20 >> b)) == 0)
        if b < 4:
            y[m, (b >> 1) * 8:(b >> 1) * 8 + 8, (b & 1) * 8:(b & 1) * 8 + 8] = 0
        else:
            (cb if b == 4 else cr)[m] = 0


def decode(olib, es, conceal_on, decode_b=False, product=True):
    """Every decode() of the oracle over `es` (as MPEG1Video drives it), with the rule when `conceal_on` and, with
    `product`, stage 2's rule for unfinished intra blocks (zero_unfinished_intra_blocks).  Yields per
    decode() a dict: "type" (picture_coding_type), "decoded" (PIC_DECODED), "start_byte" (the first byte after its
    start code), "planes" (Y | Cr | Cb of what the decoder shows after it: a copy), and for a decoded picture
    "present" (bool [mb_size]), "fwd" and "bwd" (copies of its references, bwd None for I/P) and "before" (its
    destination set before the rule and the reconstruction)."""
    from jsmpeg_b200 import decoder
    vp = ctypes.c_void_p
    olib.oracle_reconstruct.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp, ctypes.POINTER(_Planes), ctypes.POINTER(_Planes)]
    olib.oracle_reconstruct_b.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, vp, ctypes.POINTER(_Planes),
                                          ctypes.POINTER(_Planes), ctypes.POINTER(_Planes)]
    olib.oracle_set_decode_b(1 if decode_b else 0)
    d = decoder.MPEG1Video({"decodeFirstFrame": False}, lib=olib)
    try:
        d.write(0, [es])
        if not olib.mpeg1_decoder_has_sequence_header(d.decoder):
            return
        seq = olib.oracle_seq_params(d.decoder)
        mb_width, mb_size = seq.contents.mb_width, seq.contents.mb_size
        mb_height = mb_size // mb_width
        cw, ch = mb_width * 16, mb_height * 16
        forward, current = PlaneSet(cw, ch), PlaneSet(cw, ch)
        bout, b_cur, last_was_b = [PlaneSet(cw, ch), PlaneSet(cw, ch)], 0, False
        seq_ptr = ctypes.cast(seq, vp)
        while d.decode():
            info = olib.oracle_last_picture_info(d.decoder).contents
            out = {"type": info.picture_type, "decoded": info.status == PIC_DECODED, "start_byte": info.start_byte}
            if out["decoded"]:
                hdr, coef = olib.oracle_last_mb_records(d.decoder), olib.oracle_last_coefficients(d.decoder)
                present = present_mask(olib, d.decoder, mb_size)
                is_b = info.picture_type == 3
                dst, fwd, bwd = (bout[b_cur], current, forward) if is_b else (current, forward, None)
                out.update(present=present, fwd=fwd.data.copy(), bwd=None if bwd is None else bwd.data.copy(),
                           before=dst.data.copy())
                if conceal_on:
                    conceal(dst.data, fwd.data, ~present, mb_width, mb_height)
                if product:
                    zero_unfinished_intra_blocks(dst.data, records(olib, d.decoder, mb_size), mb_width, mb_height)
                p_fwd, p_dst = fwd.planes(), dst.planes()
                if is_b:
                    p_bwd = bwd.planes()
                    olib.oracle_reconstruct_b(seq_ptr, cw, ch, hdr, coef, ctypes.byref(p_fwd), ctypes.byref(p_bwd),
                                              ctypes.byref(p_dst))
                    b_cur ^= 1
                    last_was_b = True
                else:
                    olib.oracle_reconstruct(seq_ptr, cw, ch, hdr, coef, ctypes.byref(p_fwd), ctypes.byref(p_dst))
                    forward, current = current, forward
                    last_was_b = False
            out["planes"] = (bout[b_cur ^ 1] if last_was_b else forward).data.copy()
            yield out
    finally:
        d.destroy()
        olib.oracle_set_decode_b(0)


# ---- damage of the kinds the option is for

def lost_packets(es, every=6, seed=0):
    """`es` with one 184-byte run cut from inside every `every`-th listed picture (a TS packet lost), past its
    picture header and before its closing code; pictures too small for that keep their bytes."""
    rng = random.Random(seed)
    out, at = bytearray(), 0
    for e in macroblock_model.macroblock_index(es)[1::every]:
        lo, hi = e["byte_pos"] + 12, e["close"] - TS_PAYLOAD - 4
        if hi <= lo:
            continue
        cut = rng.randrange(lo, hi)
        out += es[at:cut]
        at = cut + TS_PAYLOAD
    return bytes(out + es[at:])


def repeated_row(es, every=3):
    """`es` with, in every `every`-th listed picture that has slices of vertical positions 1 and 3, the slice of
    position 3 replaced by a copy of the slice of position 1: a picture without an invalid code that writes the first
    row twice and leaves the third out, so that its walk counts exactly as many macroblocks as a whole picture has."""
    out, at = bytearray(), 0
    for e in macroblock_model.macroblock_index(es)[::every]:
        codes = [p for p in intra_model.prefixes(es) if e["byte_pos"] < p <= e["close"]]
        span = {es[p + 3]: (p, q) for p, q in zip(codes, codes[1:]) if 0x01 <= es[p + 3] <= 0xAF}
        if 1 not in span or 3 not in span:
            continue
        (p1, q1), (p3, q3) = span[1], span[3]
        out += es[at:p3] + es[p1:q1]
        at = q3
    return bytes(out + es[at:])
