"""Serial model of the key-picture index (jsmpeg_b200_batch_intra_index) and of what decode_intra must give.

Picture k of a stream is the k-th picture start code (00 00 01 00) in its buffer.  The index lists picture k when
  1. it starts at or after the end of the stream's first sequence header (where decode() begins its search),
  2. its picture_coding_type (the 3 bits after the 10-bit temporal_reference) is 1, and
  3. it is closed: a later start code has all four bytes in the buffer, and its fourth byte is no slice (01..AF),
     user data (B2) or extension (B5).
A listed picture decodes to what a fresh decoder gives for fresh_bytes(): the first sequence header (from its
00 00 01 B3 up to the next start code), the picture's bytes up to its closing code, and the closing code itself.
"""
from __future__ import annotations

START = b"\x00\x00\x01"


def prefixes(es):
    """Byte positions of every 00 00 01 in `es`, in order (what the device scan lists)."""
    out, i = [], es.find(START)
    while i >= 0:
        out.append(i)
        i = es.find(START, i + 1)
    return out


def first_sequence_header(es):
    """(position of its 00 00 01 B3, bit index right after it) of the first sequence header, as the decoder's
    did_write finds it (a start code that is not B3 is skipped whole), or None."""
    i = 0
    while i + 3 < len(es):
        if es[i] == 0 and es[i + 1] == 0 and es[i + 2] == 1:
            if es[i + 3] == 0xB3:
                break
            i += 3
        i += 1
    else:
        return None

    def bit(b):
        return (es[b >> 3] >> (7 - (b & 7))) & 1 if (b >> 3) < len(es) else 0

    b = (i + 4) * 8 + 12 + 12 + 4 + 4 + 18 + 1 + 10 + 1  # width, height, aspect, rate, bit rate, marker, vbv, constrained
    if bit(b):
        b += 512  # intra matrix
    b += 1
    if bit(b):
        b += 512  # non-intra matrix
    return i, b + 1


def _closes(code):
    return not (0x01 <= code <= 0xAF) and code not in (0xB2, 0xB5)


def intra_index(es):
    """[{"picture", "byte_pos", "temporal_reference", "close"}] of the pictures the index lists for a buffer `es`."""
    seq = first_sequence_header(es)
    if seq is None:
        return []
    floor = (seq[1] + 7) >> 3
    codes = [p for p in prefixes(es) if p + 3 < len(es)]
    out, k = [], -1
    for j, p in enumerate(codes):
        if es[p + 3] != 0:
            continue
        k += 1
        if p < floor or p + 5 >= len(es) or (es[p + 5] >> 3) & 7 != 1:
            continue
        close = next((q for q in codes[j + 1:] if _closes(es[q + 3])), None)
        if close is not None:
            out.append({"picture": k, "byte_pos": p, "temporal_reference": es[p + 4] << 2 | es[p + 5] >> 6, "close": close})
    return out


def fresh_bytes(es, entry):
    """What a fresh decoder is fed for a listed picture: first sequence header + the picture + its closing code."""
    h = first_sequence_header(es)[0]
    nxt = es.find(START, h + 4)
    header = es[h:nxt if nxt >= 0 else len(es)]
    return header + es[entry["byte_pos"]:entry["close"] + 4]
