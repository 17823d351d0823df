"""Serial model of the picture index (jsmpeg_b200_batch_picture_index) and of what decode_pictures must give.

Picture k of a stream is the k-th picture start code (00 00 01 00) in its buffer.  The index lists picture k when
  1. it starts at or after the end of the stream's first sequence header,
  2. it is closed (tools/intra_model.py),
  3. decode() reconstructs it: picture_coding_type 1; 2 with forward_f_code != 0; with decode_b, 3 with both f_codes
     != 0 (the fixed-position header bits: temporal_reference 10, type 3, vbv_delay 16, full_pel_forward_vector 1,
     forward_f_code 3, full_pel_backward_vector 1, backward_f_code 3), and
  4. it has a chain start: the greatest picture j <= k of the intra index such that at least r(k) pictures of [j, k)
     are references (I, or P with forward_f_code != 0); r is 0 for I, 1 for P, 2 for B.
A listed picture decodes to what a fresh decoder gives, right after the decode() that consumes picture k, for
fresh_bytes(): the first sequence header, then the bytes from picture j up to and including picture k's closing code.
"""
from __future__ import annotations

import intra_model


def header_bits(es, pos, bit, n):
    """`n` bits of the picture header whose start code is at `pos`, from bit `bit` after the start code (0 beyond
    the buffer)."""
    v = 0
    for b in range(bit, bit + n):
        i = pos + 4 + (b >> 3)
        v = v << 1 | ((es[i] >> (7 - (b & 7))) & 1 if i < len(es) else 0)
    return v


def picture_type(es, pos):
    return (es[pos + 5] >> 3) & 7 if pos + 5 < len(es) else 0


def is_reference(es, pos):
    t = picture_type(es, pos)
    return t == 1 or (t == 2 and header_bits(es, pos, 30, 3) != 0)


def is_decoded(es, pos, decode_b):
    """Whether decode() reconstructs the picture (the walks' PIC_DECODED)."""
    t = picture_type(es, pos)
    if t == 3:
        return decode_b and header_bits(es, pos, 30, 3) != 0 and header_bits(es, pos, 34, 3) != 0
    return is_reference(es, pos)


def picture_index(es, decode_b=False):
    """[{"picture", "byte_pos", "type", "temporal_reference", "chain_start", "chain_start_pos", "close"}] of the
    pictures the index lists for a buffer `es`."""
    seq = intra_model.first_sequence_header(es)
    if seq is None:
        return []
    floor = (seq[1] + 7) >> 3
    codes = [p for p in intra_model.prefixes(es) if p + 3 < len(es)]
    close_after = [None] * (len(codes) + 1)  # close_after[i]: the first closing code among codes[i:]
    for i in range(len(codes) - 1, -1, -1):
        close_after[i] = codes[i] if intra_model._closes(es[codes[i] + 3]) else close_after[i + 1]
    pics = [(i, p) for i, p in enumerate(codes) if es[p + 3] == 0]
    out, keys, refs_upto, refs = [], [], [], 0
    for k, (i, p) in enumerate(pics):
        refs_upto.append(refs)
        t = picture_type(es, p)
        if p >= floor and t == 1:
            keys.append(k)
        refs += is_reference(es, p)
        close = close_after[i + 1]
        if p < floor or close is None or not is_decoded(es, p, decode_b):
            continue
        need = {1: 0, 2: 1, 3: 2}[t]
        j = next((j for j in reversed(keys) if refs_upto[k] - refs_upto[j] >= need), None)
        if j is not None:
            out.append({"picture": k, "byte_pos": p, "type": t, "temporal_reference": header_bits(es, p, 0, 10),
                        "chain_start": j, "chain_start_pos": pics[j][1], "close": close})
    return out


def fresh_bytes(es, entry):
    """What a fresh decoder is fed for a listed picture: first sequence header + chain start .. closing code."""
    return intra_model.fresh_bytes(es, {"byte_pos": entry["chain_start_pos"], "close": entry["close"]})


def seek_start(es, entry, decode_b=False):
    """The seek chain start of a listed picture (jsmpeg_b200_batch_seek_pictures): the index's chain start, except
    that under decode_b an I picture needs one reference before it -- the greatest I picture j < k after the first
    sequence header, or k itself where there is none -- so that the B pictures after k (of an open GOP) get both
    their references."""
    if not decode_b or entry["type"] != 1:
        return entry["chain_start"]
    floor = (intra_model.first_sequence_header(es)[1] + 7) >> 3
    pics = picture_positions(es)
    return next((j for j in range(entry["picture"] - 1, -1, -1) if pics[j] >= floor and picture_type(es, pics[j]) == 1),
                entry["picture"])


def seek_bytes(es, entry, decode_b=False):
    """What the fresh decoder of a seek is fed: the first sequence header, then everything from the seek chain start
    to the end of the buffer.  A position in it is the same position of `es` plus len(es) - len(seek_bytes(...))."""
    start = picture_positions(es)[seek_start(es, entry, decode_b)]
    return intra_model.fresh_bytes(es, {"byte_pos": start, "close": len(es) - 4})


def picture_positions(es):
    """Byte positions of the picture start codes (00 00 01 00) of `es`: picture k is the k-th."""
    return [p for p in intra_model.prefixes(es) if p + 3 < len(es) and es[p + 3] == 0]


def target_start_byte(es, entry):
    """Where picture k's header starts (the byte after its start code) inside fresh_bytes(es, entry)."""
    header = len(fresh_bytes(es, entry)) - (entry["close"] + 4 - entry["chain_start_pos"])
    return header + entry["byte_pos"] - entry["chain_start_pos"] + 4
