"""MPEG program streams for tests: a writer with knobs and a serial model demuxer.

The model is a plain restatement of what jsmpeg_b200_batch_write_ps does on the device (psdemux.cu,
DESIGN section 3.5); the tests compare the device against it byte for byte.

Items follow one another with no gaps; by the bytes at the item start:
    00 00 01 BA, next byte 0010xxxx   ISO 11172-1 pack header          12 bytes
    00 00 01 BA, next byte 01xxxxxx   ISO 13818-1 pack header          14 + (byte 13 & 7)
    00 00 01 B9                       end code                          4
    00 00 01 BB..FF                   system header, PSM, PES packet    6 + packet_length
The chain starts at the first valid pack header (00 00 01 BA + a byte of either form).  Bytes that are
not a valid item where one should start are a break; parsing resumes at the next valid pack header.
The payload of every PES packet of the selected stream id is appended to the elementary stream; a
packet with a PTS and a non-empty payload also gives a PES table entry (ES offset, 33-bit PTS).
"""
from __future__ import annotations

import numpy as np

ITEM, NEED_MORE, BAD = 0, 1, 2


def item_at(b, p):
    """(kind, length) of what starts at b[p:] -- psdemux.cuh ps_item_at."""
    have = len(b) - p
    for k, want in enumerate((0, 0, 1)):
        if k >= have:
            return NEED_MORE, 0
        if b[p + k] != want:
            return BAD, 0
    if have < 4:
        return NEED_MORE, 0
    code = b[p + 3]
    if code == 0xBA:
        if have < 5:
            return NEED_MORE, 0
        if b[p + 4] >> 4 == 2:
            n = 12
        elif b[p + 4] >> 6 == 1:
            if have < 14:
                return NEED_MORE, 0
            n = 14 + (b[p + 13] & 7)
        else:
            return BAD, 0
    elif code == 0xB9:
        n = 4
    elif code > 0xB9:
        if have < 6:
            return NEED_MORE, 0
        n = 6 + (b[p + 4] << 8 | b[p + 5])
    else:
        return BAD, 0
    return (ITEM, n) if n <= have else (NEED_MORE, 0)


def is_pack(b, p):
    return (len(b) - p >= 5 and b[p] == 0 and b[p + 1] == 0 and b[p + 2] == 1 and b[p + 3] == 0xBA
            and (b[p + 4] >> 4 == 2 or b[p + 4] >> 6 == 1))


def read_pts(q):
    return ((q[0] >> 1) & 7) << 30 | (q[1] << 7 | q[2] >> 1) << 15 | (q[3] << 7 | q[4] >> 1)


def payload(pkt):
    """(start, length, pts or None) of the PES packet `pkt` (the whole packet) -- psdemux.cuh ps_payload."""
    n = len(pkt)
    i, pts_at = 6, None
    empty = (n, 0, None)
    if i < n and pkt[i] >> 6 == 2:  # ISO 13818-1
        if n < 9:
            return empty
        if pkt[7] & 0x80:
            pts_at = 9
        i = 9 + pkt[8]
        if pts_at is not None and n < 14:
            return empty
    else:  # ISO 11172-1
        while i < n and pkt[i] == 0xFF:
            i += 1
        if i >= n:
            return empty
        if pkt[i] >> 6 == 1:
            i += 2
            if i >= n:
                return empty
        c = pkt[i] >> 4
        if c == 2:
            pts_at, i = i, i + 5
        elif c == 3:
            pts_at, i = i, i + 10
        else:
            i += 1
    if i > n:
        return empty
    return i, n - i, (read_pts(pkt[pts_at:pts_at + 5]) if pts_at is not None else None)


def find_pack(b, start):
    q = b.find(b"\x00\x00\x01\xba", start)
    while q >= 0 and len(b) - q >= 5:
        if is_pack(b, q):
            return q
        q = b.find(b"\x00\x00\x01\xba", q + 1)
    return -1


def demux(data, stream_id=0xE0, in_sync=False, items=None):
    """One call on one buffer (leftover + new bytes).  Returns (es bytes, [(es offset, pts)], bytes
    consumed, in_sync after).  `items`, a list, receives (pos, kind, length, payload start, payload
    length, pts) of every item the chain visits."""
    b = bytes(data)
    n = len(b)
    es, pes = bytearray(), []
    pos = 0 if in_sync else -1
    search = 0
    while True:
        if pos < 0:  # out of sync: next valid pack header at or after `search`
            pos = find_pack(b, search)
            if pos < 0:
                return bytes(es), pes, max(search, n - 4, 0), False
        if pos == n:
            return bytes(es), pes, n, True
        kind, ln = item_at(b, pos)
        if kind == NEED_MORE:
            return bytes(es), pes, pos, True
        if kind == BAD:
            search, pos = pos + 1, -1
            continue
        ps, pl, pts = payload(b[pos:pos + ln]) if b[pos + 3] > 0xBB else (ln, 0, None)
        if items is not None:
            items.append((pos, kind, ln, ps, pl, pts))
        if b[pos + 3] == stream_id and pl:
            if pts is not None:
                pes.append((len(es), pts))
            es += b[pos + ps:pos + ps + pl]
        pos += ln


class Demuxer:
    """Streaming wrapper: write() any chunking, like jsmpeg_b200_batch_write_ps on one stream."""

    def __init__(self, stream_id=0xE0):
        self.stream_id = stream_id
        self.leftover = b""
        self.in_sync = False
        self.es = bytearray()
        self.pes = []

    def write(self, data):
        """Returns (ES bytes appended, [(es offset, pts)] of this call)."""
        buf = self.leftover + bytes(data)
        es, pes, consumed, self.in_sync = demux(buf, self.stream_id, self.in_sync)
        self.leftover = buf[consumed:]
        pes = [(len(self.es) + o, t) for o, t in pes]
        self.es += es
        self.pes += pes
        return len(es), pes


def demux_chunked(data, cuts, stream_id=0xE0):
    d = Demuxer(stream_id)
    prev = 0
    for c in list(cuts) + [len(data)]:
        d.write(data[prev:c])
        prev = c
    return bytes(d.es), d.pes


# ---- writer ------------------------------------------------------------------------------------

def _ts_bytes(prefix, t):
    """5-byte PTS/DTS field with a 4-bit prefix (ISO 11172-1 2.4.4.2)."""
    t &= (1 << 33) - 1
    return bytes([prefix << 4 | (t >> 29) & 0x0E | 1, (t >> 22) & 0xFF, (t >> 14) & 0xFE | 1,
                  (t >> 7) & 0xFF, (t << 1) & 0xFE | 1])


def pack_header(form, scr=0, mux_rate=2000, stuffing=0):
    if form == "mpg":  # ISO 11172-1 2.4.3.2
        return (b"\x00\x00\x01\xba" + _ts_bytes(2, scr)
                + bytes([0x80 | (mux_rate >> 15) & 0x7F, (mux_rate >> 7) & 0xFF, (mux_rate << 1) & 0xFE | 1]))
    # ISO 13818-1 2.5.3.3
    v = 1 << 46 | (scr >> 30 & 7) << 43 | 1 << 42 | (scr >> 15 & 0x7FFF) << 27 | 1 << 26 | (scr & 0x7FFF) << 11 | 1 << 10 | 1
    return (b"\x00\x00\x01\xba" + v.to_bytes(6, "big")
            + bytes([(mux_rate >> 14) & 0xFF, (mux_rate >> 6) & 0xFF, (mux_rate << 2) & 0xFC | 3, 0xF8 | stuffing])
            + b"\xff" * stuffing)


def system_header():
    body = bytes([0x80, 0x07, 0xD1, 0x04, 0xE1, 0xFF, 0xE0, 0xE0, 0x2E, 0xC0, 0xC0, 0x20])
    return b"\x00\x00\x01\xbb" + len(body).to_bytes(2, "big") + body


def pes_packet(sid, body, form, pts=None, dts=None, stuffing=0, std=False):
    if form == "mpg":
        h = b"\xff" * stuffing + (b"\x60\x2e" if std else b"")
        if pts is None:
            h += b"\x0f"
        elif dts is None:
            h += _ts_bytes(2, pts)
        else:
            h += _ts_bytes(3, pts) + _ts_bytes(1, dts)
    else:
        opt = b""
        flags = 0
        if pts is not None:
            flags = 0x80 if dts is None else 0xC0
            opt = _ts_bytes(2 if dts is None else 3, pts) + (_ts_bytes(1, dts) if dts is not None else b"")
        opt += b"\xff" * stuffing
        h = bytes([0x81, flags, len(opt)]) + opt
    return b"\x00\x00\x01" + bytes([sid]) + (len(h) + len(body)).to_bytes(2, "big") + h + body


def hostile_audio(rng, n):
    """Audio bytes that contain start codes a byte-level scanner could take for items."""
    a = bytearray(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
    for code in (b"\x00\x00\x01\xba\x21", b"\x00\x00\x01\xe0\x07", b"\x00\x00\x01\xbb\x00", b"\x00\x00\x01\xba\x44"):
        if n > 16:
            at = int(rng.integers(0, n - len(code)))
            a[at:at + len(code)] = code
    return bytes(a)


def mux(es, form="mpg", packet=2048, stuffing=0, std=False, pts_mode="pts", pts_every=1, padding=False,
        private=False, sys_every=0, end_code=False, garbage=0, audio=0, seed=0, pack_stuffing=0):
    """Program stream carrying `es` as stream 0xE0.  Returns (stream bytes, [(es offset, pts)] the demuxer
    must report).  form "mpg" = ISO 11172-1, "vob" = ISO 13818-1; packet = video payload bytes per PES
    packet; stuffing 0-16 bytes in every video header; std: STD buffer field (11172-1 form); pts_mode
    "pts" | "pts_dts" | "none", on every `pts_every`-th video packet; padding: a 0xBE packet after every
    video packet; private: a private_stream_2 packet after every pack header; sys_every: a system header
    in every sys_every-th pack (0: first pack only); end_code: an end code after the 3rd pack, then
    more packs; garbage: that many random bytes in front; audio: a 0xC0 packet of that many hostile
    bytes after every video packet."""
    rng = np.random.default_rng(seed)
    out = bytearray(rng.integers(0, 256, garbage, dtype=np.uint8).tobytes())
    table = []
    k = 0
    for off in range(0, len(es), packet):
        body = es[off:off + packet]
        out += pack_header(form, scr=off * 3, stuffing=pack_stuffing)
        if k == 0 or (sys_every and k % sys_every == 0):
            out += system_header()
        if private:
            out += b"\x00\x00\x01\xbf" + (20).to_bytes(2, "big") + bytes(range(20))
        pts = dts = None
        if pts_mode != "none" and k % pts_every == 0:
            pts = 3003 * k + 90000 + (1 << 32) * (k % 3 == 2)  # exercise bit 32
            dts = pts - 3003 if pts_mode == "pts_dts" else None
            table.append((off, pts & ((1 << 33) - 1)))
        out += pes_packet(0xE0, body, form, pts, dts, stuffing, std and form == "mpg")
        if audio:
            out += pes_packet(0xC0, hostile_audio(rng, audio), form, pts=pts)
        if padding:
            out += b"\x00\x00\x01\xbe" + (30).to_bytes(2, "big") + b"\xff" * 30
        if end_code and k == 2:
            out += b"\x00\x00\x01\xb9"
        k += 1
    out += b"\x00\x00\x01\xb9"
    return bytes(out), table
