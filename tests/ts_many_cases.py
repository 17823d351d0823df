"""MPEG-TS inputs and the per-stream model for the many-stream TS write (jsmpeg_b200_batch_write_ts_many): garbage
between packets, a PID re-bound mid-stream, two video programs in one multiplex; and src/ts.js's host mirror
(jsmpeg_b200/ts.py) driven per stream, with the PES table write_ts reports."""
import numpy as np

from jsmpeg_b200 import ts

VIDEO_PID = 0x100  # gen_streams.make_clip_ts's video PID


def packets(data):
    return [bytearray(data[i:i + 188]) for i in range(0, len(data) - 187, 188)]


def pid_of(pkt):
    return ((pkt[1] & 0x1F) << 8) | pkt[2]


def pes_header_at(pkt):
    """Index of the PES header's 00 00 01 in a payload-start packet, or None."""
    if not (pkt[1] & 0x40) or not (pkt[3] & 0x10):
        return None
    at = 4 + (1 + pkt[4] if pkt[3] & 0x20 else 0)
    return at if at + 3 < 188 and pkt[at:at + 3] == b"\x00\x00\x01" else None


def with_garbage(data, seed, places=3):
    """1..186 bytes without a sync byte before `places` packets spread over the clip, each followed by >= 6 packets
    before the next: the resync (ts.js:155-189) finds every packet again and the ES is the clip's."""
    pk = packets(data)
    rng = np.random.default_rng(seed)
    where = {(len(pk) - 6) * (j + 1) // (places + 1) for j in range(places)}
    out = bytearray()
    for k, p in enumerate(pk):
        if k in where:
            junk = rng.integers(0, 256, int(rng.integers(1, 187)), dtype=np.uint8)
            junk[junk == 0x47] = 0x46
            out += junk.tobytes()
        out += p
    return bytes(out)


def rebound(data, first, last, to=0xE1):
    """The PES headers first .. last of the video PID name stream id `to`: the PID is bound away and back."""
    out, k = [], 0
    for p in packets(data):
        at = pes_header_at(p) if pid_of(p) == VIDEO_PID else None
        if at is not None:
            if first <= k <= last:
                p[at + 3] = to
            k += 1
        out.append(bytes(p))
    return b"".join(out)


def two_programs(a, b):
    """The video packets of clip b moved to PID 0x101 and stream id 0xE1, interleaved with clip a's packets."""
    pa = [bytes(p) for p in packets(a)]
    pb = []
    for p in packets(b):
        if pid_of(p) != VIDEO_PID:
            continue
        p[1] = (p[1] & 0xE0) | 0x01
        p[2] = 0x01
        at = pes_header_at(p)
        if at is not None:
            p[at + 3] = 0xE1
        pb.append(bytes(p))
    out = []
    for k in range(max(len(pa), len(pb))):
        out += pa[k:k + 1] + pb[k:k + 1]
    return b"".join(out)


class _Recorder(ts._PesInfo):
    """A PES destination that also records, per PES header of its stream, (ES offset of its payload, 90 kHz PTS):
    the table write_ts reports."""

    def __init__(self, col):
        self.on = False
        super().__init__(col)
        self.table = []
        self.on = True

    @property
    def pts_ticks(self):
        return ts._PesInfo.pts_ticks.__get__(self)

    @pts_ticks.setter
    def pts_ticks(self, v):
        if self.on:  # (ts.py sets it once per PES header of the stream)
            self.table.append((len(self.destination.es) + sum(len(b) for b in self.buffers), v))
        ts._PesInfo.pts_ticks.__set__(self, v)


class StreamModel:
    """ts.py fed one stream's writes: after each, what write_ts on the device returns and keeps."""

    def __init__(self, stream_id=0xE0):
        self.demux = ts.TS()
        self.col = ts.ESCollector()
        self.rec = _Recorder(self.col)
        self.demux.pes_packet_info[stream_id] = self.rec

    def es(self):
        return self.col.es + b"".join(self.rec.buffers)  # delivered + still held

    def write(self, data):
        """(ES bytes appended, [(offset, pts ticks), ...]) -- no PES entries for a write that appends nothing."""
        before, k = len(self.es()), len(self.rec.table)
        self.demux.write(data)
        appended = len(self.es()) - before
        new = self.rec.table[k:]
        if not appended:
            del self.rec.table[k:]
            new = []
        return appended, new

    @property
    def table(self):
        return self.rec.table

    @property
    def leftover(self):
        return self.demux.leftover

    @property
    def bound(self):
        return {pid: sid for pid, sid in self.demux.pids_to_stream_ids.items() if sid}


def chunked(data, chunk, rng=None):
    """data cut into pieces of `chunk` bytes; chunk "random": sizes 1 .. 4000 from rng."""
    if chunk == "random":
        out, i = [], 0
        while i < len(data):
            k = int(rng.integers(1, 4000))
            out.append(data[i:i + k])
            i += k
        return out
    return [data[i:i + chunk] for i in range(0, len(data), chunk)]
