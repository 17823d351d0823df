"""Program stream inputs for the many-request demux tests (tests/test_ps_many_emu.py on the host,
tests/test_gpu_ps_many.py on the device): chunkings, a program stream of two video streams, and the counts that
fix a call's launches (candidates) and that make a damaged copy interesting (breaks)."""
import mini_ps
import ps_cases


def chunked(data, size, rng=None):
    """`data` in pieces of `size` bytes, or "random" sizes around 500 (rng picks the seed); at least one piece."""
    if size == "random":
        cuts = ps_cases.random_cuts(len(data), int(rng.integers(1 << 30)), mean=500)
        return [data[a:b] for a, b in zip([0] + cuts, cuts + [len(data)])]
    return [data[i:i + size] for i in range(0, len(data), size)] or [b""]


def two_video_program_stream(es_a, es_b, form="vob", packet=1500):
    """One program stream carrying es_a as 0xE0 and es_b as 0xE1, their packets interleaved."""
    out = bytearray()
    k = 0
    for off in range(0, max(len(es_a), len(es_b)), packet):
        out += mini_ps.pack_header(form, scr=off)
        if k == 0:
            out += mini_ps.system_header()
        for sid, es in ((0xE0, es_a), (0xE1, es_b)):
            if off < len(es):
                out += mini_ps.pes_packet(sid, es[off:off + packet], form, pts=90000 + 3003 * k + (sid & 1))
        k += 1
    return bytes(out + b"\x00\x00\x01\xb9")


def candidates(data):
    """The demuxer's candidates in one buffer: every 00 00 01 with a code >= B9 (or cut by the end)."""
    n, at, q = len(data), 0, data.find(b"\x00\x00\x01")
    count = 0
    while q >= 0:
        if q + 3 >= n or data[q + 3] >= 0xB9:
            count += 1
        at = q + 1
        q = data.find(b"\x00\x00\x01", at)
    return count


def breaks(data):
    """Breaks in the item chain of one buffer read from its first pack header: places where the model resyncs."""
    items = []
    mini_ps.demux(data, items=items)
    return sum(1 for a, b in zip(items, items[1:]) if a[0] + a[2] != b[0])
