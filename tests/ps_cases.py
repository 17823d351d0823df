"""Program stream test corpus shared by tests/test_ps_demux.py (model, CPU) and tests/test_gpu_ps_demux.py
(device): hand-written tiny streams with literal expected results, writer-made streams, damaged streams."""
import numpy as np

import mini_ps

PACK1 = "000001BA 21 0001 0001 800001"             # ISO 11172-1 pack header, 12 bytes
PACK2 = "000001BA 44 0004 0004 01 0189C3 FA FFFF"  # ISO 13818-1 pack header, 2 stuffing bytes: 16 bytes
END = "000001B9"
PTS = 32770  # "21 0003 0005": 1 << 15 | 2


def _h(*parts):
    return bytes.fromhex("".join(parts).replace(" ", ""))


# name -> (stream, expected ES, expected PES table [(ES offset, PTS)])
TINY = {
    "false_pack_in_audio": (_h(PACK1, "000001E0 0007 21 0003 0005 AABB",
                               "000001C0 0008 0F 000001BA 21 0001",
                               "000001E0 0002 0F CC", END),
                            bytes.fromhex("AABBCC"), [(0, PTS)]),
    "broken_length_resync": (_h(PACK1, "000001E0 0003 21 0003 0005 AABB",  # packet_length 7 damaged to 3
                                "000001E0 0002 0F DD",
                                PACK1, "000001E0 0002 0F EE", END),
                             bytes.fromhex("EE"), []),
    "end_code_then_pack": (_h(PACK1, "000001E0 0002 0F 11", END,
                              PACK1, "000001E0 0006 21 0003 0005 22", END),
                           bytes.fromhex("1122"), [(1, PTS)]),
    "incomplete_trailing_packet": (_h(PACK1, "000001E0 0002 0F 33", "000001E0 0010 0F 44"),
                                   bytes.fromhex("33"), []),
    "iso13818_pts_dts": (_h(PACK2, "000001E0 000F 81 C0 0A 31 0003 0005 11 0001 0001 5566", END),
                         bytes.fromhex("5566"), [(0, PTS)]),
    "stuffing16_std": (_h(PACK1, "000001E0 001E", "FF" * 16, "602E 31 0003 0005 11 0001 0001 7788", END),
                       bytes.fromhex("7788"), [(0, PTS)]),
    "leading_garbage": (_h("1234 000001BA FF 000001E0", PACK1, "000001E0 0002 0F 99", END),
                        bytes.fromhex("99"), []),
}


def video_es(n=24000, seed=5):
    """Video-like ES: random bytes with the start codes an MPEG-1 video stream has (none >= B9)."""
    rng = np.random.default_rng(seed)
    es = bytearray(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
    es[0:4] = b"\x00\x00\x01\xb3"
    for at in rng.integers(4, n - 4, n // 500):
        es[at:at + 4] = b"\x00\x00\x01" + bytes([int(rng.choice([0x00, 0x01, 0x2A, 0xB2, 0xB5, 0xB8]))])
    return bytes(es)


# writer knobs: name -> mux() keyword arguments
WRITER = {
    "mpg_plain": dict(form="mpg"),
    "vob_plain": dict(form="vob"),
    "mpg_all": dict(form="mpg", packet=1500, stuffing=16, std=True, pts_mode="pts_dts", padding=True, private=True,
                    sys_every=3, end_code=True, garbage=77, audio=400, seed=1),
    "vob_all": dict(form="vob", packet=1800, stuffing=9, pts_mode="pts_dts", padding=True, private=True, sys_every=2,
                    end_code=True, garbage=5, audio=700, seed=2, pack_stuffing=7),
    "mpg_sparse_pts": dict(form="mpg", packet=700, pts_mode="pts", pts_every=3, audio=100, seed=3),
    "vob_no_pts": dict(form="vob", packet=2300, pts_mode="none", audio=2000, seed=4),
}


def writer_case(name, n=24000):
    return mini_ps.mux(video_es(n), **WRITER[name])


def damaged(data, kind, seed):
    """A damaged copy of `data`: random byte flips, broken packet lengths or inserted garbage."""
    rng = np.random.default_rng(seed)
    b = bytearray(data)
    if kind == "flips":
        for at in rng.integers(0, len(b), max(4, len(b) // 1500)):
            b[at] = int(rng.integers(0, 256))
    elif kind == "lengths":
        starts = [i for i in range(len(b) - 6) if b[i:i + 3] == b"\x00\x00\x01" and b[i + 3] > 0xBA]
        for i in rng.choice(starts, min(len(starts), 6), replace=False):
            b[i + 4:i + 6] = int(rng.integers(0, 4096)).to_bytes(2, "big")
    elif kind == "garbage":
        for at in sorted(rng.integers(0, len(b), 5), reverse=True):
            b[at:at] = rng.integers(0, 256, int(rng.integers(1, 300)), dtype=np.uint8).tobytes() + b"\x00\x00\x01\xba"
    return bytes(b)


def random_cuts(n, seed, mean=700):
    rng = np.random.default_rng(seed)
    cuts, at = [], 0
    while True:
        at += int(rng.integers(1, 2 * mean))
        if at >= n:
            return cuts
        cuts.append(at)
