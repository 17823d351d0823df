"""ctypes wrapper of the batch extension (include/jsmpeg_b200.h, part 2): N independent streams on
one GPU, device-resident planes, one call decodes the next pictures of every stream."""
from __future__ import annotations

import bisect
import ctypes

import numpy as np

OUT_DEVICE = 0
OUT_HOST = 1
OUT_RGBA = 2
OUT_MACROBLOCKS = 4  # every reconstructed picture's macroblock entries beside its planes (device_macroblocks)
OUT_ACCUMULATED = 8  # every reconstructed I/P picture's accumulated map beside its planes (device_accumulated)
OUT_RESIDUALS = 16  # the residual of the picture the planes hold, stored by stage 2 (device_residuals)


class Stats(ctypes.Structure):
    _fields_ = [
        ("pictures", ctypes.c_uint64), ("pictures_decoded", ctypes.c_uint64),
        ("coded_blocks", ctypes.c_uint64), ("macroblocks", ctypes.c_uint64),
        ("algorithmic_bytes", ctypes.c_uint64), ("es_bytes", ctypes.c_uint64),
        ("h2d_bytes", ctypes.c_uint64), ("d2h_bytes", ctypes.c_uint64),
        ("kernel_launches", ctypes.c_uint64), ("recon_launches", ctypes.c_uint64),
        ("parse_ms", ctypes.c_double), ("recon_ms", ctypes.c_double), ("scan_ms", ctypes.c_double),
        ("parse_errors", ctypes.c_uint64), ("walk_ms", ctypes.c_double),
        ("lane_walk_pictures", ctypes.c_uint64),
    ]

    def as_dict(self):
        return {name: getattr(self, name) for name, _ in self._fields_}


class Frame(ctypes.Structure):
    """jsmpeg_b200_frame_t: what decode_frames reports per frame (16 bytes)."""
    _fields_ = [("byte_pos", ctypes.c_uint32), ("picture_type", ctypes.c_int16), ("temporal_reference", ctypes.c_int16),
                ("n_present", ctypes.c_int32), ("error", ctypes.c_int32)]


_VP = ctypes.c_void_p
# decode_macroblocks', decode_coefficients' and decode_residuals' refusal (-2)
_NOT_IN_MACROBLOCK_INDEX = "a request names a picture that is not in the stream's macroblock index"


class FrameDst(ctypes.Structure):
    """jsmpeg_b200_frame_dst_t: decode_frames_into's destination arrays (one device pointer per stream each, NULL: none)."""
    _fields_ = [("planes", _VP), ("rgba", _VP), ("res", _VP), ("mb", _VP), ("coef", _VP), ("acc", _VP)]


_BATCH_ABI = {
    "jsmpeg_b200_batch_create": (_VP, [ctypes.c_int, ctypes.c_int, ctypes.c_uint]),
    "jsmpeg_b200_batch_destroy": (None, [_VP]),
    "jsmpeg_b200_batch_get_write_ptr": (_VP, [_VP, ctypes.c_int, ctypes.c_uint]),
    "jsmpeg_b200_batch_did_write": (None, [_VP, ctypes.c_int, ctypes.c_uint]),
    "jsmpeg_b200_batch_get_index": (ctypes.c_int, [_VP, ctypes.c_int]),
    "jsmpeg_b200_batch_set_index": (None, [_VP, ctypes.c_int, ctypes.c_uint]),
    "jsmpeg_b200_batch_stream_info": (ctypes.c_int, [_VP, ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                                     ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int),
                                                     ctypes.POINTER(ctypes.c_float)]),
    "jsmpeg_b200_batch_write_ts": (ctypes.c_long, [_VP, ctypes.c_int, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_int,
                                                   _VP, _VP, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]),
    "jsmpeg_b200_batch_write_ts_many": (ctypes.c_long, [_VP, ctypes.c_int, _VP, _VP, _VP, _VP, _VP, _VP, _VP, ctypes.c_long, _VP]),
    "jsmpeg_b200_batch_write_ps": (ctypes.c_long, [_VP, ctypes.c_int, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_int,
                                                   _VP, _VP, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]),
    "jsmpeg_b200_batch_write_ps_many": (ctypes.c_long, [_VP, ctypes.c_int, _VP, _VP, _VP, _VP, _VP, _VP, _VP, ctypes.c_long, _VP]),
    "jsmpeg_b200_batch_upload": (ctypes.c_long, [_VP]),
    "jsmpeg_b200_batch_rewind": (None, [_VP]),
    "jsmpeg_b200_batch_reset": (None, [_VP]),
    "jsmpeg_b200_batch_decode": (ctypes.c_long, [_VP, ctypes.c_int, ctypes.c_int]),
    "jsmpeg_b200_batch_get_planes": (ctypes.c_int, [_VP, ctypes.c_int, ctypes.POINTER(_VP), ctypes.POINTER(_VP), ctypes.POINTER(_VP)]),
    "jsmpeg_b200_batch_get_host_planes": (ctypes.c_int, [_VP, ctypes.c_int, ctypes.POINTER(_VP), ctypes.POINTER(_VP), ctypes.POINTER(_VP)]),
    "jsmpeg_b200_batch_get_rgba": (ctypes.c_int, [_VP, ctypes.c_int, ctypes.POINTER(_VP)]),
    "jsmpeg_b200_batch_read_planes": (ctypes.c_int, [_VP, ctypes.c_int, _VP, _VP, _VP]),
    "jsmpeg_b200_batch_read_rgba": (ctypes.c_int, [_VP, ctypes.c_int, _VP]),
    "jsmpeg_b200_batch_get_macroblocks": (ctypes.c_int, [_VP, ctypes.c_int, ctypes.POINTER(_VP)]),
    "jsmpeg_b200_batch_read_macroblocks": (ctypes.c_int, [_VP, ctypes.c_int, _VP]),
    "jsmpeg_b200_batch_get_host_macroblocks": (ctypes.c_int, [_VP, ctypes.c_int, ctypes.POINTER(_VP)]),
    "jsmpeg_b200_batch_get_accumulated": (ctypes.c_int, [_VP, ctypes.c_int, ctypes.POINTER(_VP)]),
    "jsmpeg_b200_batch_read_accumulated": (ctypes.c_int, [_VP, ctypes.c_int, _VP]),
    "jsmpeg_b200_batch_get_residuals": (ctypes.c_int, [_VP, ctypes.c_int, ctypes.POINTER(_VP)]),
    "jsmpeg_b200_batch_read_residuals": (ctypes.c_int, [_VP, ctypes.c_int, _VP]),
    "jsmpeg_b200_batch_decode_frames": (ctypes.c_long, [_VP, ctypes.c_int, ctypes.c_int, _VP, _VP, _VP, _VP,
                                                        ctypes.POINTER(Frame), _VP]),
    "jsmpeg_b200_batch_decode_frames_into": (ctypes.c_long, [_VP, ctypes.c_int, ctypes.c_int, ctypes.POINTER(FrameDst),
                                                             ctypes.POINTER(Frame), _VP]),
    "jsmpeg_b200_batch_decode_frames_display": (ctypes.c_long, [_VP, ctypes.c_int, ctypes.c_int, ctypes.POINTER(FrameDst),
                                                                ctypes.POINTER(Frame), _VP]),
    "jsmpeg_b200_batch_flush_frames": (ctypes.c_long, [_VP, ctypes.POINTER(FrameDst), ctypes.POINTER(Frame), _VP]),
    "jsmpeg_b200_batch_last_picture": (ctypes.c_int, [_VP, ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]),
    "jsmpeg_b200_batch_intra_index": (ctypes.c_long, [_VP, ctypes.c_int, _VP, _VP, _VP, ctypes.c_long]),
    "jsmpeg_b200_batch_decode_intra": (ctypes.c_long, [_VP, ctypes.c_int, _VP, _VP, _VP, _VP, ctypes.c_int, _VP, _VP]),
    "jsmpeg_b200_batch_picture_index": (ctypes.c_long, [_VP, ctypes.c_int, _VP, _VP, _VP, _VP, _VP, ctypes.c_long]),
    "jsmpeg_b200_batch_decode_pictures": (ctypes.c_long, [_VP, ctypes.c_int, _VP, _VP, _VP, _VP, ctypes.c_int, _VP, _VP, _VP]),
    "jsmpeg_b200_batch_macroblock_index": (ctypes.c_long, [_VP, ctypes.c_int, _VP, _VP, _VP, _VP, ctypes.c_long]),
    "jsmpeg_b200_batch_decode_macroblocks": (ctypes.c_long, [_VP, ctypes.c_int, _VP, _VP, _VP, _VP, _VP]),
    "jsmpeg_b200_batch_decode_coefficients": (ctypes.c_long, [_VP, ctypes.c_int, _VP, _VP, _VP, _VP, _VP, _VP]),
    "jsmpeg_b200_batch_decode_residuals": (ctypes.c_long, [_VP, ctypes.c_int, _VP, _VP, _VP, _VP, _VP, _VP]),
    "jsmpeg_b200_batch_decode_accumulated": (ctypes.c_long, [_VP, ctypes.c_int, _VP, _VP, _VP, _VP, _VP, _VP]),
    "jsmpeg_b200_batch_seek_pictures": (ctypes.c_long, [_VP, ctypes.c_int, _VP, _VP, ctypes.c_int, _VP, _VP, _VP]),
    "jsmpeg_b200_batch_get_stats": (None, [_VP, ctypes.POINTER(Stats)]),
    "jsmpeg_b200_batch_reset_stats": (None, [_VP]),
    "jsmpeg_b200_debug_parse_picture": (ctypes.c_int, [_VP, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_int, ctypes.c_int,
                                                       _VP, _VP, _VP, _VP, _VP]),
    "jsmpeg_b200_debug_reconstruct": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "jsmpeg_b200_debug_read_es": (ctypes.c_long, [_VP, ctypes.c_int, _VP, ctypes.c_size_t]),
    "jsmpeg_b200_set_default_device": (None, [ctypes.c_int]),
    "jsmpeg_b200_batch_last_error": (ctypes.c_char_p, [_VP]),
    "jsmpeg_b200_batch_set_option": (ctypes.c_int, [_VP, ctypes.c_char_p, ctypes.c_int]),
    "jsmpeg_b200_decoder_last_error": (ctypes.c_char_p, [_VP]),
    "jsmpeg_b200_decoder_set_option": (ctypes.c_int, [_VP, ctypes.c_char_p, ctypes.c_int]),
    "jsmpeg_b200_decoder_last_picture": (ctypes.c_int, [_VP, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]),
    "jsmpeg_b200_decoder_get_macroblocks": (_VP, [_VP]),
    "jsmpeg_b200_bind_host_to_device": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(ctypes.c_int)]),
    "jsmpeg_b200_version": (ctypes.c_char_p, []),
}


def planes_view(t, info):
    """Y [coded_h, coded_w], Cr and Cb [coded_h / 2, coded_w / 2] as views of a decode_intra planes tensor (or of a
    decode_residuals tensor, which has the same layout); `info` is the stream's BatchDecoder.stream_info."""
    cw, ch = (info["width"] + 15) // 16 * 16, (info["height"] + 15) // 16 * 16
    n = cw * ch
    return t[:n].view(ch, cw), t[n:n + n // 4].view(ch // 2, cw // 2), t[n + n // 4:n + n // 2].view(ch // 2, cw // 2)


MACROBLOCK_BYTES = 16  # sizeof(jsmpeg_b200_macroblock_t)
MB_PRESENT, MB_INTRA, MB_SKIPPED, MB_BACKWARD, MB_FORWARD = 0x01, 0x02, 0x04, 0x08, 0x10  # JSMPEG_B200_MB_*


def macroblocks_view(t):
    """Named views of a decode_macroblocks tensor [mb_height, mb_width, 16]: "forward" and "backward" int16 [h, w, 2]
    (x, y in luma half-pel units), "flags" (MB_*), "cbp" and "qscale" uint8 [h, w]."""
    import torch
    as16 = t.view(torch.int16)  # [h, w, 8]: fwd_x, fwd_y, bwd_x, bwd_y, ...
    return {"forward": as16[..., 0:2], "backward": as16[..., 2:4], "flags": t[..., 8], "cbp": t[..., 9],
            "qscale": t[..., 10]}


ACCUMULATED_BYTES = 8  # sizeof(jsmpeg_b200_accumulated_t)


def accumulated_view(t, info):
    """Per plane (Y, Cr, Cb) of a decode_accumulated map [coded_size * 3 // 2, 4]: {"motion": int16 [h, w, 2] (dx, dy in
    half-sample units of the plane), "residual": [h, w], "back": [h, w] (-1: untraced)}; `info` as in planes_view."""
    cw, ch = (info["width"] + 15) // 16 * 16, (info["height"] + 15) // 16 * 16
    n = cw * ch
    planes = (t[:n].view(ch, cw, 4), t[n:n + n // 4].view(ch // 2, cw // 2, 4), t[n + n // 4:n + n // 2].view(ch // 2, cw // 2, 4))
    return tuple({"motion": p[..., 0:2], "residual": p[..., 2], "back": p[..., 3]} for p in planes)


def bind_batch_abi(lib):
    for name, (res, args) in _BATCH_ABI.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


class BatchDecoder:
    """``n_streams`` independent MPEG-1 video decoders on one GPU."""

    def __init__(self, n_streams, device=0, max_slots=0, lib=None, decode_b=None, slice_walk=None,
                 conceal=None):
        from . import capi
        self.lib = lib if lib is not None else capi.product_library()
        self.n_streams = n_streams
        self.device = device
        self._pes = [[] for _ in range(n_streams)]  # per stream: every (payload byte offset, pts seconds) write_ts/write_ps returned
        self.last_intra_info = []  # per request of the last decode_intra: {"n_present", "error"} (picture_info_t)
        self.last_pictures_info = []  # per request of the last decode_pictures: {"status", "n_present", "error"}
        self.last_macroblocks_info = []  # per request of the last decode_macroblocks: {"n_present", "error"}
        self.last_coefficients_info = []  # per request of the last decode_coefficients: {"n_present", "error"}
        self.last_residuals_info = []  # per request of the last decode_residuals: {"n_present", "error"}
        self.last_accumulated_info = []  # per request of the last decode_accumulated: {"status", "n_present", "error"}
        self.last_seek_info = []  # per request of the last seek_pictures: {"status", "n_present", "error"}
        self.last_frames_batch = {}  # per kind of the last decode_frames: its [S, n, ...] tensor when the streams share one geometry
        self.handle = self.lib.jsmpeg_b200_batch_create(n_streams, device, max_slots)
        err = self.lib.jsmpeg_b200_batch_last_error(self.handle)
        if err:  # no usable CUDA device: the C ABI answers "false" for ever; the Python host says so loudly
            self.close()
            raise RuntimeError(err.decode(errors="replace"))
        if slice_walk is not None:  # I/P pictures of many slices: one lane per slice (same records, another walk kernel)
            self.set_option("slice_walk", slice_walk)
        if decode_b is not None:  # the B-picture extension (the reference skips B pictures, and so does the default)
            self.set_option("decode_b", decode_b)
        if conceal is not None:  # the macroblocks a damaged picture lacks are copied from its forward reference
            self.set_option("conceal", conceal)

    def close(self):
        if self.handle:
            self.lib.jsmpeg_b200_batch_destroy(self.handle)
            self.handle = None

    __del__ = close

    def set_option(self, name, value):
        if self.lib.jsmpeg_b200_batch_set_option(self.handle, name.encode(), int(value)) != 0:
            raise ValueError(f"unknown option {name!r}")

    def last_error(self):
        err = self.lib.jsmpeg_b200_batch_last_error(self.handle)
        return err.decode(errors="replace") if err else None

    def write(self, stream, data):
        """Two-phase write of the reference ABI (get_write_ptr / memcpy / did_write)."""
        data = bytes(data) if not isinstance(data, bytes) else data
        ptr = self.lib.jsmpeg_b200_batch_get_write_ptr(self.handle, stream, len(data))
        ctypes.memmove(ptr, data, len(data))
        self.lib.jsmpeg_b200_batch_did_write(self.handle, stream, len(data))

    def _write_one(self, name, capacity, refused, stream, data, stream_id):
        """write_ts / write_ps through the C call `name`, with room for capacity(len(data)) PES entries.  A -2 raises
        ValueError(refused) where the format refuses a stream id, any other failure RuntimeError."""
        data = bytes(data)
        n_max = capacity(len(data))
        pts = np.zeros(n_max, np.uint64)
        off = np.zeros(n_max, np.uint32)
        n = ctypes.c_int()
        total = getattr(self.lib, name)(self.handle, stream, data, len(data), stream_id, pts.ctypes.data, off.ctypes.data,
                                        n_max, ctypes.byref(n))
        if total == -2 and refused:
            raise ValueError(refused.format(stream_id=stream_id))
        if total < 0:
            raise RuntimeError(self.last_error() or f"{name} failed")
        table = [(int(off[i]), float(pts[i]) / 90000.0) for i in range(n.value)]
        self._pes[stream] += table
        return total, table

    def _write_many(self, name, capacity, refused, writes):
        """write_ts_many / write_ps_many through the C call `name`; a -2 raises ValueError(refused)."""
        writes = [(w[0], bytes(w[1]), w[2] if len(w) > 2 else 0xE0) for w in writes]
        n = len(writes)
        streams = np.array([w[0] for w in writes], np.int32)
        bufs = [w[1] for w in writes]
        ptrs = (ctypes.c_char_p * max(n, 1))(*bufs)
        sizes = np.array([len(b) for b in bufs], np.uint64)
        sids = np.array([w[2] for w in writes], np.int32)
        appended = np.zeros(n, np.int64)
        n_pes = np.zeros(n, np.int32)
        n_max = sum(capacity(len(b)) for b in bufs)
        pts = np.zeros(max(n_max, 1), np.uint64)
        off = np.zeros(max(n_max, 1), np.uint32)
        total = getattr(self.lib, name)(self.handle, n, streams.ctypes.data, ctypes.addressof(ptrs), sizes.ctypes.data,
                                        sids.ctypes.data, appended.ctypes.data, pts.ctypes.data, off.ctypes.data, n_max,
                                        n_pes.ctypes.data)
        if total == -2:
            raise ValueError(refused)
        if total < 0:
            raise RuntimeError(self.last_error() or f"{name} failed")
        out, k = [], 0
        for (stream, _, _), a, m in zip(writes, appended, n_pes):
            table = [(int(off[k + j]), float(pts[k + j]) / 90000.0) for j in range(m)]
            k += m
            self._pes[stream] += table
            out.append((int(a), table))
        return out

    @staticmethod
    def _ts_pes_capacity(n_bytes):
        """PES starts a TS write of n_bytes can report: one per packet of the bytes and of what the stream's last write
        left over (up to 188 x 6 - 1 bytes of a pending resync)."""
        return (n_bytes + 188 * 6 - 1) // 188 + 1

    def write_ts(self, stream, ts_bytes, stream_id=0xE0):
        """MPEG-TS in, demultiplexed on the GPU (any chunking, resyncs like src/ts.js).  Returns (ES bytes
        appended, [(payload byte offset, pts seconds), ...] per PES packet of `stream_id` that starts in it)."""
        return self._write_one("jsmpeg_b200_batch_write_ts", self._ts_pes_capacity, None, stream, ts_bytes, stream_id)

    def write_ts_many(self, writes):
        """MPEG-TS of many streams in one GPU pass: `writes` is an iterable of (stream, bytes) or (stream, bytes,
        stream_id), each stream at most once.  Returns one (ES bytes appended, [(payload byte offset, pts seconds),
        ...]) per write, what write_ts returns for it."""
        return self._write_many("jsmpeg_b200_batch_write_ts_many", self._ts_pes_capacity,
                                "write_ts_many: a stream out of range or named twice, or 4 GiB of input or more", writes)

    @staticmethod
    def _ps_pes_capacity(n_bytes):
        """PES table entries a PS write of n_bytes can report: a table entry needs >= 12 bytes (6 + a 5-byte PTS + 1
        payload byte); the call may also finish items of up to 65,541 bytes that an earlier call left over."""
        return (n_bytes + 65541) // 12 + 1

    def write_ps(self, stream, ps_bytes, stream_id=0xE0):
        """MPEG program stream in (.mpg: ISO 11172-1, .vob: ISO 13818-1), demultiplexed on the GPU (any
        chunking, resyncs at the next pack header).  Returns (ES bytes appended, [(payload byte offset, pts
        seconds), ...] per PES packet of `stream_id` with a PTS in it)."""
        return self._write_one("jsmpeg_b200_batch_write_ps", self._ps_pes_capacity,
                               "stream_id {stream_id:#x} is not a video stream id (0xE0..0xEF)", stream, ps_bytes, stream_id)

    def write_ps_many(self, writes):
        """MPEG program streams of many streams in one GPU pass: `writes` is an iterable of (stream, bytes) or (stream,
        bytes, stream_id), each stream at most once.  Returns one (ES bytes appended, [(payload byte offset, pts
        seconds), ...]) per write, what write_ps returns for it."""
        return self._write_many("jsmpeg_b200_batch_write_ps_many", self._ps_pes_capacity,
                                "write_ps_many: a stream out of range or named twice, a stream id outside 0xE0..0xEF, "
                                "or 4 GiB of input or more", writes)

    def read_es(self, stream):
        """The stream's elementary stream as it is resident in HBM (test hook)."""
        n = self.lib.jsmpeg_b200_debug_read_es(self.handle, stream, None, 0)
        if n < 0:
            raise RuntimeError(self.last_error() or "jsmpeg_b200_debug_read_es failed")
        buf = ctypes.create_string_buffer(max(n, 1))
        self.lib.jsmpeg_b200_debug_read_es(self.handle, stream, buf, n)
        return buf.raw[:n]

    def get_index(self, stream):
        return self.lib.jsmpeg_b200_batch_get_index(self.handle, stream)

    def set_index(self, stream, index):
        self.lib.jsmpeg_b200_batch_set_index(self.handle, stream, index)

    def stream_info(self, stream):
        w, h, cs, fr = ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_float()
        has = self.lib.jsmpeg_b200_batch_stream_info(self.handle, stream, w, h, cs, fr)
        return {"has_sequence_header": bool(has), "width": w.value, "height": h.value,
                "coded_size": cs.value, "frame_rate": fr.value}

    def upload(self):
        return self.lib.jsmpeg_b200_batch_upload(self.handle)

    def rewind(self):
        self.lib.jsmpeg_b200_batch_rewind(self.handle)

    def reset(self):
        self.lib.jsmpeg_b200_batch_reset(self.handle)
        self._pes = [[] for _ in range(self.n_streams)]

    def decode(self, n_pictures=1, flags=OUT_DEVICE):
        return self.lib.jsmpeg_b200_batch_decode(self.handle, n_pictures, flags)

    _FRAME_KINDS = ("planes", "rgba", "residuals", "macroblocks", "coefficients", "accumulated")

    def decode_frames(self, n_pictures, flags=OUT_DEVICE, planes=True, rgba=False, residuals=False, macroblocks=False,
                      coefficients=False, accumulated=False, display_order=False):
        """decode(n_pictures, flags) that also hands back every picture it reconstructs (include/jsmpeg_b200.h,
        jsmpeg_b200_batch_decode_frames): frame j of a stream is the j-th picture the call reconstructs for it (I and P,
        and B under decode_b; skipped pictures have none), in coded order.  Returns per stream a dict with "n_frames",
        "info" (per frame {"byte_pos", "type", "temporal_reference", "n_present", "error", "pts"}, pts as in
        intra_index) and each kind asked for, a CUDA tensor cut to n_frames: "planes" uint8 [F, coded_size * 3 // 2]
        (see planes_view), "rgba" uint8 [F, height, width, 4], "residuals" int16 [F, coded_size * 3 // 2],
        "macroblocks" uint8 [F, mb_height, mb_width, 16] (see macroblocks_view); None for a stream without a sequence
        header.  When every stream has one and all share one geometry, each kind is allocated as one [S, n_pictures,
        ...] tensor (last_frames_batch[kind]; RGBA only where a stream's n_pictures images are a multiple of 16 bytes) and
        the per-stream tensors are views of it: a clip batch without a gather.
        coefficients=True and accumulated=True (jsmpeg_b200_batch_decode_frames_into) add "coefficients" int16 [F,
        mb_height, mb_width, 6, 8, 8] (as decode_coefficients) and "accumulated" int16 [F, coded_size * 3 // 2, 4] (see
        accumulated_view; a B frame's is all untraced); accumulated=True needs OUT_ACCUMULATED in `flags`.
        display_order=True (jsmpeg_b200_batch_decode_frames_display) hands the frames over in presentation order: frame
        j of a stream is the j-th picture the call presents (a B picture at once, an I/P picture when the next I/P
        picture arrives, one held by an earlier call included; see flush_frames), "info" in that order, each tensor
        allocated for n_pictures + 1 frames ([S, n_pictures + 1, ...] in last_frames_batch) and cut to n_frames."""
        n = int(n_pictures)
        if n < 0:
            raise ValueError("n_pictures must be >= 0")
        if accumulated and not int(flags) & OUT_ACCUMULATED:
            raise ValueError("accumulated frames need OUT_ACCUMULATED in flags")
        want = {"planes": planes, "rgba": rgba, "residuals": residuals, "macroblocks": macroblocks,
                "coefficients": coefficients, "accumulated": accumulated}
        cap = n + 1 if display_order else n  # frames per stream
        full, dst, into = self._frame_destinations(cap, want)
        info_out = (Frame * max(self.n_streams * cap, 1))()
        n_frames = (ctypes.c_int32 * max(self.n_streams, 1))()
        if display_order:
            got = self.lib.jsmpeg_b200_batch_decode_frames_display(self.handle, n, int(flags), ctypes.byref(into), info_out, n_frames)
        elif coefficients or accumulated:
            got = self.lib.jsmpeg_b200_batch_decode_frames_into(self.handle, n, int(flags), ctypes.byref(into), info_out, n_frames)
        else:
            got = self.lib.jsmpeg_b200_batch_decode_frames(self.handle, n, int(flags), dst.get("planes"), dst.get("rgba"),
                                                           dst.get("residuals"), dst.get("macroblocks"), info_out, n_frames)
        if got == -2:
            raise ValueError("decode_frames refused its arguments")
        if got < 0:
            raise RuntimeError(self.last_error() or "jsmpeg_b200_batch_decode_frames failed")
        return self._frames_out(full, info_out, n_frames, cap)

    def flush_frames(self, planes=True, rgba=False, residuals=False, macroblocks=False, coefficients=False, accumulated=False):
        """End of clip for decode_frames(display_order=True) (jsmpeg_b200_batch_flush_frames): every stream's held I/P
        picture, as decode_frames' result of one frame (n_frames 0 or 1), and the holds released.  A stream that holds a
        picture must have been asked for every kind asked for here (ValueError otherwise, with nothing changed)."""
        want = {"planes": planes, "rgba": rgba, "residuals": residuals, "macroblocks": macroblocks,
                "coefficients": coefficients, "accumulated": accumulated}
        full, _, into = self._frame_destinations(1, want)
        info_out = (Frame * max(self.n_streams, 1))()
        n_frames = (ctypes.c_int32 * max(self.n_streams, 1))()
        got = self.lib.jsmpeg_b200_batch_flush_frames(self.handle, ctypes.byref(into), info_out, n_frames)
        if got == -2:
            raise ValueError("flush_frames refused its arguments")
        if got < 0:
            raise RuntimeError(self.last_error() or "jsmpeg_b200_batch_flush_frames failed")
        return self._frames_out(full, info_out, n_frames, 1)

    def _frame_destinations(self, n, want):
        """Room for n frames per stream of each kind in `want` (decode_frames' tensor rules): the tensors per kind, the
        per-stream pointer arrays per kind, and a FrameDst over them"""
        import torch
        dev = torch.device("cuda", self.device)
        infos = [self.stream_info(s) for s in range(self.n_streams)]

        def shape(kind, info):
            cs, w, h = info["coded_size"], info["width"], info["height"]
            return {"planes": (cs * 3 // 2,), "rgba": (h, w, 4), "residuals": (cs * 3 // 2,),
                    "macroblocks": ((h + 15) // 16, (w + 15) // 16, MACROBLOCK_BYTES),
                    "coefficients": ((h + 15) // 16, (w + 15) // 16, 6, 8, 8), "accumulated": (cs * 3 // 2, 4)}[kind]

        dtype = {"planes": torch.uint8, "rgba": torch.uint8, "residuals": torch.int16, "macroblocks": torch.uint8,
                 "coefficients": torch.int16, "accumulated": torch.int16}
        geometries = {(i["width"], i["height"]) for i in infos}
        shared = all(i["has_sequence_header"] for i in infos) and len(geometries) == 1
        full, self.last_frames_batch = {}, {}
        for kind in self._FRAME_KINDS:
            if not want[kind]:
                continue
            slab = n * int(np.prod(shape(kind, infos[0]))) * dtype[kind].itemsize
            if shared and slab % 16 == 0:  # (every stream's frame 0 16-byte aligned)
                self.last_frames_batch[kind] = t = torch.empty((self.n_streams, n, *shape(kind, infos[0])), dtype=dtype[kind], device=dev)
                full[kind] = list(t.unbind(0))
            else:  # (torch's allocations are 512-byte aligned)
                full[kind] = [torch.empty((n, *shape(kind, i)), dtype=dtype[kind], device=dev) if i["has_sequence_header"] else None
                              for i in infos]
        S = max(self.n_streams, 1)
        dst = {kind: (_VP * S)(*[t.data_ptr() if t is not None and n else None for t in full[kind]]) for kind in full}
        if full:
            torch.cuda.current_stream(dev).synchronize()  # the allocations are the caller's stream's; the call uses its own
        into = FrameDst(*[ctypes.addressof(dst[k]) if k in dst else None for k in self._FRAME_KINDS])
        return full, dst, into

    def _frames_out(self, full, info_out, n_frames, n):
        """Per stream: decode_frames' dict of the frames the call wrote (info rows n apart)"""
        out = []
        for s in range(self.n_streams):
            f = n_frames[s]
            rows = [info_out[s * n + j] for j in range(f)]
            d = {"n_frames": f, "info": [{"byte_pos": r.byte_pos, "type": r.picture_type, "temporal_reference": r.temporal_reference,
                                          "n_present": r.n_present, "error": r.error, "pts": self._pts(s, r.byte_pos)} for r in rows]}
            for kind in full:
                t = full[kind][s]
                d[kind] = None if t is None else t[:f]
            out.append(d)
        return out

    def device_planes(self, stream):
        y, cr, cb = _VP(), _VP(), _VP()
        if self.lib.jsmpeg_b200_batch_get_planes(self.handle, stream, y, cr, cb) != 0:
            return None
        return y.value, cr.value, cb.value

    def read_planes(self, stream):
        n = self.stream_info(stream)["coded_size"]
        y = np.empty(n, np.uint8)
        cr = np.empty(n >> 2, np.uint8)
        cb = np.empty(n >> 2, np.uint8)
        rc = self.lib.jsmpeg_b200_batch_read_planes(self.handle, stream, y.ctypes.data, cr.ctypes.data, cb.ctypes.data)
        if rc != 0:
            raise RuntimeError("stream has no sequence header yet")
        return y, cr, cb

    def host_planes(self, stream):
        n = self.stream_info(stream)["coded_size"]
        y, cr, cb = _VP(), _VP(), _VP()
        if self.lib.jsmpeg_b200_batch_get_host_planes(self.handle, stream, y, cr, cb) != 0:
            return None

        def view(p, size):
            return np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(ctypes.c_uint8)), shape=(size,))

        return view(y, n), view(cr, n >> 2), view(cb, n >> 2)

    def _entries_shape(self, stream):
        """(mb_height, mb_width, 16) of the stream's macroblock entries; ValueError unless the stream is in range and
        has a sequence header."""
        info = self._request_stream_info(stream)
        return (info["height"] + 15) // 16, (info["width"] + 15) // 16, MACROBLOCK_BYTES

    def _entries_ptr(self, fn, stream):
        ptr = _VP()
        if fn(self.handle, stream, ctypes.byref(ptr)) != 0:
            raise RuntimeError(self.last_error() or f"{fn.__name__} failed")
        return ptr.value

    def device_macroblocks(self, stream):
        """The stream's macroblock entries (decode / seek_pictures with OUT_MACROBLOCKS, include/jsmpeg_b200.h): a
        torch.uint8 CUDA view [mb_height, mb_width, 16] of the library's buffer beside the planes of the picture
        device_planes gives (see macroblocks_view).  Borrowed: valid until the next decode / seek; clone to keep it."""
        import torch
        shape = self._entries_shape(stream)
        ptr = self._entries_ptr(self.lib.jsmpeg_b200_batch_get_macroblocks, stream)

        class _Entries:  # (zero copy: torch wraps memory that exposes __cuda_array_interface__)
            __cuda_array_interface__ = {"data": (ptr, False), "shape": shape, "typestr": "|u1", "version": 2}

        return torch.as_tensor(_Entries(), device=torch.device("cuda", self.device))

    def read_macroblocks(self, stream):
        """A numpy copy [mb_height, mb_width, 16] of the entries device_macroblocks views (synchronous)."""
        out = np.empty(self._entries_shape(stream), np.uint8)
        if self.lib.jsmpeg_b200_batch_read_macroblocks(self.handle, stream, out.ctypes.data) != 0:
            raise RuntimeError(self.last_error() or "jsmpeg_b200_batch_read_macroblocks failed")
        return out

    def host_macroblocks(self, stream):
        """Under OUT_HOST | OUT_MACROBLOCKS: a numpy view [mb_height, mb_width, 16] of the pinned entries of the
        picture host_planes gives (the same host-ring slot).  Borrowed like host_planes."""
        shape = self._entries_shape(stream)
        ptr = self._entries_ptr(self.lib.jsmpeg_b200_batch_get_host_macroblocks, stream)
        return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_uint8)), shape=shape)

    def _map_shape(self, stream):
        """(coded_size * 3 // 2, 4) of the stream's accumulated map; ValueError unless the stream is in range and has a
        sequence header."""
        return self._request_stream_info(stream)["coded_size"] * 3 // 2, 4

    def device_accumulated(self, stream):
        """The accumulated map of the stream's newest I/P picture (decode / seek_pictures with OUT_ACCUMULATED,
        include/jsmpeg_b200.h): a torch.int16 CUDA view [coded_size * 3 // 2, 4] of the library's map (see
        accumulated_view), all untraced where no call with the flag wrote it.  Borrowed: valid until the next decode /
        seek; clone to keep it."""
        import torch
        shape = self._map_shape(stream)
        ptr = self._entries_ptr(self.lib.jsmpeg_b200_batch_get_accumulated, stream)

        class _Map:  # (zero copy, as device_macroblocks)
            __cuda_array_interface__ = {"data": (ptr, False), "shape": shape, "typestr": "<i2", "version": 2}

        return torch.as_tensor(_Map(), device=torch.device("cuda", self.device))

    def read_accumulated(self, stream):
        """A numpy copy int16 [coded_size * 3 // 2, 4] of the map device_accumulated views (synchronous)."""
        out = np.empty(self._map_shape(stream), np.int16)
        if self.lib.jsmpeg_b200_batch_read_accumulated(self.handle, stream, out.ctypes.data) != 0:
            raise RuntimeError(self.last_error() or "jsmpeg_b200_batch_read_accumulated failed")
        return out

    def _residuals_shape(self, stream):
        """(coded_size * 3 // 2,) of the stream's residual; ValueError unless the stream is in range and has a sequence
        header."""
        return (self._request_stream_info(stream)["coded_size"] * 3 // 2,)

    def device_residuals(self, stream):
        """The residual of the picture device_planes gives (decode / seek_pictures with OUT_RESIDUALS,
        include/jsmpeg_b200.h): a torch.int16 CUDA view [coded_size * 3 // 2] of the library's buffer in
        decode_residuals' layout (planes_view splits it into Y, Cr, Cb), 0 where no call with the flag wrote it.
        Borrowed: valid until the next decode / seek; clone to keep it."""
        import torch
        shape = self._residuals_shape(stream)
        ptr = self._entries_ptr(self.lib.jsmpeg_b200_batch_get_residuals, stream)

        class _Residual:  # (zero copy, as device_macroblocks)
            __cuda_array_interface__ = {"data": (ptr, False), "shape": shape, "typestr": "<i2", "version": 2}

        return torch.as_tensor(_Residual(), device=torch.device("cuda", self.device))

    def read_residuals(self, stream):
        """A numpy copy int16 [coded_size * 3 // 2] of the residual device_residuals views (synchronous)."""
        out = np.empty(self._residuals_shape(stream), np.int16)
        if self.lib.jsmpeg_b200_batch_read_residuals(self.handle, stream, out.ctypes.data) != 0:
            raise RuntimeError(self.last_error() or "jsmpeg_b200_batch_read_residuals failed")
        return out

    def read_rgba(self, stream):
        info = self.stream_info(stream)
        out = np.empty((info["height"], info["width"], 4), np.uint8)
        if self.lib.jsmpeg_b200_batch_read_rgba(self.handle, stream, out.ctypes.data) != 0:
            raise RuntimeError("no RGBA picture (decode with OUT_RGBA first)")
        return out

    def intra_index(self, stream):
        """The I pictures of `stream` that decode_intra can decode now (include/jsmpeg_b200.h): one dict per picture,
        {"picture": k, "byte_pos", "temporal_reference", "pts"}.  `pts` (seconds) is that of the last PES packet
        write_ts / write_ps reported at or before the picture's start code (src/decoder.js:36-47), or None."""
        return self._index(self.lib.jsmpeg_b200_batch_intra_index, stream,
                           [("picture", np.uint32), ("byte_pos", np.uint32), ("temporal_reference", np.int32)])

    def _index(self, fn, stream, fields):
        """The index `fn` (jsmpeg_b200_batch_*_index) of `stream`: one dict per picture with the (key, dtype) `fields`
        in the order of fn's output arrays ("picture" and "byte_pos" first), then "pts"."""
        n = fn(self.handle, stream, *[None] * len(fields), 0)
        if n == -2:
            raise ValueError(f"stream {stream} out of range")
        if n < 0:
            raise RuntimeError(self.last_error() or f"{fn.__name__} failed")
        arrays = [np.zeros(n, dtype) for _, dtype in fields]
        n = fn(self.handle, stream, *[a.ctypes.data for a in arrays], n)
        return [{**{key: int(a[i]) for (key, _), a in zip(fields, arrays)}, "pts": self._pts(stream, int(arrays[1][i]))}
                for i in range(min(n, len(arrays[0])))]

    def _pts(self, stream, byte_pos):
        """PTS (seconds) of the last PES packet write_ts / write_ps reported at or before `byte_pos`, or None."""
        pes = self._pes[stream]
        j = bisect.bisect_right([o for o, _ in pes], byte_pos) - 1
        return pes[j][1] if j >= 0 else None

    def picture_index(self, stream):
        """The pictures of `stream` that decode_pictures can decode now (include/jsmpeg_b200.h): one dict per picture,
        {"picture": k, "byte_pos", "type" (picture_coding_type), "temporal_reference", "chain_start", "pts"}; `pts`
        as in intra_index.  Follows the decode_b option's current value."""
        return self._index(self.lib.jsmpeg_b200_batch_picture_index, stream,
                           [("picture", np.uint32), ("byte_pos", np.uint32), ("type", np.int32),
                            ("temporal_reference", np.int32), ("chain_start", np.uint32)])

    def decode_pictures(self, requests, rgba=False):
        """Decode pictures listed by picture_index, of any streams, in one call: `requests` is an iterable of (stream,
        picture).  Returns what decode_intra returns; last_pictures_info gets {"status", "n_present", "error"} per
        request (status 1: decoded; 0: the fresh decoder never reached the picture, whose planes are then 0)."""
        reqs = [(int(s), int(p)) for s, p in requests]
        status = (ctypes.c_int32 * max(len(reqs), 1))()
        out, n_present, errors = self._decode_requests(self.lib.jsmpeg_b200_batch_decode_pictures, reqs, rgba, [status],
                                                       "a request names a picture that is not in the stream's picture index")
        self.last_pictures_info = [{"status": status[i], "n_present": n_present[i], "error": errors[i]} for i in range(len(reqs))]
        return out

    def decode_intra(self, requests, rgba=False):
        """Decode I pictures listed by intra_index, of any streams, in one call: `requests` is an iterable of (stream,
        picture).  Returns per request a torch.uint8 CUDA tensor of coded_size * 3 // 2 bytes (Y | Cr | Cb, see
        planes_view), or with rgba=True a pair (planes, rgba [height, width, 4])."""
        reqs = [(int(s), int(p)) for s, p in requests]
        out, n_present, errors = self._decode_requests(self.lib.jsmpeg_b200_batch_decode_intra, reqs, rgba, [],
                                                       "a request names a picture that is not in the stream's intra index")
        self.last_intra_info = [{"n_present": n_present[i], "error": errors[i]} for i in range(len(reqs))]
        return out

    def macroblock_index(self, stream):
        """The pictures of `stream` that decode_macroblocks can describe now (include/jsmpeg_b200.h): one dict per
        picture, {"picture": k, "byte_pos", "type" (picture_coding_type), "temporal_reference", "pts"}; `pts` as in
        intra_index.  B pictures are listed whatever the decode_b option says."""
        return self._index(self.lib.jsmpeg_b200_batch_macroblock_index, stream,
                           [("picture", np.uint32), ("byte_pos", np.uint32), ("type", np.int32),
                            ("temporal_reference", np.int32)])

    def decode_macroblocks(self, requests):
        """Macroblock types and motion vectors of pictures listed by macroblock_index, of any streams, in one call:
        `requests` is an iterable of (stream, picture).  Returns per request a torch.uint8 CUDA tensor [mb_height,
        mb_width, 16] of jsmpeg_b200_macroblock_t entries (see macroblocks_view); last_macroblocks_info gets
        {"n_present", "error"} per request.  The tensors are views of one allocation per picture size (thousands of
        requests cost a few allocations, not thousands)."""
        import torch
        (out,), self.last_macroblocks_info = self._export_requests(
            self.lib.jsmpeg_b200_batch_decode_macroblocks, requests,
            [(lambda h, w: (h, w, MACROBLOCK_BYTES), torch.uint8)], [], _NOT_IN_MACROBLOCK_INDEX)
        return out

    def decode_coefficients(self, requests, macroblocks=False):
        """Dequantised DCT coefficients of pictures listed by macroblock_index, of any streams, in one call: `requests`
        is an iterable of (stream, picture).  Returns per request a torch.int16 CUDA tensor [mb_height, mb_width, 6, 8,
        8]: per macroblock the blocks 0-3 luma, 4 Cb, 5 Cr, each in raster order, as the inverse transform consumes
        them (include/jsmpeg_b200.h); 0 for uncoded blocks and absent macroblocks.  A DC image is c[..., 0, 0] (8 x the
        DC of intra blocks).  With macroblocks=True each item is a pair (coefficients, entries), entries as
        decode_macroblocks returns them, from the same walk.  last_coefficients_info gets {"n_present", "error"} per
        request.  The tensors are views of one allocation per picture size."""
        import torch
        entries = (lambda h, w: (h, w, MACROBLOCK_BYTES), torch.uint8) if macroblocks else None
        (coefs, entries), self.last_coefficients_info = self._export_requests(
            self.lib.jsmpeg_b200_batch_decode_coefficients, requests,
            [(lambda h, w: (h, w, 6, 8, 8), torch.int16), entries], [], _NOT_IN_MACROBLOCK_INDEX)
        return list(zip(coefs, entries)) if macroblocks else coefs

    def decode_residuals(self, requests, macroblocks=False):
        """Pixel-domain residuals of pictures listed by macroblock_index, of any streams, in one call: `requests` is an
        iterable of (stream, picture).  Returns per request a flat torch.int16 CUDA tensor of coded_size * 3 // 2 values
        in the planes' layout (Y | Cr | Cb, see planes_view): every 8 x 8 block the reference's integer inverse
        transform of what decode_coefficients gives for it (include/jsmpeg_b200.h), 0 for uncoded blocks and absent
        macroblocks -- what stage 2 adds to the prediction, or for an intra macroblock clamps.  With macroblocks=True
        each item is a pair (residual, entries), entries as decode_macroblocks returns them, from the same walk.
        last_residuals_info gets {"n_present", "error"} per request.  The tensors are views of one allocation per
        picture size."""
        import torch
        entries = (lambda h, w: (h, w, MACROBLOCK_BYTES), torch.uint8) if macroblocks else None
        (res, entries), self.last_residuals_info = self._export_requests(
            self.lib.jsmpeg_b200_batch_decode_residuals, requests,
            [(lambda h, w: (h * w * 384,), torch.int16), entries], [], _NOT_IN_MACROBLOCK_INDEX)
        return list(zip(res, entries)) if macroblocks else res

    def decode_accumulated(self, requests):
        """Accumulated motion and residuals of I and P pictures listed by picture_index (type 1 or 2), of any streams,
        in one call: `requests` is an iterable of (stream, picture).  Returns per request a torch.int16 CUDA tensor
        [coded_size * 3 // 2, 4] in the planes' layout (see accumulated_view): per sample (dx, dy, residual, back), the
        sample traced through the reference chain to its key picture (include/jsmpeg_b200.h).  B pictures between
        references are skipped, whatever the decode_b option says.  last_accumulated_info gets {"status",
        "n_present", "error"} per request (status 0: the fresh decoder never reached the picture, whose samples are
        then all untraced).  The tensors are views of one allocation per picture size."""
        import torch
        reqs = [(int(s), int(p)) for s, p in requests]
        status = (ctypes.c_int32 * max(len(reqs), 1))()
        (maps,), info = self._export_requests(
            self.lib.jsmpeg_b200_batch_decode_accumulated, reqs, [(lambda h, w: (h * w * 384, 4), torch.int16)],
            [status], "a request names a picture that is not an I or P picture of the stream's picture index")
        self.last_accumulated_info = [{"status": status[i], **row} for i, row in enumerate(info)]
        return maps

    def seek_pictures(self, requests, flags=OUT_DEVICE):
        """Move decode() of chosen streams to pictures listed by picture_index, in one call: `requests` is an iterable of
        (stream, picture), each stream at most once.  Afterwards each named stream is where decode() is right after
        consuming that picture (include/jsmpeg_b200.h): bit index, planes -- under `flags` (OUT_HOST, OUT_RGBA, as for
        decode) also the host ring and RGBA -- reference sets and last_picture; the next decode() goes on from there.
        Streams not named are left alone.  Returns the number of requests; last_seek_info gets {"status",
        "n_present", "error"} per request (status 1: the picture was consumed; 0: the fresh decoder never reached it,
        and the stream is where that decoder stopped)."""
        reqs = [(int(s), int(p)) for s, p in requests]
        n = len(reqs)
        streams, pictures, n_present, errors = self._request_arrays(reqs)
        status = (ctypes.c_int32 * max(n, 1))()
        got = self.lib.jsmpeg_b200_batch_seek_pictures(self.handle, n, streams, pictures, int(flags), status, n_present, errors)
        if got == -2:
            raise ValueError("a request names a stream twice, or a picture that is not in the stream's picture index")
        if got < 0:
            raise RuntimeError(self.last_error() or "jsmpeg_b200_batch_seek_pictures failed")
        self.last_seek_info = [{"status": status[i], "n_present": n_present[i], "error": errors[i]} for i in range(n)]
        return got

    def _per_picture_views(self, reqs, shape, dtype):
        """Per (stream, picture) request a CUDA tensor of shape shape(mb_height, mb_width) and `dtype`, the views of one
        allocation per picture size (thousands of requests cost a few allocations, not thousands).  A view starts a
        whole number of pictures into its allocation: with 16 * k bytes per macroblock it is 16-byte aligned."""
        import torch
        shapes = {}  # per stream: (mb_height, mb_width)
        for s, _ in reqs:
            if s not in shapes:
                info = self._request_stream_info(s)
                shapes[s] = ((info["height"] + 15) // 16, (info["width"] + 15) // 16)
        by_shape = {}  # per picture size: the requests of that size
        for i, (s, _) in enumerate(reqs):
            by_shape.setdefault(shapes[s], []).append(i)
        out = [None] * len(reqs)
        for mb_shape, idx in by_shape.items():
            views = torch.empty((len(idx), *shape(*mb_shape)), dtype=dtype, device=torch.device("cuda", self.device)).unbind(0)
            for i, t in zip(idx, views):
                out[i] = t
        return out

    @staticmethod
    def _request_arrays(reqs):
        """ctypes arrays of (stream, picture) requests: streams, pictures, and n_present / error outputs."""
        n = max(len(reqs), 1)
        return ((ctypes.c_int * n)(*[s for s, _ in reqs]), (ctypes.c_uint32 * n)(*[p for _, p in reqs]),
                (ctypes.c_int32 * n)(), (ctypes.c_int32 * n)())

    def _request_stream_info(self, s):
        """stream_info of the stream a request names; ValueError unless it is in range and has a sequence header."""
        if not 0 <= s < self.n_streams:
            raise ValueError(f"stream {s} out of range")
        info = self.stream_info(s)
        if not info["has_sequence_header"]:
            raise ValueError(f"stream {s} has no sequence header yet")
        return info

    def _export_requests(self, fn, requests, kinds, extra_out, refused):
        """Allocate the destinations of (stream, picture) `requests` and call `fn` (decode_macroblocks,
        decode_coefficients, decode_residuals or decode_accumulated) with one pointer array per kind, then `extra_out`,
        n_present and error.  `kinds`: per destination array of fn, (shape, dtype) as _per_picture_views takes them, or
        None for an array not given (NULL).  Returns (per kind its tensors or None, [{"n_present", "error"} per
        request])."""
        import torch
        reqs = [(int(s), int(p)) for s, p in requests]
        n = len(reqs)
        out = [self._per_picture_views(reqs, *kind) if kind else None for kind in kinds]
        streams, pictures, n_present, errors = self._request_arrays(reqs)
        dst = [(_VP * max(n, 1))(*[t.data_ptr() for t in views]) if views is not None else None for views in out]
        torch.cuda.current_stream(torch.device("cuda", self.device)).synchronize()  # the allocations are the caller's stream's; the call uses its own
        got = fn(self.handle, n, streams, pictures, *dst, *extra_out, n_present, errors)
        if got == -2:
            raise ValueError(refused)
        if got < 0:
            raise RuntimeError(self.last_error() or f"{fn.__name__} failed")
        return out, [{"n_present": n_present[i], "error": errors[i]} for i in range(n)]

    def _decode_requests(self, fn, reqs, rgba, extra_out, refused):
        """Allocate the destinations of (stream, picture) requests and call `fn` (decode_intra / decode_pictures) with
        `extra_out` before n_present and error.  Returns (outputs, n_present, errors)."""
        import torch
        n = len(reqs)
        dev = torch.device("cuda", self.device)
        planes, images = [], []
        for s, _ in reqs:
            info = self._request_stream_info(s)
            planes.append(torch.empty(info["coded_size"] * 3 // 2, dtype=torch.uint8, device=dev))
            if rgba:
                images.append(torch.empty((info["height"], info["width"], 4), dtype=torch.uint8, device=dev))
        streams = (ctypes.c_int * max(n, 1))(*[s for s, _ in reqs])
        pictures = (ctypes.c_uint32 * max(n, 1))(*[p for _, p in reqs])
        planes_dst = (_VP * max(n, 1))(*[t.data_ptr() for t in planes])
        rgba_dst = (_VP * max(n, 1))(*[t.data_ptr() for t in images]) if rgba else None
        n_present = (ctypes.c_int32 * max(n, 1))()
        errors = (ctypes.c_int32 * max(n, 1))()
        torch.cuda.current_stream(dev).synchronize()  # the allocations are the caller's stream's; the call uses its own
        got = fn(self.handle, n, streams, pictures, planes_dst, rgba_dst, OUT_RGBA if rgba else OUT_DEVICE, *extra_out,
                 n_present, errors)
        if got == -2:
            raise ValueError(refused)
        if got < 0:
            raise RuntimeError(self.last_error() or f"{fn.__name__} failed")
        return (list(zip(planes, images)) if rgba else planes), n_present, errors

    def last_picture(self, stream):
        """(picture_coding_type, temporal_reference) of the picture the stream's last decode() consumed, or None."""
        t, r = ctypes.c_int(), ctypes.c_int()
        if self.lib.jsmpeg_b200_batch_last_picture(self.handle, stream, t, r) != 0:
            return None
        return t.value, r.value

    def stats(self):
        st = Stats()
        self.lib.jsmpeg_b200_batch_get_stats(self.handle, ctypes.byref(st))
        return st.as_dict()

    def reset_stats(self):
        self.lib.jsmpeg_b200_batch_reset_stats(self.handle)
