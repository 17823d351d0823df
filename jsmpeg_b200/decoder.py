"""Host-side mirror of the reference decoder surface.

``MPEG1Video`` keeps the surface of ``JSMpeg.Decoder.MPEG1Video`` / ``MPEG1VideoWASM``
(reference src/decoder.js:3-106, src/mpeg1.js:6-64, src/mpeg1-wasm.js:1-132):

    ctor(options)  keys: videoBufferSize, streaming, decodeFirstFrame, onVideoDecode
                   (+ our extensions `device`: CUDA device index; `decodeBPictures`: decode B pictures, which
                   the reference skips (src/mpeg1.js:181-184), in coded order -- `lastPicture()` tells type and
                   temporal_reference; with `displayOrder` the destination gets them in DISPLAY order: an I/P
                   picture is held back (a copy) until the next I/P picture arrives, `flush()` renders the last;
                   `exportMacroblocks`: `macroblocks()` gives the macroblock types and motion vectors of the
                   picture the last decode() rendered; `concealErrors`: each macroblock a damaged picture lacks
                   gets the co-located samples of the picture it predicts from, instead of keeping what the plane
                   held two pictures ago)
    connect(destination) / destroy()
    bufferGetIndex() / bufferSetIndex(i) / bufferWrite(buffers)
    write(pts, buffers) / seek(time) / decode() -> bool
    currentTime, startTime, decodedTime, canPlay
    width, height, frameRate, codedSize, currentY / currentCr / currentCb
    destination.resize(w, h) on the first sequence header, destination.render(y, cr, cb, False)
    per decoded picture (coded-size planes, src/mpeg1-wasm.js:103-119)

The reference is JavaScript and this image has no JS engine (see INTEGRATION.md), so the host
side is Python over the same C ABI the reference's WASM glue binds (src/mpeg1-wasm.js:29,52-70,
103-116).  All compute happens behind that ABI in CUDA; this file is bookkeeping only
(PTS table, seek) exactly as in src/decoder.js.
"""
from __future__ import annotations

import ctypes
import time

import numpy as np

from . import capi


class MPEG1Video:
    def __init__(self, options=None, lib=None):
        options = dict(options or {})
        # -- Decoder.Base ctor, src/decoder.js:3-17
        self.destination = None
        self.canPlay = False
        self.collectTimestamps = not options.get("streaming", False)
        self.bytesWritten = 0
        self.timestamps = []
        self.timestampIndex = 0
        self.startTime = 0
        self.decodedTime = 0
        # -- MPEG1WASM ctor, src/mpeg1-wasm.js:3-16
        self.onDecodeCallback = options.get("onVideoDecode")
        self.bufferSize = options.get("videoBufferSize") or 512 * 1024
        self.bufferMode = (capi.BIT_BUFFER_MODE_EVICT if options.get("streaming")
                           else capi.BIT_BUFFER_MODE_EXPAND)
        self.decodeFirstFrame = options.get("decodeFirstFrame", True) is not False
        self.hasSequenceHeader = False
        self.frameRate = 30.0
        self.codedSize = 0
        self.width = 0
        self.height = 0
        self.currentY = self.currentCr = self.currentCb = None
        self.functions = lib if lib is not None else capi.product_library()
        if options.get("device") is not None and hasattr(self.functions, "jsmpeg_b200_set_default_device"):
            self.functions.jsmpeg_b200_set_default_device(int(options["device"]))
        self.decoder = self.functions.mpeg1_decoder_create(self.bufferSize, self.bufferMode)
        # the product library never fails in create (reference behaviour); a decoder without a usable CUDA
        # device is dead and answers decode() == False for ever.  The Python host says so loudly instead.
        if hasattr(self.functions, "jsmpeg_b200_decoder_last_error"):
            err = self.functions.jsmpeg_b200_decoder_last_error(self.decoder)
            if err:
                self.destroy()
                raise RuntimeError(err.decode(errors="replace"))
        self.displayOrder = False
        self._held = None  # displayOrder: the I/P picture waiting for the B pictures shown before it
        if options.get("decodeBPictures"):
            if not hasattr(self.functions, "jsmpeg_b200_decoder_set_option"):
                raise ValueError("decodeBPictures: this library has no B-picture extension")
            self.functions.jsmpeg_b200_decoder_set_option(self.decoder, b"decode_b", 1)
            self.displayOrder = bool(options.get("displayOrder"))
        self.exportMacroblocks = bool(options.get("exportMacroblocks"))
        if self.exportMacroblocks:
            if not hasattr(self.functions, "jsmpeg_b200_decoder_get_macroblocks"):
                raise ValueError("exportMacroblocks: this library has no macroblock export")
            self.functions.jsmpeg_b200_decoder_set_option(self.decoder, b"macroblocks", 1)
        self.concealErrors = bool(options.get("concealErrors"))
        if self.concealErrors:
            if not hasattr(self.functions, "jsmpeg_b200_decoder_set_option") or \
                    self.functions.jsmpeg_b200_decoder_set_option(self.decoder, b"conceal", 1) != 0:
                self.destroy()
                raise ValueError("concealErrors: this library has no error concealment")

    # ---- src/decoder.js:19-35 / src/mpeg1-wasm.js:32-50
    def destroy(self):
        if self.decoder:
            self.functions.mpeg1_decoder_destroy(self.decoder)
            self.decoder = None

    def connect(self, destination):
        self.destination = destination

    def bufferGetIndex(self):
        return self.functions.mpeg1_decoder_get_index(self.decoder)

    def bufferSetIndex(self, index):
        self.functions.mpeg1_decoder_set_index(self.decoder, index)

    # ---- src/mpeg1-wasm.js:52-70
    def bufferWrite(self, buffers):
        total = sum(len(b) for b in buffers)
        ptr = self.functions.mpeg1_decoder_get_write_ptr(self.decoder, total)
        for b in buffers:
            n = len(b)
            if n:
                ctypes.memmove(ptr, b if isinstance(b, bytes) else bytes(b), n)
                ptr += n
        self.functions.mpeg1_decoder_did_write(self.decoder, total)
        return total

    # ---- src/decoder.js:36-47 then src/mpeg1-wasm.js:72-94
    def write(self, pts, buffers):
        if self.collectTimestamps:
            if len(self.timestamps) == 0:
                self.startTime = pts
                self.decodedTime = pts
            self.timestamps.append((self.bytesWritten << 3, pts))
        self.bytesWritten += self.bufferWrite(buffers)
        self.canPlay = True
        if not self.hasSequenceHeader and self.functions.mpeg1_decoder_has_sequence_header(self.decoder):
            self._load_sequence_header()

    def _load_sequence_header(self):
        self.hasSequenceHeader = True
        self.frameRate = self.functions.mpeg1_decoder_get_frame_rate(self.decoder)
        self.codedSize = self.functions.mpeg1_decoder_get_coded_size(self.decoder)
        self.width = self.functions.mpeg1_decoder_get_width(self.decoder)
        self.height = self.functions.mpeg1_decoder_get_height(self.decoder)
        if self.destination is not None:
            self.destination.resize(self.width, self.height)
        if self.decodeFirstFrame:
            self.decode()

    # ---- src/decoder.js:49-71
    def seek(self, t):
        if not self.collectTimestamps:
            return
        self.timestampIndex = 0
        for i, (_, ts_time) in enumerate(self.timestamps):
            if ts_time > t:
                break
            self.timestampIndex = i
        if self.timestamps:
            index, ts_time = self.timestamps[self.timestampIndex]
            self.bufferSetIndex(index)
            self.decodedTime = ts_time
        else:
            self.bufferSetIndex(0)
            self.decodedTime = self.startTime

    # ---- src/mpeg1-wasm.js:96-129
    def decode(self):
        t0 = time.perf_counter()
        if not self.decoder:
            return False
        if not self.functions.mpeg1_decoder_decode(self.decoder):
            return False
        self.currentY, self.currentCr, self.currentCb = self.planes()
        if self.displayOrder:
            self._render_in_display_order()
        elif self.destination is not None:
            self.destination.render(self.currentY, self.currentCr, self.currentCb, False)
        self.advanceDecodedTime(1.0 / self.frameRate if self.frameRate else 0.0)
        if self.onDecodeCallback:
            self.onDecodeCallback(self, (time.perf_counter() - t0) * 1000.0)
        return True

    def _render_in_display_order(self):
        """Extension (decodeBPictures + displayOrder): a B picture is shown at once, an I/P picture when the next
        I/P picture arrives -- the B pictures that follow it in the stream come before it on the screen
        (ISO 11172-2 2.4.1: pictures are transmitted in decoding order).  The planes the library hands out are
        borrowed until the next decode(), so the held picture is a copy."""
        kind = self.lastPicture()
        if kind is None or kind[0] not in (1, 2, 3):
            return  # a D picture / unknown type: nothing was decoded (mpeg1.js:181-184)
        if kind[0] == 3:
            if self.destination is not None:
                self.destination.render(self.currentY, self.currentCr, self.currentCb, False)
            return
        self.flush()
        self._held = (self.currentY.copy(), self.currentCr.copy(), self.currentCb.copy())

    def flush(self):
        """displayOrder: render the I/P picture still held back (end of stream, or before a seek)."""
        if self._held is not None and self.destination is not None:
            self.destination.render(*self._held, False)
        self._held = None

    def lastPicture(self):
        """(picture_coding_type, temporal_reference) of the picture the last decode() consumed (extension)."""
        t, r = ctypes.c_int(), ctypes.c_int()
        if self.functions.jsmpeg_b200_decoder_last_picture(self.decoder, ctypes.byref(t), ctypes.byref(r)) != 0:
            return None
        return t.value, r.value

    def planes(self):
        """Zero-copy views of the most recently decoded picture (borrowed; valid until the next
        decode(), like the ``heapU8.subarray`` views of src/mpeg1-wasm.js:110-116)."""
        n = self.codedSize

        def view(ptr, size):
            return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_uint8)), shape=(size,))

        f = self.functions
        return (view(f.mpeg1_decoder_get_y_ptr(self.decoder), n),
                view(f.mpeg1_decoder_get_cr_ptr(self.decoder), n >> 2),
                view(f.mpeg1_decoder_get_cb_ptr(self.decoder), n >> 2))

    def macroblocks(self):
        """exportMacroblocks (extension): a zero-copy uint8 view [mb_height, mb_width, 16] of the macroblock entries
        (include/jsmpeg_b200.h: jsmpeg_b200_macroblock_t; jsmpeg_b200.batch.macroblocks_view names the fields) of the
        picture the last decode() rendered -- borrowed like planes(); None without the option or before the sequence
        header."""
        ptr = self.functions.jsmpeg_b200_decoder_get_macroblocks(self.decoder) if self.exportMacroblocks else None
        if not ptr:
            return None
        shape = ((self.height + 15) // 16, (self.width + 15) // 16, 16)
        return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_uint8)), shape=shape)

    # ---- src/decoder.js:77-106
    def advanceDecodedTime(self, seconds):
        if self.collectTimestamps:
            new_index = -1
            current = self.bufferGetIndex()
            for i in range(self.timestampIndex, len(self.timestamps)):
                if self.timestamps[i][0] > current:
                    break
                new_index = i
            if new_index != -1 and new_index != self.timestampIndex:
                self.timestampIndex = new_index
                self.decodedTime = self.timestamps[new_index][1]
                return
        self.decodedTime += seconds

    @property
    def currentTime(self):
        return self.decodedTime


class PlaneRecorder:
    """A minimal ``destination`` (renderer contract, reference src/jsmpeg.js:40-62): records a copy
    of every rendered picture.  Used by tests, tools and the smoke check."""

    def __init__(self, keep=True):
        self.size = None
        self.frames = []
        self.keep = keep
        self.count = 0

    def resize(self, w, h):
        self.size = (w, h)

    def render(self, y, cr, cb, is_clamped):
        self.count += 1
        if self.keep:
            self.frames.append((y.copy(), cr.copy(), cb.copy()))
