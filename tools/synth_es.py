#!/usr/bin/env python
"""Synthetic MPEG-1 video elementary streams generated at the SYNTAX level (SURVEY.md section 7,
step 0(b)): random but valid sequences of syntax elements, written with the VLC tables of
tools/vlc_tables.py.  There is no image content and no DCT: the point is to drive a decoder through
the corners of the bitstream syntax that FFmpeg's encoder never produces, so that the oracle, the
compiled reference and the CUDA path can be compared bit for bit on them:

  * several slices per picture, slices spanning rows, gaps between slices (macroblocks no slice
    covers), first-macroblock address increments > 1
  * macroblock_stuffing, macroblock_escape, long skipped runs in P pictures
  * every I and P macroblock type, quantiser changes, all coded_block_pattern values
  * forward_f_code 1..7, full_pel_forward_vector, all four half-pel parities, vector wrap-around,
    by default keeping the whole 17x17 / 9x9 reference footprint inside the coded planes (SURVEY Q11);
    Knobs.vectors opens the rest of the vector domain: the f_code's whole range, footprints that wrap
    from one row into the next, and taps outside the plane
  * intra DC sizes 0..8, DC-only blocks, the (0,1) first-coefficient form, long runs, index 63,
    escapes in the one- and two-byte forms, positive and negative
  * custom intra / non-intra quantiser matrices, extension and user data after the picture header,
    pictures the reference ignores (B / D type, forward_f_code 0), a repeated sequence header

Start-code emulation is avoided by construction where the syntax allows it and checked per slice
(a slice whose bytes contain an aligned 00 00 0x pattern is re-rolled).
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import vlc_tables as V  # noqa: E402

_inv = lambda table: {v: k for k, v in table.items()}  # noqa: E731
MBA_CODE = _inv(V.MBA_INCREMENT)
TYPE_I_CODE = _inv(V.MB_TYPE_INTRA)
TYPE_P_CODE = _inv(V.MB_TYPE_PREDICTIVE)
TYPE_B_CODE = _inv(V.MB_TYPE_B)
CBP_CODE = _inv(V.CODE_BLOCK_PATTERN)
MOTION_CODE = _inv(V.MOTION)
DC_LUMA_CODE = _inv(V.DCT_DC_SIZE_LUMINANCE)
DC_CHROMA_CODE = _inv(V.DCT_DC_SIZE_CHROMINANCE)
MAX_SLICE_ROW = 0xAF - 1  # the last macroblock row a slice start code (0x01..0xAF) names
MAX_LEVEL_FOR_RUN = {}
for (_r, _l) in V.DCT_RUN_LEVEL_CODE:
    MAX_LEVEL_FOR_RUN[_r] = max(MAX_LEVEL_FOR_RUN.get(_r, 0), _l)


class BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, value, n):
        for i in range(n - 1, -1, -1):
            self.bits.append((value >> i) & 1)

    def code(self, s):
        self.bits.extend(1 if c == "1" else 0 for c in s)

    def align(self):
        while len(self.bits) % 8:
            self.bits.append(0)

    def start_code(self, code):
        self.align()
        self.put(0x000001, 24)
        self.put(code, 8)

    def tobytes(self):
        assert len(self.bits) % 8 == 0
        return np.packbits(np.array(self.bits, dtype=np.uint8)).tobytes()


class Knobs:
    """Probabilities / ranges of the random syntax generator."""

    def __init__(self, **kw):
        self.width = 96
        self.height = 64
        self.pictures = 8
        self.gop = 4                 # an I picture every `gop` pictures
        self.slices = "rows"         # "one" | "rows" | "random"
        self.slice_gap_prob = 0.0    # leave a run of macroblocks uncovered between slices ...
        self.gap_from_picture = 2    # ... but only once both plane sets have been fully written: the
        #                              compiled C reference mallocs its planes (mpeg1.c:935-941) where JS
        #                              zero-fills them (SURVEY Q19), so earlier gaps are not comparable
        self.stuffing_prob = 0.05
        self.skip_prob = 0.15        # P pictures: probability of starting a skipped run
        self.max_skip = 40
        self.intra_in_p_prob = 0.15
        self.quant_change_prob = 0.2
        self.f_codes = (1, 2, 3)
        self.full_pel_prob = 0.2
        self.escape_prob = 0.12
        self.big_escape_prob = 0.3   # of the escapes, two-byte form
        self.dc_only_prob = 0.25
        self.max_coefs = 12
        self.custom_matrices = False
        self.extension_user_data = False
        self.ignored_pictures = False
        self.repeat_sequence_header = False
        self.gop_headers = True
        # B pictures (the opt-in extension; the reference skips them): b_frames > 0 puts that many B pictures
        # behind every I/P picture in CODED order (I B B P B B ...: the first ones have one reference only,
        # an open GOP), `gop` then counts I/P pictures.  0 = none, and no random numbers are drawn for them:
        # the streams of the committed cases stay byte-identical.
        self.b_frames = 0
        self.b_skip_prob = 0.2
        self.b_intra_prob = 0.08
        self.b_f_codes = (1, 2, 3)
        # Where motion vectors point (SURVEY Q11: prediction by flat index, a tap outside the plane zeroes its sample):
        #   "inside"   small vectors (at most 24 half-pel) whose 17x17 / 9x9 footprints stay inside the 2-D planes
        #   "wide"     the whole [-16f, 16f - 1] range of the picture's f_code, footprints inside the 2-D planes
        #   "wrap"     footprints that cross the left or right edge with every tap's flat index inside its plane
        #   "outside"  at least one tap outside its plane: mostly near misses, some far out
        #   "mixed"    one of the four per macroblock
        # "inside" draws exactly what it always drew: the streams of the committed cases stay byte-identical.
        self.vectors = "inside"
        # The value domain (VALUE_CASES).  None / 0 / "canonical" draw exactly what they always drew: the streams of
        # the committed cases stay byte-identical.
        #   dc_walk        None: every intra DC target in 0..255.  Else one mode per DC predictor (Y, the one of block
        #                  4, the one of block 5): "keep" (a target in 0..255), "climb" / "descend" (every differential
        #                  +-dc_step, turning back at +-dc_limit), "wander" (runs of dc_run blocks in one direction)
        #   ac_cross_prob  of the intra blocks, the share whose AC coefficients are escapes of level +-255 signed like the
        #                  transform's basis at one sample: |ac(x)| of several thousand, so that dc + ac(x) crosses 0 and
        #                  255 when the DC is far outside 0..255
        #   escape_forms   "all": besides the canonical escapes, the two-byte forms of small levels, (0, 0) = level 0
        #                  and (128, 0) = level -256
        #   qscales        None: quantiser scales 1..31; else the scales the slice and macroblock headers draw from
        #   matrix_entries None: the default custom matrices; else the values every entry (intra Q[0] included) draws from
        self.dc_walk = None
        self.dc_step = (128, 255)
        self.dc_limit = 300_000
        self.dc_run = 24
        self.ac_cross_prob = 0.0
        self.escape_forms = "canonical"
        self.qscales = None
        self.matrix_entries = None
        # How the bits spread over the picture (GEOMETRY_CASES).  None draws exactly what it always drew.
        #   "letterbox"  the first and last `bar` of the macroblock rows (a (top, bottom) pair: each its own share) are
        #                black bars: DC-only intra macroblocks of about 30 bits in I pictures, skipped runs and
        #                zero-vector uncoded macroblocks in P pictures
        #   "flat"       the whole picture is bar (a fade to black)
        self.profile = None
        self.bar = 0.12
        self.__dict__.update(kw)
        assert self.dc_limit + 255 < 1 << 23  # the reference keeps dc << 8 in an int


class SynthStream:
    def __init__(self, knobs: Knobs, seed: int):
        self.k = knobs
        self.rng = np.random.default_rng(seed)
        self.mbw = (knobs.width + 15) // 16
        self.mbh = (knobs.height + 15) // 16
        self.out = BitWriter()

    # ---------------------------------------------------------------- headers
    def sequence_header(self):
        w = self.out
        w.start_code(0xB3)
        w.put(self.k.width, 12)
        w.put(self.k.height, 12)
        w.put(1, 4)          # aspect
        w.put(5, 4)          # 30 fps
        w.put(0x3FFFF, 18)   # bit rate
        w.put(1, 1)          # marker
        w.put(20, 10)        # vbv buffer size
        w.put(0, 1)          # constrained
        if self.k.custom_matrices and self.k.matrix_entries is not None:
            for _ in range(2):
                w.put(1, 1)
                for i in range(64):
                    w.put(int(self.rng.choice(self.k.matrix_entries)), 8)
        elif self.k.custom_matrices:
            w.put(1, 1)
            for i in range(64):
                w.put(8 if i == 0 else int(self.rng.integers(4, 64)), 8)
            w.put(1, 1)
            for i in range(64):
                w.put(int(self.rng.integers(8, 48)), 8)
        else:
            w.put(0, 1)
            w.put(0, 1)

    def gop_header(self):
        w = self.out
        w.start_code(0xB8)
        w.put(0, 25)  # time code
        w.put(1, 1)   # closed gop
        w.put(0, 1)   # broken link

    def picture_header(self, temporal, ptype, full_pel=0, f_code=1, full_pel_b=0, f_code_b=1):
        w = self.out
        w.start_code(0x00)
        w.put(temporal & 1023, 10)
        w.put(ptype, 3)
        w.put(0xFFFF, 16)  # vbv delay
        if ptype in (2, 3):
            w.put(full_pel, 1)
            w.put(f_code, 3)
        if ptype == 3:
            w.put(full_pel_b, 1)
            w.put(f_code_b, 3)
        w.put(0, 1)  # extra_bit_picture
        if self.k.extension_user_data and self.rng.random() < 0.5:
            w.start_code(0xB5)
            for _ in range(int(self.rng.integers(1, 6))):
                w.put(int(self.rng.integers(1, 256)) | 0x80, 8)
            w.start_code(0xB2)
            for _ in range(int(self.rng.integers(1, 9))):
                w.put(int(self.rng.integers(1, 256)) | 0x40, 8)

    # ---------------------------------------------------------------- blocks
    def block(self, w, intra, luma, dc_pred, which=0):
        """One coded block (`which`: its DC predictor, 0 = Y, 1 = block 4's, 2 = block 5's).  Returns the new DC
        predictor (intra)."""
        rng = self.rng
        if intra:
            if self.k.dc_walk is None or self.k.dc_walk[which] == "keep":
                # keep the reconstructed DC in 0..255
                target = int(rng.integers(0, 256)) if rng.random() < 0.7 else dc_pred
            else:
                target = dc_pred + self.dc_step(which, dc_pred)
            diff = target - dc_pred
            size = 0 if diff == 0 else int(abs(diff)).bit_length()
            w.code((DC_LUMA_CODE if luma else DC_CHROMA_CODE)[size])
            if size:
                w.put(diff if diff > 0 else diff + (1 << size) - 1, size)
            dc_pred = target
            n = 1
            if self.k.ac_cross_prob and rng.random() < self.k.ac_cross_prob:
                self.crossing_ac(w)
                return dc_pred
        else:
            n = 0
        if intra and rng.random() < self.k.dc_only_prob:
            count = 0
        else:
            count = int(rng.integers(1, self.k.max_coefs + 1))
        first = not intra
        zero_tail = False  # the last escape ended in a zero byte: the next code is an escape too (5 leading zeros)
        for c in range(count):
            remaining = 63 - n
            if remaining < 0:
                break
            if c == count - 1 and rng.random() < 0.1:
                run = remaining  # land exactly on index 63
            else:
                run = int(min(remaining, rng.geometric(0.35) - 1))
            if zero_tail or rng.random() < self.k.escape_prob:
                zero_tail = self.escape(w, run)
            else:
                run_t = min(run, 31)
                level = int(rng.integers(1, MAX_LEVEL_FOR_RUN[run_t] + 1))
                if rng.random() < 0.6:
                    level = 1 if MAX_LEVEL_FOR_RUN[run_t] == 1 else int(rng.integers(1, 3))
                level = min(level, MAX_LEVEL_FOR_RUN[run_t])
                code = V.DCT_RUN_LEVEL_CODE[(run_t, level)]
                if first and code == "1":
                    w.code("1")
                elif code == "1":
                    w.code("11")
                else:
                    w.code(code)
                w.put(int(rng.integers(0, 2)), 1)
                run = run_t
            first = False
            n += run + 1
        if not intra and count == 0:
            # a coded non-intra block has at least one coefficient
            w.code("1")
            w.put(int(rng.integers(0, 2)), 1)
        w.code(V.DCT_EOB_CODE)
        return dc_pred

    def dc_step(self, which, dc_pred):
        """The next DC differential of predictor `which` under Knobs.dc_walk: +-1..255, turning back at +-dc_limit"""
        rng, k = self.rng, self.k
        mode = k.dc_walk[which]
        if mode == "wander":
            self.wander = getattr(self, "wander", [1, 1, 1])
            if rng.random() < 1.0 / k.dc_run:
                self.wander[which] = -self.wander[which]
            sign = self.wander[which]
        else:
            sign = 1 if mode == "climb" else -1
        step = sign * int(rng.integers(k.dc_step[0], k.dc_step[1] + 1))
        if abs(dc_pred + step) > k.dc_limit:
            step = -step
            if mode == "wander":
                self.wander[which] = -self.wander[which]
        return step

    def crossing_ac(self, w):
        """The AC coefficients of an intra block as escapes of level +-255 at zig-zag positions 1..K, each signed like
        the 2-D cosine basis at one sample (y, x) -- all of them the same way or all the opposite way -- so that the
        transform moves that sample by thousands; then end_of_block"""
        rng = self.rng
        y, x = int(rng.integers(0, 8)), int(rng.integers(0, 8))
        s = 1 if rng.random() < 0.5 else -1
        count = int(rng.integers(11, 64))
        for n in range(1, count + 1):
            r = V.ZIG_ZAG[n]
            basis = np.cos((2 * x + 1) * (r % 8) * np.pi / 16) * np.cos((2 * y + 1) * (r // 8) * np.pi / 16)
            level = 255 if s * basis > 0 else -255
            if level < 0 and self.k.escape_forms == "all" and rng.random() < 0.3:
                level = -256
            self.escape_level(w, 0, level)
        w.code(V.DCT_EOB_CODE)

    def escape_level(self, w, run, level):
        """An escape of `level` in -256..255 (0 and -256 only in their two-byte forms (0, 0) and (128, 0))"""
        w.code(V.DCT_ESCAPE_CODE)
        w.put(run, 6)
        if 0 < abs(level) < 128:
            w.put(level & 255, 8)
        elif level >= 0:
            w.put(0, 8)
            w.put(level, 8)
        else:
            w.put(128, 8)
            w.put(level + 256, 8)

    def escape(self, w, run):
        rng = self.rng
        if self.k.escape_forms == "all" and rng.random() < 0.5:
            # the two-byte forms of any level (0 and -256 only have those); level 0 only behind an odd run, and a
            # level ending in a zero byte is followed by an escape or end_of_block, so that the zeros of the escape,
            # the run, the level and the next code never make 23 in a row.  Returns whether it ends in a zero byte.
            form = int(rng.integers(0, 4))
            level = (0 if run & 1 else -256, -256, int(rng.integers(1, 128)), -int(rng.integers(1, 128)))[form]
            w.code(V.DCT_ESCAPE_CODE)
            w.put(run, 6)
            w.put(0 if level >= 0 else 128, 8)
            w.put(level & 255, 8)
            return level in (0, -256)
        w.code(V.DCT_ESCAPE_CODE)
        w.put(run, 6)
        if rng.random() < self.k.big_escape_prob:
            level = int(rng.integers(128, 256))
            if rng.random() < 0.5:
                w.put(0, 8)
                w.put(level, 8)             # +128..+255
            else:
                w.put(128, 8)
                w.put(256 - level, 8)       # -255..-128 (second byte 1..128)
        else:
            level = int(rng.integers(1, 128))
            w.put(level if rng.random() < 0.5 else 256 - level, 8)
        return False

    def qscale(self):
        return int(self.rng.integers(1, 32)) if self.k.qscales is None else int(self.rng.choice(self.k.qscales))

    # ---------------------------------------------------------------- motion
    def motion_component(self, w, target, prev, f, r_size):
        """Encode so that the decoder's predictor becomes `target` (mpeg1.js:395-457)."""
        d = target - prev
        if d > 16 * f - 1:
            d -= 32 * f
        elif d < -16 * f:
            d += 32 * f
        if f == 1 or d == 0:
            w.code(MOTION_CODE[d])
        else:
            a = abs(d) - 1
            code = (a >> r_size) + 1
            w.code(MOTION_CODE[code if d > 0 else -code])
            w.put(a & (f - 1), r_size)
        return target

    def pick_vector(self, mb_col, mb_row, f, full_pel):
        """A predictor value (in the units the bitstream carries) in the vector domain of Knobs.vectors; for "inside"
        one whose luma AND chroma footprints stay inside the coded planes."""
        rng = self.rng
        lo, hi = -16 * f, 16 * f - 1
        scale = 2 if full_pel else 1
        mode = self.k.vectors
        if mode == "mixed":
            mode = ("inside", "wide", "wrap", "outside")[int(rng.integers(0, 4))]
        if mode != "inside":
            return self._pick_in_domain(mode, mb_col, mb_row, lo, hi, scale)
        for _ in range(50):
            vx = int(rng.integers(max(lo, -24), min(hi, 24) + 1))
            vy = int(rng.integers(max(lo, -24), min(hi, 24) + 1))
            if self.footprint_inside(mb_col, mb_row, vx * scale, vy * scale):
                return vx, vy
        return 0, 0

    def _pick_in_domain(self, mode, mb_col, mb_row, lo, hi, scale):
        """A predictor of domain "wide", "wrap" or "outside" (Knobs.vectors) for macroblock (mb_col, mb_row): targets
        drawn around the plane edges the domain needs, kept when the predictor is representable and the domain's rule
        holds."""
        rng = self.rng
        cw, ch = self.mbw * 16, self.mbh * 16
        x_here, y_here = mb_col * 16, mb_row * 16

        def unit(m):  # a half-pel target -> the predictor value that gives it, or None when out of range
            v = m // scale
            return v if lo <= v <= hi else None

        def spread(here, size):  # a luma half-pel component anywhere the f_code reaches
            return int(rng.integers(lo, hi + 1)) * scale if rng.random() < 0.3 else \
                2 * (int(rng.integers(-here, size - here - 16 + 1))) + int(rng.integers(0, 2))

        def edge(here, size, reach):  # a component that puts the footprint's first sample around an edge of one axis
            at = int(rng.integers(-reach, 1)) if rng.random() < 0.5 else size - 16 + int(rng.integers(0, reach + 1))
            return 2 * (at - here) + int(rng.integers(-1, 2))

        for _ in range(60):
            if mode == "wide":
                mx, my, rule = spread(x_here, cw), spread(y_here, ch), "inside"
            elif mode == "wrap":
                mx = edge(x_here, cw, 17 if rng.random() < 0.8 else 40)
                my = spread(y_here, ch) if rng.random() < 0.5 else 2 * int(rng.integers(-2, 3)) + int(rng.integers(0, 2))
                rule = "wrap"
            else:
                kind, rule = rng.random(), "out"
                if kind < 0.45:    # a row just past the top or bottom edge (the half-pel row, one row, chroma alone)
                    mx = 2 * int(rng.integers(-3, 4)) + int(rng.integers(-1, 2))
                    my = edge(y_here, ch, 2)
                elif kind < 0.7:   # a column just past the left or right edge in the first or last rows
                    mx = edge(x_here, cw, 2)
                    my = edge(y_here, ch, 1) if rng.random() < 0.6 else \
                        2 * int(rng.integers(-2, 3)) + int(rng.integers(-1, 2))
                elif kind < 0.85:  # the chroma taps out, the luma ones inside (a wrap a row further for luma)
                    mx = edge(x_here, cw, 40)
                    my = 2 * int(rng.integers(-3, 4)) + int(rng.integers(-1, 2))
                    rule = "chroma_out"
                else:              # anywhere in the f_code's range
                    mx, my = int(rng.integers(lo, hi + 1)) * scale, int(rng.integers(lo, hi + 1)) * scale
            vx, vy = unit(mx), unit(my)
            if vx is not None and vy is not None and self._obeys(rule, mb_col, mb_row, vx * scale, vy * scale):
                return vx, vy
        # a macroblock too far from the edges the domain needs: a "wide" vector instead
        return self._pick_in_domain("wide", mb_col, mb_row, lo, hi, scale) if mode != "wide" else (0, 0)

    def _obeys(self, rule, mb_col, mb_row, mx, my):
        """Whether vector (mx, my) (luma half-pel units) at macroblock (mb_col, mb_row) follows `rule`: "inside" (both
        footprints inside the 2-D planes), "wrap" (every flat-index tap inside, a footprint across the left or right
        edge), "out" (some tap outside its plane) or "chroma_out" (the luma taps inside, some chroma tap outside)"""
        if rule == "inside":
            return self.footprint_inside(mb_col, mb_row, mx, my)
        if rule == "wrap":
            return self.flat_inside(mb_col, mb_row, mx, my) and not self.footprint_inside(mb_col, mb_row, mx, my)
        if rule == "out":
            return not self.flat_inside(mb_col, mb_row, mx, my)
        return self.flat_inside(mb_col, mb_row, mx, my, "luma") and not self.flat_inside(mb_col, mb_row, mx, my, "chroma")

    def flat_inside(self, mb_col, mb_row, mx, my, planes="both"):
        """Vector (mx, my) in luma half-pel units at macroblock (mb_col, mb_row): every tap of the luma and of the chroma
        prediction ("luma" / "chroma": of that one), addressed by flat index (a sample past a row's end is the next
        row's first, mpeg1.js:479, 567), lies inside its plane."""
        def plane(px, stride, size, h, v):
            first = (mb_row * px + (v >> 1)) * stride + mb_col * px + (h >> 1)
            return first >= 0 and first + (px - 1) * stride + px - 1 + (v & 1) * stride + (h & 1) < size
        cw = self.mbw * 16
        ysize = cw * self.mbh * 16
        luma = planes == "chroma" or plane(16, cw, ysize, mx, my)
        return luma and (planes == "luma" or plane(8, cw // 2, ysize // 4, int(mx / 2), int(my / 2)))

    def skip_keeps_domain(self, mb_col, mb_row, mx, my):
        """Whether a skipped B macroblock may repeat vector (mx, my) (luma half-pel units) under Knobs.vectors"""
        if self.k.vectors in ("inside", "wide"):
            return self.footprint_inside(mb_col, mb_row, mx, my)
        if self.k.vectors == "wrap":
            return self.flat_inside(mb_col, mb_row, mx, my)
        return True

    def footprint_inside(self, mb_col, mb_row, mx, my):
        """Vector (mx, my) in luma half-pel units at macroblock (mb_col, mb_row): the luma and the chroma
        footprint both stay inside the coded planes."""
        cw, ch = self.mbw * 16, self.mbh * 16
        x0 = mb_col * 16 + (mx >> 1)
        y0 = mb_row * 16 + (my >> 1)
        x1 = x0 + 16 + (mx & 1)
        y1 = y0 + 16 + (my & 1)
        if x0 < 0 or y0 < 0 or x1 > cw or y1 > ch:
            return False
        cx, cy = int(mx / 2), int(my / 2)  # truncation toward zero (mpeg1.js:562-565)
        x0 = mb_col * 8 + (cx >> 1)
        y0 = mb_row * 8 + (cy >> 1)
        x1 = x0 + 8 + (cx & 1)
        y1 = y0 + 8 + (cy & 1)
        return not (x0 < 0 or y0 < 0 or x1 > cw // 2 or y1 > ch // 2)

    # ---------------------------------------------------------------- slices
    def address_increment(self, w, inc):
        if self.rng.random() < self.k.stuffing_prob:
            for _ in range(int(self.rng.integers(1, 4))):
                w.code(MBA_CODE[34])
        while inc > 33:
            w.code(MBA_CODE[35])
            inc -= 33
        w.code(MBA_CODE[inc])

    def slice(self, ptype, first_mb, last_mb, f_code, full_pel, f_code_b=1, full_pel_b=0):
        """Macroblocks first_mb..last_mb (inclusive, raster addresses) as one slice whose start
        code is the row of first_mb + 1.  Returns the slice bytes (re-rolled on start-code emulation)."""
        for _attempt in range(20):
            w = BitWriter()
            if ptype == 3:
                data = self._slice_once_b(w, first_mb, last_mb, f_code, full_pel, f_code_b, full_pel_b)
            else:
                data = self._slice_once(w, ptype, first_mb, last_mb, f_code, full_pel)
            body = data[4:]
            # the decoder ends a slice where the next whole byte starts a start code (buffer.c:101-110): a last
            # macroblock that begins in the slice's final byte would never be read
            if (self.last_mb_bit + 7) // 8 >= len(data):
                continue
            bad = any(body[i] == 0 and body[i + 1] == 0 and body[i + 2] <= 1 for i in range(len(body) - 2))
            if not bad and not (len(body) >= 2 and body[-1] == 0 and body[-2] == 0) and not (len(body) >= 1 and body[-1] == 0):
                return data
        raise RuntimeError("could not generate an emulation-free slice")

    def _slice_once(self, w, ptype, first_mb, last_mb, f_code, full_pel):
        rng = self.rng
        mbw = self.mbw
        row = first_mb // mbw
        w.start_code(row + 1)
        qscale = self.qscale()
        w.put(qscale, 5)
        if rng.random() < 0.1:          # extra_information_slice
            w.put(1, 1)
            w.put(int(rng.integers(1, 256)), 8)
        w.put(0, 1)
        f = 1 << (f_code - 1)
        r_size = f_code - 1
        prev_h = prev_v = 0
        dc = [128, 128, 128]
        addr = row * mbw - 1
        mb = first_mb
        first = True
        while mb <= last_mb:
            inc = mb - addr
            skipped = 0
            if self.in_bar(mb):
                mb, addr, first, dc, prev_h, prev_v = self._bar_macroblock(w, ptype, mb, addr, first, last_mb, dc, prev_h,
                                                                          prev_v, f, r_size)
                continue
            if not first and ptype == 2 and rng.random() < self.k.skip_prob and mb < last_mb:
                skipped = int(min(rng.integers(1, self.k.max_skip + 1), last_mb - mb))
                while skipped and self.in_bar(mb + skipped):  # (a bar's macroblocks are coded as bars)
                    skipped -= 1
                mb += skipped
                inc = mb - addr
            if skipped:
                dc = [128, 128, 128]
                prev_h = prev_v = 0
            self.last_mb_bit = len(w.bits)
            self.address_increment(w, inc)
            addr = mb
            first = False
            mb_row, mb_col = divmod(mb, mbw)
            if ptype == 1:
                mtype = 0x11 if rng.random() < self.k.quant_change_prob else 0x01
                w.code(TYPE_I_CODE[mtype])
            else:
                if rng.random() < self.k.intra_in_p_prob:
                    mtype = 0x11 if rng.random() < self.k.quant_change_prob else 0x01
                else:
                    mtype = int(rng.choice([0x0A, 0x02, 0x08, 0x1A, 0x12]))
                w.code(TYPE_P_CODE[mtype])
            if mtype & 0x10:
                qscale = self.qscale()
                w.put(qscale, 5)
            intra = mtype & 0x01
            if intra:
                prev_h = prev_v = 0
            else:
                dc = [128, 128, 128]
                if mtype & 0x08:
                    th, tv = self.pick_vector(mb_col, mb_row, f, full_pel)
                    prev_h = self.motion_component(w, th, prev_h, f, r_size)
                    prev_v = self.motion_component(w, tv, prev_v, f, r_size)
                else:
                    prev_h = prev_v = 0
            if mtype & 0x02:
                cbp = int(rng.integers(1, 64))
                w.code(CBP_CODE[cbp])
            else:
                cbp = 0x3F if intra else 0
            for blk in range(6):
                if cbp & (0x20 >> blk):
                    which = 0 if blk < 4 else blk - 3
                    dc[which] = self.block(w, intra, blk < 4, dc[which], which)
            mb += 1
        w.align()
        return w.tobytes()

    def in_bar(self, mb):
        """Whether macroblock `mb` lies in a black bar of Knobs.profile"""
        if self.k.profile is None:
            return False
        if self.k.profile == "flat":
            return True
        top, bottom = self.k.bar if isinstance(self.k.bar, tuple) else (self.k.bar, self.k.bar)
        row = mb // self.mbw
        return row < round(top * self.mbh) or row >= self.mbh - round(bottom * self.mbh)

    def _bar_macroblock(self, w, ptype, mb, addr, first, last_mb, dc, prev_h, prev_v, f, r_size):
        """A black-bar macroblock at `mb` (after a skipped run through the bar in P pictures): intra and DC-only near
        black in I pictures, a zero vector without coded blocks in P pictures.  Returns the slice state after it."""
        rng = self.rng
        if ptype == 2 and not first and mb < last_mb and rng.random() < 0.8:
            run = 1
            while run < 4 * self.mbw and mb + run < last_mb and self.in_bar(mb + run):
                run += 1
            mb += int(rng.integers(1, run + 1))
            dc = [128, 128, 128]
            prev_h = prev_v = 0
        self.last_mb_bit = len(w.bits)
        self.address_increment(w, mb - addr)
        if ptype == 1:
            w.code(TYPE_I_CODE[0x01])
            for blk in range(6):
                which = 0 if blk < 4 else blk - 3
                target = (16 if blk < 4 else 128) + (int(rng.integers(0, 3)) if rng.random() < 0.2 else 0)
                diff = target - dc[which]
                size = 0 if diff == 0 else abs(diff).bit_length()
                w.code((DC_LUMA_CODE if blk < 4 else DC_CHROMA_CODE)[size])
                if size:
                    w.put(diff if diff > 0 else diff + (1 << size) - 1, size)
                dc[which] = target
                w.code(V.DCT_EOB_CODE)
        else:
            w.code(TYPE_P_CODE[0x08])
            prev_h = self.motion_component(w, 0, prev_h, f, r_size)
            prev_v = self.motion_component(w, 0, prev_v, f, r_size)
            dc = [128, 128, 128]
        return mb + 1, mb, False, dc, prev_h, prev_v

    def _slice_once_b(self, w, first_mb, last_mb, f_code, full_pel, f_code_b, full_pel_b):
        """A slice of a B picture (ISO 11172-2 2.4.3.6, 2.4.4.2, 2.4.4.3; types: table B.2d)."""
        rng = self.rng
        mbw = self.mbw
        row = first_mb // mbw
        w.start_code(row + 1)
        qscale = self.qscale()
        w.put(qscale, 5)
        w.put(0, 1)
        f, r_size = 1 << (f_code - 1), f_code - 1
        fb, r_size_b = 1 << (f_code_b - 1), f_code_b - 1
        sf, sb = (2 if full_pel else 1), (2 if full_pel_b else 1)
        pf = [0, 0]   # forward predictors (bitstream units), kept by macroblocks that do not use them
        pb = [0, 0]
        last = None   # (uses forward, uses backward) of the previous macroblock; None = intra / slice start
        dc = [128, 128, 128]
        addr = row * mbw - 1
        mb = first_mb
        first = True
        while mb <= last_mb:
            skipped = 0
            if not first and last is not None and rng.random() < self.k.b_skip_prob and mb < last_mb:
                # skipped macroblocks repeat the previous one's prediction: its vectors must fit where they land
                want = int(min(rng.integers(1, self.k.max_skip + 1), last_mb - mb))
                while skipped < want:
                    r2, c2 = divmod(mb + skipped, mbw)
                    if last[0] and not self.skip_keeps_domain(c2, r2, pf[0] * sf, pf[1] * sf):
                        break
                    if last[1] and not self.skip_keeps_domain(c2, r2, pb[0] * sb, pb[1] * sb):
                        break
                    skipped += 1
                mb += skipped
            if skipped:
                dc = [128, 128, 128]
            self.last_mb_bit = len(w.bits)
            self.address_increment(w, mb - addr)
            addr = mb
            first = False
            mb_row, mb_col = divmod(mb, mbw)
            if rng.random() < self.k.b_intra_prob:
                mtype = 0x11 if rng.random() < self.k.quant_change_prob else 0x01
            else:
                mtype = int(rng.choice([0x0C, 0x0E, 0x04, 0x06, 0x08, 0x0A, 0x1E, 0x1A, 0x16]))
            w.code(TYPE_B_CODE[mtype])
            if mtype & 0x10:
                qscale = self.qscale()
                w.put(qscale, 5)
            intra = mtype & 0x01
            if intra:
                pf = [0, 0]
                pb = [0, 0]
                last = None
            else:
                dc = [128, 128, 128]
                if mtype & 0x08:
                    th, tv = self.pick_vector(mb_col, mb_row, f, full_pel)
                    pf[0] = self.motion_component(w, th, pf[0], f, r_size)
                    pf[1] = self.motion_component(w, tv, pf[1], f, r_size)
                if mtype & 0x04:
                    th, tv = self.pick_vector(mb_col, mb_row, fb, full_pel_b)
                    pb[0] = self.motion_component(w, th, pb[0], fb, r_size_b)
                    pb[1] = self.motion_component(w, tv, pb[1], fb, r_size_b)
                last = (bool(mtype & 0x08), bool(mtype & 0x04))
            if mtype & 0x02:
                cbp = int(rng.integers(1, 64))
                w.code(CBP_CODE[cbp])
            else:
                cbp = 0x3F if intra else 0
            for blk in range(6):
                if cbp & (0x20 >> blk):
                    which = 0 if blk < 4 else blk - 3
                    dc[which] = self.block(w, intra, blk < 4, dc[which], which)
            mb += 1
        w.align()
        return w.tobytes()

    # ---------------------------------------------------------------- pictures
    def picture(self, index):
        rng = self.rng
        k = self.k
        ptype = 1 if index % k.gop == 0 else 2
        if k.b_frames:  # coded order: a reference picture, then the B pictures shown before it
            ref, pos = divmod(index, k.b_frames + 1)
            ptype = 3 if pos else (1 if ref % k.gop == 0 else 2)
        if ptype == 1 and k.gop_headers:
            self.gop_header()
        if k.repeat_sequence_header and index and ptype == 1:
            self.sequence_header()
        if k.ignored_pictures and index % 3 == 2:
            # a picture the reference skips: B type, D type or a P picture with forward_f_code 0
            kind = int(rng.integers(0, 3))
            if kind == 0:
                self.picture_header(index, 3, 0, 1)
                self.out.align()
                self.out.bits.extend(BitWriter_bits(self.slice(1, 0, self.mbw - 1, 1, 0)))
            elif kind == 1:
                self.picture_header(index, 4)
            else:
                self.picture_header(index, 2, 0, 0)
                self.out.align()
                self.out.bits.extend(BitWriter_bits(self.slice(1, 0, self.mbw - 1, 1, 0)))
        f_code = int(rng.choice(k.f_codes))
        full_pel = int(rng.random() < k.full_pel_prob)
        f_code_b, full_pel_b = 1, 0
        if ptype == 3:
            f_code_b = int(rng.choice(k.b_f_codes))
            full_pel_b = int(rng.random() < k.full_pel_prob)
        self.picture_header(index, ptype, full_pel, f_code, full_pel_b, f_code_b)
        total = self.mbw * self.mbh
        if k.slices == "one":
            spans = [(0, total - 1)]
        elif k.slices == "rows":
            spans = [(r * self.mbw, (r + 1) * self.mbw - 1) for r in range(self.mbh)]
        else:
            spans = []
            at = 0
            while at < total:
                # a slice must start where its start code says: row of its first macroblock
                length = int(rng.integers(1, 2 * self.mbw + 1))
                end = min(total - 1, at + length - 1)
                spans.append((at, end))
                at = end + 1
                if at < total and index >= k.gap_from_picture and rng.random() < k.slice_gap_prob:
                    at = min(total, at + int(rng.integers(1, self.mbw)))
        if self.mbh > MAX_SLICE_ROW + 1:
            # slice start codes end at 0xAF (row 174): the slice that starts in the last row a code can name runs to
            # the picture's end, and a slice that would start further down is not written
            spans = [s for s in spans if s[0] // self.mbw <= MAX_SLICE_ROW]
            spans[-1] = (spans[-1][0], total - 1)
        self.out.align()
        for (a, b) in spans:
            self.out.bits.extend(BitWriter_bits(self.slice(ptype, a, b, f_code, full_pel, f_code_b, full_pel_b)))

    def generate(self):
        self.sequence_header()
        for i in range(self.k.pictures):
            self.picture(i)
        # a trailing sequence_end_code, like FFmpeg writes
        self.out.start_code(0xB7)
        return self.out.tobytes()


def BitWriter_bits(data: bytes):
    return np.unpackbits(np.frombuffer(data, dtype=np.uint8)).tolist()


# Named corner-case streams used by the tests and committed (as ES + reference checksums) under
# tests/golden/ by tools/make_golden.py.
CASES = {
    "i_only_320x240": dict(knobs=dict(width=320, height=240, pictures=8, gop=1, slices="one"), seed=11),
    "rows_ip": dict(knobs=dict(width=96, height=64, pictures=10, gop=4, slices="rows"), seed=12),
    "random_slices_gaps": dict(knobs=dict(width=112, height=80, pictures=10, gop=5, slices="random", slice_gap_prob=0.3), seed=13),
    "fcodes_fullpel": dict(knobs=dict(width=176, height=144, pictures=10, gop=5, slices="rows", f_codes=(1, 2, 3, 4, 5, 6, 7),
                                      full_pel_prob=0.4, skip_prob=0.05), seed=14),
    "escapes_matrices": dict(knobs=dict(width=64, height=48, pictures=8, gop=4, slices="one", escape_prob=0.5, big_escape_prob=0.5,
                                        custom_matrices=True, max_coefs=20), seed=15),
    "skips_stuffing_escape_mba": dict(knobs=dict(width=720, height=32, pictures=8, gop=4, slices="one", skip_prob=0.5, max_skip=80,
                                                 stuffing_prob=0.3, intra_in_p_prob=0.05), seed=16),
    "ignored_pictures_userdata": dict(knobs=dict(width=96, height=64, pictures=9, gop=3, slices="rows", ignored_pictures=True,
                                                 extension_user_data=True, repeat_sequence_header=True), seed=17),
    "odd_size": dict(knobs=dict(width=100, height=50, pictures=6, gop=3, slices="random"), seed=18),
}

# B-picture streams (the opt-in extension; the reference skips every B picture of them).  Not part of CASES:
# the golden vectors of tests/golden/ come from the compiled reference, which cannot decode these.
B_CASES = {
    "b_rows": dict(knobs=dict(width=96, height=64, pictures=13, gop=2, slices="rows", b_frames=2), seed=21),
    "b_one_slice_fcodes": dict(knobs=dict(width=176, height=144, pictures=10, gop=3, slices="one", b_frames=2, f_codes=(1, 2, 3, 4),
                                          b_f_codes=(1, 2, 3, 4, 5), full_pel_prob=0.3, b_skip_prob=0.35), seed=22),
    "b_random_slices": dict(knobs=dict(width=112, height=80, pictures=9, gop=2, slices="random", b_frames=1, stuffing_prob=0.2,
                                       escape_prob=0.3, custom_matrices=True), seed=23),
    "b_three": dict(knobs=dict(width=64, height=48, pictures=12, gop=1, slices="one", b_frames=3, b_intra_prob=0.3), seed=24),
}


# Streams over the whole motion-vector domain (Knobs.vectors), I/P and I/P/B, every macroblock of every picture coded
# (no slice gaps).  The compiled reference decodes the I/P ones whose taps all lie inside the planes ("wide", "wrap"):
# tests/golden/reference/decodes.json holds its decodes of them.
VECTOR_CASES = {
    "vec_wide_720p": dict(knobs=dict(width=1280, height=720, pictures=4, gop=4, slices="rows", f_codes=(4, 5, 6, 7),
                                     full_pel_prob=0.3, vectors="wide"), seed=31),
    "vec_wide_1080p": dict(knobs=dict(width=1920, height=1080, pictures=3, gop=3, slices="one", f_codes=(5, 6, 7),
                                      full_pel_prob=0.3, vectors="wide"), seed=32),
    "vec_wrap": dict(knobs=dict(width=176, height=144, pictures=6, gop=3, slices="rows", f_codes=(2, 3, 4, 5),
                                full_pel_prob=0.3, vectors="wrap"), seed=33),
    "vec_outside": dict(knobs=dict(width=112, height=80, pictures=6, gop=3, slices="random", f_codes=(1, 2, 3, 5, 7),
                                   full_pel_prob=0.3, vectors="outside"), seed=34),
    "vec_mixed": dict(knobs=dict(width=160, height=96, pictures=6, gop=3, slices="one", f_codes=(2, 3, 4, 6),
                                 full_pel_prob=0.3, vectors="mixed"), seed=35),
    "vec_wide_b": dict(knobs=dict(width=1280, height=720, pictures=7, gop=2, slices="rows", b_frames=2, f_codes=(4, 6),
                                  b_f_codes=(5, 7), full_pel_prob=0.3, vectors="wide"), seed=36),
    "vec_wrap_b": dict(knobs=dict(width=176, height=144, pictures=10, gop=2, slices="rows", b_frames=2,
                                  f_codes=(2, 3, 4), b_f_codes=(3, 4, 5), full_pel_prob=0.3, b_skip_prob=0.35,
                                  vectors="wrap"), seed=37),
    "vec_outside_b": dict(knobs=dict(width=112, height=80, pictures=10, gop=2, slices="random", b_frames=2,
                                     f_codes=(1, 3, 7), b_f_codes=(2, 4, 6), full_pel_prob=0.3, b_skip_prob=0.35,
                                     vectors="outside"), seed=38),
    "vec_mixed_b": dict(knobs=dict(width=160, height=96, pictures=10, gop=2, slices="one", b_frames=3, f_codes=(2, 4),
                                   b_f_codes=(3, 5), full_pel_prob=0.3, b_skip_prob=0.35, vectors="mixed"), seed=39),
}


# Streams over the value domain of intra DC and coefficients (the Knobs after `vectors`): DC predictors far outside
# 0..255 -- past +-4095 (where 8 * dc leaves int16), past the intra DC clamp of stage 2's records (+-16,000) and up to
# about +-300,000 -- next to AC coefficients that make dc + ac(x) cross 0 and 255; every escape form, quantiser scales 0
# and 31, matrix entries 0 and 255.  Every DC walk is reset in between by slice starts, non-intra macroblocks or skips,
# depending on the case.  The compiled reference decodes every I and P picture of them: tests/golden/reference/decodes.json
# holds its decodes.
_CROSS = dict(ac_cross_prob=0.35, escape_forms="all", qscales=(31,))
VALUE_CASES = {
    "val_repro_96x16": None,  # value_repro(): the smallest stream that shows the 8 * dc saturation
    "val_i_one_slice_300k": dict(knobs=dict(width=320, height=240, pictures=2, gop=1, slices="one", dc_walk=("climb", "descend", "wander"),
                                            dc_step=(250, 255), dc_only_prob=0.1, **_CROSS), seed=41),
    "val_i_one_slice_down": dict(knobs=dict(width=320, height=240, pictures=1, gop=1, slices="one", dc_walk=("descend", "wander", "climb"),
                                            dc_step=(250, 255), dc_only_prob=0.1, **_CROSS), seed=42),
    "val_i_rows_wander": dict(knobs=dict(width=352, height=96, pictures=3, gop=1, slices="rows", dc_walk=("wander", "wander", "wander"),
                                         dc_run=12, dc_limit=20_000, **_CROSS), seed=43),
    "val_i_random_slices": dict(knobs=dict(width=176, height=144, pictures=3, gop=1, slices="random", dc_walk=("wander", "climb", "descend"),
                                           dc_limit=40_000, **_CROSS), seed=44),
    "val_p_intra_resets": dict(knobs=dict(width=352, height=64, pictures=6, gop=3, slices="one", dc_walk=("wander", "climb", "descend"),
                                          dc_limit=24_000, intra_in_p_prob=0.85, skip_prob=0.04, max_skip=3, **_CROSS), seed=45),
    "val_lanes_640x480": dict(knobs=dict(width=640, height=480, pictures=2, gop=2, slices="one", dc_walk=("wander", "wander", "wander"),
                                         dc_run=40, dc_limit=30_000, intra_in_p_prob=0.6, skip_prob=0.02, max_skip=2, ac_cross_prob=0.2,
                                         escape_forms="all", qscales=(31,)), seed=46),
    "val_quant_matrices": dict(knobs=dict(width=96, height=64, pictures=6, gop=3, slices="rows", custom_matrices=True,
                                          matrix_entries=(0, 1, 255, 255, 37), qscales=(0, 31, 31, 1), escape_prob=0.5,
                                          big_escape_prob=0.5, escape_forms="all", max_coefs=20, dc_walk=("wander", "wander", "wander"),
                                          dc_run=8, dc_limit=9_000, ac_cross_prob=0.2), seed=47),
    "val_quant_default": dict(knobs=dict(width=112, height=48, pictures=6, gop=2, slices="one", qscales=(0, 31), escape_prob=0.6,
                                         escape_forms="all", max_coefs=24, dc_walk=("climb", "keep", "descend"), dc_limit=12_000), seed=48),
}

# B-picture streams over the same value domain: intra macroblocks of B pictures (decode_b).  No reference decodes of the
# B pictures (the reference skips them); their expected values come from the oracle.
VALUE_B_CASES = {
    "val_b_intra": dict(knobs=dict(width=320, height=96, pictures=7, gop=2, slices="one", b_frames=2, b_intra_prob=0.85, b_skip_prob=0.05,
                                   intra_in_p_prob=0.5, dc_walk=("climb", "wander", "descend"), dc_limit=60_000, **_CROSS), seed=49),
    "val_b_rows": dict(knobs=dict(width=176, height=64, pictures=7, gop=2, slices="rows", b_frames=1, b_intra_prob=0.9,
                                  dc_walk=("wander", "climb", "wander"), dc_run=10, dc_limit=20_000, **_CROSS), seed=50),
}


# Streams over the picture's geometry and the spread of its bits, I/P and every macroblock coded: from one macroblock
# (one lane of the lane walk) and a 1x1 display to 4095x4095 (256 x 256 macroblocks, the bit fields' whole range);
# 256 one-macroblock rows; 250 rows, where the slice that starts in row 174 (code 0xAF, the last) spans the rest; and
# letterboxed pictures whose black bars -- many short macroblocks -- overflow a lane's share of the lane walk's staging
# area, so that it stores its records in a second pass.  The compiled reference decodes the cases whose taps all stay
# inside the planes (GEOMETRY_REFERENCE_CASES): tests/golden/reference/decodes.json holds its decodes of them.
_LETTERBOX = dict(pictures=3, gop=2, slices="one", profile="letterbox", bar=0.12)
GEOMETRY_CASES = {
    "geo_1mb": dict(knobs=dict(width=16, height=16, pictures=8, gop=4, slices="one", f_codes=(1, 2, 3), vectors="mixed"), seed=61),
    "geo_1x1": dict(knobs=dict(width=1, height=1, pictures=6, gop=3, slices="one"), seed=62),
    "geo_column": dict(knobs=dict(width=16, height=4095, pictures=4, gop=2, slices="rows", f_codes=(1, 2, 3), vectors="wrap"), seed=63),
    "geo_row": dict(knobs=dict(width=4095, height=16, pictures=6, gop=3, slices="random", f_codes=(1, 3, 5)), seed=64),
    "geo_max": dict(knobs=dict(width=4095, height=4095, pictures=2, gop=2, slices="one", max_coefs=4, skip_prob=0.05), seed=65),
    "geo_tall_rows": dict(knobs=dict(width=336, height=4000, pictures=3, gop=2, slices="rows", max_coefs=6), seed=66),
    "geo_odd_4k": dict(knobs=dict(width=4070, height=2303, pictures=2, gop=2, slices="random", max_coefs=4, skip_prob=0.05), seed=67),
    "geo_letterbox_720p": dict(knobs=dict(width=1280, height=720, **_LETTERBOX), seed=68),
    "geo_letterbox_1080p": dict(knobs=dict(width=1920, height=1088, **_LETTERBOX), seed=69),
    # all the detail in the first macroblock row, dense enough that the bars below fill whole lanes
    "geo_letterbox_qcif": dict(knobs=dict(width=176, height=144, **dict(_LETTERBOX, bar=(0.0, 0.9)), max_coefs=63,
                                          dc_only_prob=0.0), seed=70),
    "geo_flat_1080p": dict(knobs=dict(width=1920, height=1080, pictures=3, gop=2, slices="one", profile="flat"), seed=71),
}
# B-picture twins (decode_b) of the smallest and the most lopsided pictures
GEOMETRY_B_CASES = {
    "geo_1mb_b": dict(knobs=dict(width=16, height=16, pictures=10, gop=2, slices="one", b_frames=2, f_codes=(1, 2, 3),
                                 b_f_codes=(1, 2, 3), vectors="mixed"), seed=72),
    "geo_column_b": dict(knobs=dict(width=16, height=4095, pictures=7, gop=2, slices="rows", b_frames=2, f_codes=(1, 2),
                                    b_f_codes=(1, 2), vectors="wrap", b_skip_prob=0.35), seed=73),
    "geo_row_b": dict(knobs=dict(width=4095, height=16, pictures=7, gop=2, slices="random", b_frames=2, f_codes=(1, 3),
                                 b_f_codes=(2, 4)), seed=74),
}
# the I/P cases the compiled reference decodes: every tap inside its planes ("outside" taps read the reference's heap)
GEOMETRY_REFERENCE_CASES = sorted(n for n, c in GEOMETRY_CASES.items() if c["knobs"].get("vectors") != "mixed")


def value_repro():
    """A 96x16 I picture, one slice, quantiser scale 31, six intra macroblocks whose luma DC differentials are all
    +255: the Y predictor is 128 + 17 * 255 = 4463 at block 0 of macroblock 4, which also carries escapes of level -255
    at zig-zag positions 1-11.  Saturating 8 * dc at 32767 changes its samples (255 in the reference)."""
    s = SynthStream(Knobs(width=96, height=16, pictures=1, gop=1, slices="one"), 0)
    s.sequence_header()
    s.gop_header()
    s.picture_header(0, 1)
    s.out.align()
    w = BitWriter()
    w.start_code(1)
    w.put(31, 5)
    w.put(0, 1)
    for mb in range(6):
        w.code(MBA_CODE[1])
        w.code(TYPE_I_CODE[0x01])
        for blk in range(6):
            if blk < 4:
                w.code(DC_LUMA_CODE[8])
                w.put(255, 8)
            else:
                w.code(DC_CHROMA_CODE[0])
            if mb == 4 and blk == 0:
                for _ in range(11):
                    s.escape_level(w, 0, -255)
            w.code(V.DCT_EOB_CODE)
    w.align()
    s.out.bits.extend(w.bits)
    s.out.start_code(0xB7)
    return s.out.tobytes()


def make_case(name):
    if name == "val_repro_96x16":
        return value_repro()
    spec = next(c[name] for c in (CASES, B_CASES, VECTOR_CASES, VALUE_CASES, VALUE_B_CASES, GEOMETRY_CASES, GEOMETRY_B_CASES)
                if name in c)
    return SynthStream(Knobs(**spec["knobs"]), spec["seed"]).generate()


if __name__ == "__main__":
    for name in list(CASES) + list(B_CASES):
        es = make_case(name)
        print(f"{name}: {len(es)} bytes")
