#!/usr/bin/env python
"""Synthetic MPEG-1 video test clips (MPEG-TS, program streams, raw ES) encoded with cv2's bundled FFmpeg (mpeg1video encoder +
mpegts muxer), SURVEY.md section 7 step 0(a) / section 8(d).

Content is seeded numpy: low-resolution noise upsampled bicubically (smooth, moving background),
a moving disc, and +-noise uniform noise per sample.  cv2 gives no bitrate/GOP control: FFmpeg's
defaults apply (GOP 12 = 1 I + 11 P, no B pictures, one slice per picture).

Clips are cached under $JSMPEG_B200_CACHE (default jsmpeg_b200_cache_<uid> in the system temporary
directory, one per user, so that another user's cache never blocks a write) because encoding 1080p
takes seconds.
"""
from __future__ import annotations

import hashlib
import os
import sys
import tempfile

import numpy as np

CACHE = os.environ.get("JSMPEG_B200_CACHE", os.path.join(tempfile.gettempdir(), f"jsmpeg_b200_cache_{os.getuid()}"))


def make_clip_ts(width, height, frames, seed=1234, noise=6, fps=30):
    """Returns the bytes of an MPEG-TS clip (video PID 0x100, stream id 0xE0)."""
    return _make_clip("ts", width, height, frames, seed, noise, fps)


def make_clip_ps(width, height, frames, seed=1234, noise=6, fps=30, form="mpg"):
    """The same encode in a program stream: form "mpg" = FFmpeg's mpeg muxer (ISO 11172-1 packs and PES),
    "vob" = its vob muxer (ISO 13818-1 packs and PES).  Video stream id 0xE0."""
    if form not in ("mpg", "vob"):
        raise ValueError(f"form {form!r}: 'mpg' or 'vob'")
    return _make_clip(form, width, height, frames, seed, noise, fps)


def make_clip_m1v(width, height, frames, seed=1234, noise=6, fps=30):
    """The same encode as a raw MPEG-1 video elementary stream."""
    return _make_clip("m1v", width, height, frames, seed, noise, fps)


def _make_clip(ext, width, height, frames, seed, noise, fps):
    """Encodes the scene; FFmpeg picks the container from the file extension."""
    import cv2

    os.makedirs(CACHE, exist_ok=True)
    tag = "v2" if ext == "ts" else f"v2-{ext}"
    key = hashlib.sha1(f"{tag}-{width}x{height}-{frames}-{seed}-{noise}-{fps}-{cv2.__version__}".encode()).hexdigest()[:16]
    path = os.path.join(CACHE, f"clip_{width}x{height}_{frames}f_s{seed}_{key}.{ext}")
    if os.path.exists(path):
        with open(path, "rb") as f:
            return f.read()
    rng = np.random.default_rng(seed)
    lo = rng.integers(0, 256, (height // 32 + 3, width // 32 + 3, 3), dtype=np.uint8)
    base = cv2.resize(lo, (width + 64, height + 64), interpolation=cv2.INTER_CUBIC).astype(np.int16)
    tmp = path + f".{os.getpid()}.tmp.{ext}"
    devnull = os.open(os.devnull, os.O_WRONLY)
    saved = os.dup(2)
    os.dup2(devnull, 2)  # FFmpeg prints a harmless "tag mpg1 not supported" warning
    try:
        vw = cv2.VideoWriter(tmp, cv2.CAP_FFMPEG, cv2.VideoWriter_fourcc(*"mpg1"), fps, (width, height))
        if not vw.isOpened():
            raise RuntimeError(f"cv2/FFmpeg cannot open an mpeg1video .{ext} writer")
        for i in range(frames):
            dx, dy = (i * 3) % 64, (i * 2) % 64
            f = base[dy:dy + height, dx:dx + width].copy()
            cx = width // 2 + int(width / 3 * np.sin(i / 7.0))
            cy = height // 2 + int(height / 3 * np.cos(i / 9.0))
            cv2.circle(f, (cx, cy), max(height // 8, 4), (255, 64, 32), -1)
            if noise:
                f += rng.integers(-noise, noise + 1, f.shape, dtype=np.int16)
            vw.write(np.clip(f, 0, 255).astype(np.uint8))
        vw.release()
    finally:
        os.dup2(saved, 2)
        os.close(devnull)
        os.close(saved)
    os.replace(tmp, path)
    with open(path, "rb") as f:
        return f.read()


def make_clip_es(width, height, frames, seed=1234, noise=6):
    """Demuxed video PES payloads [(pts, bytes)...] of make_clip_ts (host demux, jsmpeg_b200/ts.py)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    from jsmpeg_b200.ts import demux_video_es

    return demux_video_es(make_clip_ts(width, height, frames, seed, noise))


if __name__ == "__main__":
    for (w, h, n) in [(320, 240, 24), (1280, 720, 60), (1920, 1080, 60)]:
        pk = make_clip_es(w, h, n)
        total = sum(len(p) for _, p in pk)
        print(f"{w}x{h}: {len(pk)} pictures, {total} ES bytes, {total / len(pk):.0f} B/picture, {total * 8 * 30 / len(pk) / 1e6:.1f} Mbit/s @30")
