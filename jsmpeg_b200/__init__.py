"""jsmpeg_b200 -- H100-native (sm_90a) MPEG-1 video decode path behind jsmpeg's decoder surface.

Only what the hot path needs lives here: ``csrc/`` (CUDA kernels + the C ABI), and the host-side
mirror of the reference interface (``decoder.MPEG1Video``, ``ts.TS``, ``batch.BatchDecoder``).
"""
from .decoder import MPEG1Video, PlaneRecorder  # noqa: F401
from .ts import TS, demux_video_es  # noqa: F401
