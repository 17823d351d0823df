// conceal.cuh -- the per-macroblock copy of the opt-in `conceal` option (DESIGN 3.19), kept apart from its kernel
// shell (conceal.cu) so that the host compiler builds it too: with JSMPEG_WALK_EMU defined,
// tests/emu/conceal_check.cpp runs it between the emulated expand and reconstruct.
//
// A macroblock whose record lacks MBF_PRESENT gets the co-located samples of the picture's forward plane set (16x16
// luma, 8x8 Cr and Cb: zero motion, a plain copy), written into the destination set before stage 2 runs.  Stage 2
// leaves such a macroblock alone, so everything it derives from the set (RGBA, planar frame, host copy, later
// predictions) sees the copy.  A PRESENT macroblock is not touched.
#pragma once
#include "common.cuh"

// Request i conceals one picture: `mb_size` macroblock records at `hdr`, `mb_width` macroblocks to a row, samples
// from `fwd` into `cur` (planes of mb_width * 16 luma samples to a row).  `first` is the number of macroblocks of
// requests 0 .. i-1.
struct ConcealTask {
	const mb_record_t *hdr;
	PlaneSet cur;
	PlaneSet fwd;
	int32_t mb_width, mb_size;
	uint32_t first;
	int32_t pad;
};
// One warp per macroblock of all `n_tasks` requests (`total_mb` macroblocks), one launch (conceal.cu)
void launch_conceal(const ConcealTask *tasks, int n_tasks, uint32_t total_mb, cudaStream_t stream);

// Lane `lane` (0..31) of the warp that handles macroblock `mb` of `t`.  Lanes 0-15 copy luma row `lane` (16 bytes),
// lanes 16-23 Cr rows 0-7 and lanes 24-31 Cb rows 0-7 (8 bytes each).  Luma rows are 16-byte aligned and chroma rows
// 8-byte aligned: a plane set's planes start 16-byte aligned and a row holds a multiple of 16 (8) samples.
__host__ __device__ inline void conceal_macroblock(const ConcealTask &t, int mb, int lane) {
	if (t.hdr[mb].flags & MBF_PRESENT) return;
	const int row = mb / t.mb_width, col = mb - row * t.mb_width;
	if (lane < 16) {
		const size_t stride = (size_t)t.mb_width * 16;
		const size_t at = ((size_t)row * 16 + lane) * stride + (size_t)col * 16;
		*reinterpret_cast<uint4 *>(t.cur.y + at) = *reinterpret_cast<const uint4 *>(t.fwd.y + at);
	} else {
		const int r = lane & 7;
		const size_t stride = (size_t)t.mb_width * 8;
		const size_t at = ((size_t)row * 8 + r) * stride + (size_t)col * 8;
		uint8_t *dst = lane < 24 ? t.cur.cr : t.cur.cb;
		const uint8_t *src = lane < 24 ? t.fwd.cr : t.fwd.cb;
		*reinterpret_cast<uint2 *>(dst + at) = *reinterpret_cast<const uint2 *>(src + at);
	}
}
