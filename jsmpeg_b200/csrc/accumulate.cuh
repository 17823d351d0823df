// accumulate.cuh -- one depth step of the accumulated map for one 8x8 block (DESIGN 3.11): the block code of
// accumulate_kernel (accumulate.cu).  The same text compiles for the host when JSMPEG_WALK_EMU is defined
// (tests/emu/accumulate_check.cpp), as recon.cuh and idct.cuh do.
//
// A map record is {dx, dy, residual, back}, int16 each, held as a uint2: x = dx | dy << 16, y = residual | back << 16.
#pragma once
#include <string.h>

#include "common.cuh"

namespace {

constexpr uint32_t ACC_UNTRACED = 0xffff0000u;  // record word y of an untraced sample: residual 0, back -1

__device__ __forceinline__ int acc_sat16(int x) { return x < -32768 ? -32768 : (x > 32767 ? 32767 : x); }
__device__ __forceinline__ uint32_t acc_pack(int lo, int hi) { return (uint32_t)(uint16_t)lo | (uint32_t)hi << 16; }

__device__ __forceinline__ uint2 acc_load(const uint2 *p) {
#ifndef JSMPEG_WALK_EMU
	return __ldg(p);
#else
	uint2 v;
	memcpy(&v, p, sizeof v);
	return v;
#endif
}

__device__ __forceinline__ void acc_store(uint2 *p, uint2 a, uint2 b) {  // two records, one 16-byte store
	const uint4 v = make_uint4(a.x, a.y, b.x, b.y);
#ifndef JSMPEG_WALK_EMU
	*reinterpret_cast<uint4 *>(p) = v;
#else
	memcpy(p, &v, sizeof v);
#endif
}

// The map of block b (0-3 luma, 4 Cb, 5 Cr) of macroblock (mb_row, mb_col) of a picture of W x H macroblocks into
// `dst`, from the macroblock's record words `rec` (x: the forward vector, y: flags | cbp << 8 | ...), the block's
// residual v (raster order; read only for a traced block) and `prev`, the previous reference picture's map (nullptr:
// none).  Per sample i of the block:
//   macroblock not PRESENT                          untraced (0, 0, 0, -1)
//   INTRA, or the prediction not inside the plane    the trace ends here (0, 0, 0, 0)
//   otherwise, p = prev[i + (mv >> 1) * stride + (mh >> 1)] (the sample's first prediction tap):
//     p untraced (or no prev)                        untraced
//     else                                           (sat16(p.dx + mh), sat16(p.dy + mv), sat16(p.residual + v), p.back + 1)
// with (mh, mv) the plane's vector: luma as recorded, chroma halved with truncation toward zero (as stage 2).  Each
// row reads eight consecutive records of prev (64 bytes, 8-byte aligned) and writes eight (four 16-byte stores).
__device__ __forceinline__ void accumulate_block(uint2 rec, int b, int mb_row, int mb_col, int W, int H, const int (&v)[64],
                                                 const uint2 *prev, uint2 *dst) {
	const int stride_y = W * 16;
	const int ysize = stride_y * H * 16;
	int stride, plane_off, plane_size, origin;
	if (b < 4) {
		stride = stride_y; plane_off = 0; plane_size = ysize;
		origin = (mb_row * 16 + (b >> 1) * 8) * stride + mb_col * 16 + (b & 1) * 8;
	} else {
		stride = stride_y >> 1; plane_size = ysize >> 2;
		plane_off = b == 4 ? ysize + plane_size : ysize;  // Cb is the third plane, Cr the second
		origin = mb_row * 8 * stride + mb_col * 8;
	}
	const int flags = rec.y & 0xff;
	const bool present = flags & MBF_PRESENT;
	int mh = (int)(int16_t)(rec.x & 0xffffu), mv = (int)(int16_t)(rec.x >> 16);
	if (b >= 4) { mh /= 2; mv /= 2; }
	const int src = origin + (mv >> 1) * stride + (mh >> 1);
	const bool predicted = present && !(flags & MBF_INTRA) && PREDICTION_INSIDE(src, stride, plane_size, mh & 1, mv & 1);
	const bool traced = predicted && prev != nullptr;
	// what a sample that reads nothing back gets: the end of a trace (rule 2), else untraced
	const uint2 none = make_uint2(0u, present && !predicted ? 0u : ACC_UNTRACED);
	uint2 *out = dst + plane_off + origin;
	const uint2 *in = traced ? prev + plane_off + src : nullptr;
#pragma unroll
	for (int r = 0; r < 8; r++) {
		uint2 o[8];
#pragma unroll
		for (int c = 0; c < 8; c++) {
			o[c] = none;
			if (traced) {
				const uint2 p = acc_load(in + r * stride + c);
				const int back = (int)(int16_t)(p.y >> 16);
				if (back >= 0)
					o[c] = make_uint2(acc_pack(acc_sat16((int)(int16_t)(p.x & 0xffffu) + mh), acc_sat16((int)(int16_t)(p.x >> 16) + mv)),
					                  acc_pack(acc_sat16((int)(int16_t)(p.y & 0xffffu) + v[r * 8 + c]), back + 1));
			}
		}
#pragma unroll
		for (int c = 0; c < 8; c += 2) acc_store(out + r * stride + c, o[c], o[c + 1]);
	}
}

}  // namespace
