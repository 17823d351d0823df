// idct.cuh -- the reference's integer inverse transform of one 8x8 block (sm_90a), the one copy of it: stage 2
// (recon.cuh) adds its output to the prediction, the residual export (residuals.cu) stores it.
//
// Like recon.cuh the same text compiles for the host when JSMPEG_WALK_EMU is defined (tests/emu/walk_emu.cpp,
// tests/emu/residuals_check.cpp): `__device__` comes from cuda_runtime.h's host definitions, __dp2a_lo from the emulation.
#pragma once

namespace {

// PREMULTIPLIER_MATRIX (src/mpeg1.js:1026-1035) = outer product of these AAN scales, rounded as the
// reference's table is; kept as a constexpr so that every use folds into an immediate.
__device__ constexpr int PM[64] = {
    32, 44, 42, 38, 32, 25, 17, 9,  44, 62, 58, 52, 44, 35, 24, 12, 42, 58, 55, 49, 42, 33, 23, 12,
    38, 52, 49, 44, 38, 30, 20, 10, 32, 44, 42, 38, 32, 25, 17, 9,  25, 35, 33, 30, 25, 20, 14, 7,
    17, 24, 23, 20, 17, 14, 9,  5,  9,  12, 12, 10, 9,  7,  5,  2};

// One 8-point pass of the reference IDCT on v[o], v[o+s], ... v[o+7s].
// Column pass: no scaling; row pass: (v + 128) >> 8.
template <bool ROW, int O, int S>
__device__ __forceinline__ void idct8(int (&v)[64]) {
	const int b1 = v[O + 4 * S];
	const int b3 = v[O + 2 * S] + v[O + 6 * S];
	const int b4 = v[O + 5 * S] - v[O + 3 * S];
	const int t1 = v[O + 1 * S] + v[O + 7 * S];
	const int t2 = v[O + 3 * S] + v[O + 5 * S];
	const int b6 = v[O + 1 * S] - v[O + 7 * S];
	const int b7 = t1 + t2;
	const int m0 = v[O];
	const int x4 = ((b6 * 473 - b4 * 196 + 128) >> 8) - b7;
	const int x0 = x4 - (((t1 - t2) * 362 + 128) >> 8);
	const int x1 = m0 - b1;
	const int x2 = (((v[O + 2 * S] - v[O + 6 * S]) * 362 + 128) >> 8) - b3;
	const int x3 = m0 + b1;
	const int y3 = x1 + x2, y4 = x3 + b3, y5 = x1 - x2, y6 = x3 - b3;
	const int y7 = -x0 - ((b4 * 473 + b6 * 196 + 128) >> 8);
	if (ROW) {
		v[O] = (b7 + y4 + 128) >> 8;         v[O + 1 * S] = (x4 + y3 + 128) >> 8;
		v[O + 2 * S] = (y5 - x0 + 128) >> 8; v[O + 3 * S] = (y6 - y7 + 128) >> 8;
		v[O + 4 * S] = (y6 + y7 + 128) >> 8; v[O + 5 * S] = (x0 + y5 + 128) >> 8;
		v[O + 6 * S] = (y3 - x4 + 128) >> 8; v[O + 7 * S] = (y4 - b7 + 128) >> 8;
	} else {
		v[O] = b7 + y4;         v[O + 1 * S] = x4 + y3; v[O + 2 * S] = y5 - x0; v[O + 3 * S] = y6 - y7;
		v[O + 4 * S] = y6 + y7; v[O + 5 * S] = x0 + y5; v[O + 6 * S] = y3 - x4; v[O + 7 * S] = y4 - b7;
	}
}

template <int I>
__device__ __forceinline__ void idct_columns(int (&v)[64]) {
	if constexpr (I < 8) {
		idct8<false, I, 8>(v);
		idct_columns<I + 1>(v);
	}
}
template <int I>
__device__ __forceinline__ void idct_rows(int (&v)[64]) {
	if constexpr (I < 8) {
		idct8<true, I * 8, 1>(v);
		idct_rows<I + 1>(v);
	}
}

// The premultiplied coefficient 0: an intra block's is its dc (records.h), x 256 = the reference's dc << 8
// (src/mpeg1.js:747); any other block's is a level, x PREMULTIPLIER[0].  `lo` holds it in its low 16 bits.
__device__ __forceinline__ int premultiplied_c0(uint32_t lo, bool intra) {
	return intra ? (int)(lo << 16) >> 8 : __dp2a_lo((int)lo, PM[0], 0);
}

// The residual of one block from its 64 coefficients in raster order, eight per uint4 (int16 pairs, low half first):
// each times its premultiplier (dp2a: lo16 * byte 0 + hi16 * byte 1, one instruction per coefficient), then the
// column and the row passes -- px[] of the reference before the add or clamp (src/mpeg1.js:916-983).  `intra`: the
// block is an intra one, whose coefficient 0 is its dc (premultiplied_c0); without it, a level like any other.
__device__ __forceinline__ void idct_block(const uint4 (&q)[8], int (&v)[64], bool intra = false) {
#pragma unroll
	for (int i = 0; i < 8; i++) {
		v[i * 8 + 0] = i ? __dp2a_lo((int)q[i].x, PM[i * 8 + 0], 0) : premultiplied_c0(q[0].x, intra);
		v[i * 8 + 1] = __dp2a_lo((int)q[i].x, PM[i * 8 + 1] << 8, 0);
		v[i * 8 + 2] = __dp2a_lo((int)q[i].y, PM[i * 8 + 2], 0); v[i * 8 + 3] = __dp2a_lo((int)q[i].y, PM[i * 8 + 3] << 8, 0);
		v[i * 8 + 4] = __dp2a_lo((int)q[i].z, PM[i * 8 + 4], 0); v[i * 8 + 5] = __dp2a_lo((int)q[i].z, PM[i * 8 + 5] << 8, 0);
		v[i * 8 + 6] = __dp2a_lo((int)q[i].w, PM[i * 8 + 6], 0); v[i * 8 + 7] = __dp2a_lo((int)q[i].w, PM[i * 8 + 7] << 8, 0);
	}
	idct_columns<0>(v);
	idct_rows<0>(v);
}

// The residual of a DC-only block, every sample: the reference's shortcut (mpeg1.js:838-853), which the full
// transform of such a block equals (column 0 comes out as eight copies of the premultiplied c0, every other term of a
// row is 0): (c0 * 256 + 128) >> 8 = c0 for an intra block
__device__ __forceinline__ int idct_dc(int c0, bool intra = false) { return intra ? c0 : (c0 * PM[0] + 128) >> 8; }

}  // namespace
