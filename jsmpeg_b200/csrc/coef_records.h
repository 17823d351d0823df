/*
 * coef_records.h -- the compact coefficient record that stage 1b (expand) hands stage 2 (reconstruct).
 *
 * A coded block of a typical stream carries a handful of coefficients (about 4.6 on average, 99.45 % of them at
 * most 12), yet its dense record (records.h) is 64 x int16 = 128 bytes.  The compact record is 32 bytes per block
 * slot mb * 6 + b:
 *     uint64_t mask       bit k set <=> zig-zag position k was written by the block's codes
 *     int16_t  level[12]  the written values in zig-zag order: the k-th set bit of `mask` goes with level[k]
 * The values are exactly those of the dense record: dequantised, oddified, clipped, intra DC as dc (records.h).  Positions
 * inside a block only increase (run >= 0; a store past position 63 is dropped), so the order is well defined.
 * A block with more than COEF_RECORD_LEVELS positions has mask == COEF_RECORD_DENSE: its dense 128-byte record
 * holds it, at its usual place in the coefficient plane.  Uncoded blocks write and read nothing.
 *
 * This header is the only place that knows the layout; the expand, reconstruct, coefficient and residual export
 * kernels, the host engine's debug hooks and the tests all go through it.  It compiles as CUDA (host and device) and as plain C++.
 */
#ifndef JSMPEG_B200_COEF_RECORDS_H
#define JSMPEG_B200_COEF_RECORDS_H

#include <stdint.h>

#ifdef __CUDACC__
#define COEF_FN __host__ __device__ __forceinline__
#else
#define COEF_FN static inline
#endif

#define COEF_RECORD_LEVELS 12
#define COEF_RECORD_DENSE (~(uint64_t)0) /* mask value: the block lives in the dense coefficient plane */

struct alignas(32) coef_record_t {
	uint64_t mask;
	int16_t level[COEF_RECORD_LEVELS];
};
static_assert(sizeof(coef_record_t) == 32, "one 32-byte record per block slot");

COEF_FN int coef_popc64(uint64_t x) {
#ifdef __CUDA_ARCH__
	return __popcll(x);
#else
	return __builtin_popcountll(x);
#endif
}

// index of the lowest set bit of a nonzero x
COEF_FN int coef_lowest64(uint64_t x) {
#ifdef __CUDA_ARCH__
	return __ffsll((long long)x) - 1;
#else
	return __builtin_ctzll(x);
#endif
}

// raster index of zig-zag position k (0..63) (ISO 11172-2 2.4.4.1, the reference's ZIG_ZAG).  The scan runs along
// the anti-diagonals d = row + col, down-left on odd d and up-right on even d, and is symmetric about the centre:
// raster(63 - k) = 63 - raster(k), so the second half mirrors the first.
COEF_FN int coef_zigzag_raster(int k) {
	const bool first = k < 36;
	const int j = first ? k : 63 - k;
	const int d = (j >= 1) + (j >= 3) + (j >= 6) + (j >= 10) + (j >= 15) + (j >= 21) + (j >= 28);
	const int o = j - d * (d + 1) / 2;  // step along the diagonal
	const int row = (d & 1) ? o : d - o;
	const int r = row * 8 + (d - row);
	return first ? r : 63 - r;
}

// zig-zag position of raster index r (0..63), the inverse of coef_zigzag_raster: on anti-diagonal d = row + col < 8
// the position is d (d + 1) / 2 plus the step along it (row on odd d, col on even d); the rest mirrors about the centre.
COEF_FN int coef_raster_zigzag(int r) {
	const bool first = (r >> 3) + (r & 7) < 8;
	const int j = first ? r : 63 - r;
	const int row = j >> 3, col = j & 7, d = row + col;
	const int k = d * (d + 1) / 2 + ((d & 1) ? row : col);
	return first ? k : 63 - k;
}

// raster row `row` (0..7) of a compact record (mask != COEF_RECORD_DENSE): out[c] = value at raster row * 8 + c.
// Per value: its zig-zag position k, bit k of the mask, and the level index popc(mask & ((1 << k) - 1)); the levels
// are read as three 64-bit words selected by that index, so nothing is indexed at run time (no local memory on the
// device) and no value takes a branch.  An index of 12 (bit clear, 12 positions below) selects a word too; the clear
// bit discards it.
COEF_FN void coef_record_row(const coef_record_t &r, int row, int16_t out[8]) {
	uint64_t w[3] = {0, 0, 0};
	for (int i = 0; i < COEF_RECORD_LEVELS; i++) w[i >> 2] |= (uint64_t)(uint16_t)r.level[i] << (16 * (i & 3));
	for (int c = 0; c < 8; c++) {
		const int k = coef_raster_zigzag(row * 8 + c);
		const int idx = coef_popc64(r.mask & ((((uint64_t)1) << k) - 1));
		const uint64_t word = idx < 4 ? w[0] : (idx < 8 ? w[1] : w[2]);
		const int16_t v = (int16_t)(uint16_t)(word >> (16 * (idx & 3)));
		out[c] = ((r.mask >> k) & 1) ? v : (int16_t)0;
	}
}

// the values of a compact record (mask != COEF_RECORD_DENSE) into their raster places of a block whose other values
// the caller has set: at most COEF_RECORD_LEVELS stores, and no index into the record at run time
COEF_FN void coef_record_scatter(const coef_record_t &r, int16_t *raster) {
	uint64_t m = r.mask;
	for (int k = 0; k < COEF_RECORD_LEVELS; k++) {
		if (m) {
			raster[coef_zigzag_raster(coef_lowest64(m))] = r.level[k];
			m &= m - 1;
		}
	}
}

// coefficient 0 of a compact record (mask != COEF_RECORD_DENSE): the first level when zig-zag position 0 is written
COEF_FN int coef_record_dc(const coef_record_t &r) { return (r.mask & 1) ? r.level[0] : 0; }

// whether a block with the zig-zag positions `written` fits a compact record
COEF_FN bool coef_record_fits(uint64_t written) { return coef_popc64(written) <= COEF_RECORD_LEVELS; }

// the compact record of a block from its dense raster values and the zig-zag positions its codes wrote
// (coef_record_fits(written) must hold); unused levels are 0
COEF_FN coef_record_t coef_record_pack(uint64_t written, const int16_t *raster) {
	coef_record_t r;
	r.mask = written;
	for (int k = 0; k < COEF_RECORD_LEVELS; k++) {
		r.level[k] = 0;
		if (written) {
			r.level[k] = raster[coef_zigzag_raster(coef_lowest64(written))];
			written &= written - 1;
		}
	}
	return r;
}

// the dense raster values of a compact record (mask != COEF_RECORD_DENSE)
COEF_FN void coef_record_unpack(const coef_record_t &r, int16_t *raster) {
	for (int i = 0; i < 64; i++) raster[i] = 0;
	uint64_t m = r.mask;
	for (int k = 0; m; k++, m &= m - 1) raster[coef_zigzag_raster(coef_lowest64(m))] = r.level[k];
}

// the zig-zag positions of the nonzero values of a dense raster block: for a block whose codes are not at hand
// (a zero level adds nothing to the transform, so packing these positions reproduces the block)
COEF_FN uint64_t coef_nonzero_positions(const int16_t *raster) {
	uint64_t m = 0;
	for (int k = 0; k < 64; k++)
		if (raster[coef_zigzag_raster(k)]) m |= (uint64_t)1 << k;
	return m;
}

#endif
