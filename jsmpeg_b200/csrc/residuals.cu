// residuals.cu -- export of the pixel-domain residual, the inverse transform of every block, into the public layout
// (sm_90a), for jsmpeg_b200_batch_decode_residuals (engine.cu, DESIGN 3.10).
//
// One thread per 8x8 block.  A warp takes 32 consecutive block slots of one request in stage 2's numbering
// (reconstruct_block, recon.cuh): per macroblock row [luma top 2W | luma bottom 2W | Cb W | Cr W], so the 32 lanes
// hold horizontally adjacent blocks of one plane row, each of a lane's 8 output rows is one 16-byte store and a warp's
// row store is 512 contiguous bytes.  Each request's 6 * mb_size slots are rounded up to whole warps, so a warp
// belongs to one request; the grid runs over the warps of all requests of a wave, and a warp finds its request by the
// 32-ary search of export_coefficients_kernel over the per-request prefix `first`.
//
// One path per warp, as in stage 2: a warp with no block that needs the transform (every block uncoded, DC-only or
// outside the picture) stores zeros or the DC shortcut's constant; otherwise every lane runs the transform --
// uncoded lanes on zeros, DC-only lanes on their record (which the transform turns into the shortcut's value).  A
// coded block's values come from its compact record, scattered (coef_record_scatter) into a zeroed row of shared
// memory owned by the lane, or, for a block marked dense, from its dense record as it is.  Every store is streaming:
// nothing rereads the residual.
#include <string.h>

#include "common.cuh"
#include "idct.cuh"

namespace {

constexpr int RES_WARPS = 4;  // warps per CTA
constexpr int RES_PITCH = 144;  // bytes per lane's staging row: 128 + 16 (the 16-byte accesses of a warp spread over the banks)

__global__ void __launch_bounds__(RES_WARPS * 32)
export_residuals_kernel(const ResExportTask *__restrict__ tasks, int n_tasks, uint32_t total_warps) {
	__shared__ __align__(16) uint8_t stage[RES_WARPS][32 * RES_PITCH];
	const uint32_t warp = blockIdx.x * RES_WARPS + threadIdx.x / 32;
	if (warp >= total_warps) return;  // (the whole warp)
	const int lane = threadIdx.x & 31;
	// the last request with first <= warp (export_coefficients_kernel's search)
	int lo = 0, len = n_tasks;
	while (len > 1) {
		const int step = (len + 31) >> 5;
		const int at = lo + lane * step;
		const unsigned below = __ballot_sync(~0u, lane * step < len && __ldg(&tasks[at].first) <= warp);
		const int j = 31 - __clz(below);  // (lane 0's probe, first[lo] <= warp, always holds)
		lo += j * step;
		len = min(step, len - j * step);
	}
	const ResExportTask t = tasks[lo];
	const int W = t.mb_width;
	const int slot = (int)(warp - t.first) * 32 + lane;
	const bool in_picture = slot < 6 * W * t.mb_height;
	// block b of macroblock (mb_row, mb_col), as reconstruct_block numbers the slots
	const int mb_row = in_picture ? slot / (6 * W) : 0;
	const int s = in_picture ? slot - mb_row * 6 * W : 0;
	int b, mb_col;
	if (s < 4 * W) {
		const int by = s >= 2 * W;
		const int bx = s - by * 2 * W;
		mb_col = bx >> 1;
		b = by * 2 + (bx & 1);
	} else {
		const int c = s - 4 * W;
		const int second = c >= W;
		mb_col = c - second * W;
		b = 4 + second;  // block 4 -> Cb plane, block 5 -> Cr plane
	}
	const int mb = mb_row * W + mb_col;
	// flags (byte 0), cbp (byte 1) and dc_only (byte 2) of the record's second word
	const uint32_t rec = in_picture ? __ldg(reinterpret_cast<const uint32_t *>(t.hdr + mb) + 1) : 0u;
	const uint32_t bit = 0x20u >> b;
	const bool coded = (rec & MBF_PRESENT) && ((rec >> 8) & bit);
	const bool full = coded && !((rec >> 16) & bit);
	coef_record_t cr;
	cr.mask = 0;
	if (coded) {
		const uint4 *crec = reinterpret_cast<const uint4 *>(t.compact + (size_t)mb * 6 + b);
		const uint4 c0 = __ldg(crec), c1 = __ldg(crec + 1);
		memcpy(&cr, &c0, 16);
		memcpy(reinterpret_cast<uint8_t *>(&cr) + 16, &c1, 16);
	}
	const bool dense = coded && cr.mask == COEF_RECORD_DENSE;
	const uint4 *drec = reinterpret_cast<const uint4 *>(t.coef + ((size_t)mb * 6 + b) * 64);  // (a dense block's 8 rows)

	int v[64];
	if (__any_sync(~0u, full)) {
		uint4 q[8];
		if (dense) {
#pragma unroll
			for (int i = 0; i < 8; i++) q[i] = __ldg(drec + i);
		} else if (coded) {
			uint8_t *row = stage[threadIdx.x / 32] + lane * RES_PITCH;
#pragma unroll
			for (int i = 0; i < 8; i++) reinterpret_cast<uint4 *>(row)[i] = make_uint4(0u, 0u, 0u, 0u);
			coef_record_scatter(cr, reinterpret_cast<int16_t *>(row));
#pragma unroll
			for (int i = 0; i < 8; i++) q[i] = reinterpret_cast<const uint4 *>(row)[i];
		} else {
#pragma unroll
			for (int i = 0; i < 8; i++) q[i] = make_uint4(0u, 0u, 0u, 0u);
		}
		idct_block(q, v);
	} else {
		const int c0 = !coded ? 0 : (dense ? (int)__ldg(t.coef + ((size_t)mb * 6 + b) * 64) : coef_record_dc(cr));
		const int dc = coded ? idct_dc(c0) : 0;
#pragma unroll
		for (int i = 0; i < 64; i++) v[i] = dc;
	}
	if (!in_picture) return;

	const int stride_y = W * 16;
	const int ysize = stride_y * t.mb_height * 16;
	int stride, origin;
	if (b < 4) {
		stride = stride_y;
		origin = (mb_row * 16 + (b >> 1) * 8) * stride + mb_col * 16 + (b & 1) * 8;
	} else {
		stride = stride_y >> 1;
		origin = (b == 4 ? ysize + (ysize >> 2) : ysize) + mb_row * 8 * stride + mb_col * 8;  // Cb third, Cr second
	}
	int16_t *dst = t.dst + origin;
#pragma unroll
	for (int r = 0; r < 8; r++) {
		const uint4 o = make_uint4(__byte_perm(v[r * 8 + 0], v[r * 8 + 1], 0x5410), __byte_perm(v[r * 8 + 2], v[r * 8 + 3], 0x5410),
		                           __byte_perm(v[r * 8 + 4], v[r * 8 + 5], 0x5410), __byte_perm(v[r * 8 + 6], v[r * 8 + 7], 0x5410));
		__stcs(reinterpret_cast<uint4 *>(dst + r * stride), o);
	}
}

}  // namespace

void launch_export_residuals(const ResExportTask *tasks, int n_tasks, uint32_t total_warps, cudaStream_t stream) {
	if (n_tasks <= 0 || total_warps == 0) return;
	export_residuals_kernel<<<(total_warps + RES_WARPS - 1) / RES_WARPS, RES_WARPS * 32, 0, stream>>>(tasks, n_tasks, total_warps);
	CUDA_CHECK(cudaGetLastError());
}
