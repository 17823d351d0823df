// accumulate.cu -- one chain depth of the accumulated motion and residual maps (sm_90a), for
// jsmpeg_b200_batch_decode_accumulated (engine.cu, DESIGN 3.11).
//
// The geometry of export_residuals_kernel (residuals.cu): one thread per 8x8 block, a warp on 32 horizontally adjacent
// blocks of one task in stage 2's numbering, each task's 6 * mb_size block slots rounded up to whole warps, and a
// warp finds its task by the 32-ary ballot search over the per-task prefix `first`.  One launch covers the pictures of
// one depth of every chain of a wave; each reads the map the launch before it wrote for the same chain.
//
// A lane transforms its block (idct.cuh) only when the block is coded and traced from (PRESENT, not INTRA), with the
// one-path-per-warp rule of residuals.cu: a warp with no such block that needs the full transform takes the DC
// shortcut's constant (0 for an uncoded block), otherwise every lane runs the transform.  accumulate_block
// (accumulate.cuh) then gathers and stores the block's map rows.
#include <string.h>

#include "accumulate.cuh"
#include "common.cuh"
#include "idct.cuh"

namespace {

constexpr int ACC_WARPS = 4;     // warps per CTA
constexpr int ACC_PITCH = 144;   // bytes per lane's staging row (residuals.cu's RES_PITCH)

__global__ void __launch_bounds__(ACC_WARPS * 32)
accumulate_kernel(const AccTask *__restrict__ tasks, int n_tasks, uint32_t total_warps) {
	__shared__ __align__(16) uint8_t stage[ACC_WARPS][32 * ACC_PITCH];
	const uint32_t warp = blockIdx.x * ACC_WARPS + threadIdx.x / 32;
	if (warp >= total_warps) return;  // (the whole warp)
	const int lane = threadIdx.x & 31;
	// the last task with first <= warp (export_residuals_kernel's search)
	int lo = 0, len = n_tasks;
	while (len > 1) {
		const int step = (len + 31) >> 5;
		const int at = lo + lane * step;
		const unsigned below = __ballot_sync(~0u, lane * step < len && __ldg(&tasks[at].first) <= warp);
		const int j = 31 - __clz(below);
		lo += j * step;
		len = min(step, len - j * step);
	}
	const AccTask t = tasks[lo];
	const int W = t.mb_width;
	const int slot = (int)(warp - t.first) * 32 + lane;
	const bool in_picture = slot < 6 * W * t.mb_height;
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
		b = 4 + second;
	}
	const int mb = mb_row * W + mb_col;
	const uint2 rec = in_picture ? __ldg(reinterpret_cast<const uint2 *>(t.hdr + mb)) : make_uint2(0u, 0u);
	const uint32_t bit = 0x20u >> b;
	const bool coded = (rec.y & MBF_PRESENT) && !(rec.y & MBF_INTRA) && ((rec.y >> 8) & bit);
	const bool full = coded && !((rec.y >> 16) & bit);
	coef_record_t cr;
	cr.mask = 0;
	if (coded) {
		const uint4 *crec = reinterpret_cast<const uint4 *>(t.compact + (size_t)mb * 6 + b);
		const uint4 c0 = __ldg(crec), c1 = __ldg(crec + 1);
		memcpy(&cr, &c0, 16);
		memcpy(reinterpret_cast<uint8_t *>(&cr) + 16, &c1, 16);
	}
	const bool dense = coded && cr.mask == COEF_RECORD_DENSE;
	const uint4 *drec = reinterpret_cast<const uint4 *>(t.coef + ((size_t)mb * 6 + b) * 64);

	int v[64];
	if (__any_sync(~0u, full)) {
		uint4 q[8];
		if (dense) {
#pragma unroll
			for (int i = 0; i < 8; i++) q[i] = __ldg(drec + i);
		} else if (coded) {
			uint8_t *row = stage[threadIdx.x / 32] + lane * ACC_PITCH;
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
	accumulate_block(rec, b, mb_row, mb_col, W, t.mb_height, v, t.prev, t.dst);
}

}  // namespace

void launch_accumulate(const AccTask *tasks, int n_tasks, uint32_t total_warps, cudaStream_t stream) {
	if (n_tasks <= 0 || total_warps == 0) return;
	accumulate_kernel<<<(total_warps + ACC_WARPS - 1) / ACC_WARPS, ACC_WARPS * 32, 0, stream>>>(tasks, n_tasks, total_warps);
	CUDA_CHECK(cudaGetLastError());
}
