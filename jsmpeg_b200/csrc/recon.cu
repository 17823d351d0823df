// recon.cu -- stage 2: integer IDCT + half-pel motion compensation + add/clamp -> planar Y/Cr/Cb.
//
// Replaces the pixel half of the reference's decodeMacroblock/decodeBlock: copyMacroblock
// (src/mpeg1.js:459-687), IDCT (:916-983) and Copy/Add{Block,Value}ToDestination (:864-914).
// Every macroblock of a picture reads only the PREVIOUS picture's planes and writes only its own
// 16x16 / 8x8 / 8x8 pixels, so all blocks of a picture (and of all streams) are independent.
//
// Mapping: ONE THREAD PER 8x8 BLOCK, the whole block in registers.
//   * the block's 32-byte compact coefficient record (coef_records.h: position mask + at most 12
//     values) is loaded with two LDG.128; the lane zeroes its 144-byte-pitched row of the warp's
//     staging area and scatters the values into it.  A block with more values has a dense
//     128-byte record: it is fetched by ONE instruction per lane, a TMA 1-D bulk copy
//     (cp.async.bulk global -> shared, SASS UBLKCP) into the row, completion counted on a
//     per-warp mbarrier.  Either way the lane then reads its row back with eight conflict-free
//     LDS.128.  (Eight per-lane LDG.128 at a 128-byte stride cost 32 L1 wavefronts per
//     instruction and made the kernel L1TEX-bound.)
//     The coefficients are multiplied by PREMULTIPLIER (src/mpeg1.js:810, 1026-1035) -- compile-time immediates,
//     the loops are fully unrolled -- and go through the 8 column passes (mpeg1.js:925-947) and
//     the 8 row passes with (v+128)>>8 (mpeg1.js:952-981) without leaving the register file:
//     no shared memory, no barriers, all per-thread overhead amortised over 64 samples;
//   * blocks are numbered so that the 32 lanes of a warp hold 32 horizontally adjacent blocks of
//     one plane row ([luma top | luma bottom | Cb | Cr] per macroblock row): every row of the
//     output is one 8-byte store per lane = 256 contiguous bytes per warp, and the forward-plane
//     fetches of neighbouring lanes (similar vectors) fall into the same sectors;
//   * prediction: 9 (+9) samples per row as three aligned 32-bit words + funnel shifts; per
//     output sample one PRMT gathers the four taps and one dp4a applies the lane's half-pel tap
//     weights (exact (a+b+1)>>1 / (a+b+c+d+2)>>2, mpeg1.js:481-556, for every parity with the
//     same instruction stream); + residual, saturate (cvt.pack.sat), store.
//   * the kernel is bound by the integer ALU pipe, so multiplies/byte selects go to the dot-product
//     unit where possible: dp2a for coefficient x premultiplier, dp4a for the taps.
// Blocks taking the reference's DC-only shortcut (mpeg1.js:838-841, 850-853) skip the IDCT.
// The per-launch task table (pointers + sizes per stream) travels in the kernel parameters
// (constant bank), so the first global access of a thread is already its macroblock header.
// A vector whose footprint leaves the plane (non-conforming, SURVEY Q11) takes a per-tap
// bounds-checked path.
//
// HBM roofline accounting (DESIGN.md): per macroblock 16 B header + 32 B per coded block (its
// compact record; the about 0.5 % of blocks with a dense record are not counted) + 384 B written +
// 384 B of forward-plane samples (P pictures), each counted once.
#include <algorithm>
#include <vector>

#include "recon.cuh"

namespace {

// H100, 60 launches per 64 x 1080p x 60 step: 20.9 ms with 5 resident CTAs per SM, 21.8 ms with 4, 25.8 ms
// with 6 (register cap too low)
#ifndef JSMPEG_RECON_MIN_CTAS
#define JSMPEG_RECON_MIN_CTAS 5
#endif
__global__ void __launch_bounds__(THREADS, JSMPEG_RECON_MIN_CTAS)
reconstruct_kernel(const __grid_constant__ ReconParams params) {
	__shared__ __align__(16) uint8_t stage[(THREADS / 32) * WARP_STAGE];
	reconstruct_block(params, blockIdx.y, blockIdx.x * THREADS, threadIdx.x, stage);
}

// OUT_RGBA: the same reconstruction with the planar -> RGBA conversion fused in (recon.cuh)
struct ReconRgbaParams {
	ReconParamsT<MAX_TASKS_RGBA> p;
	RgbaTarget out[MAX_TASKS_RGBA];
};
static_assert(sizeof(ReconRgbaParams) <= 4096, "kernel parameters");

__global__ void __launch_bounds__(RGBA_THREADS)
reconstruct_rgba_kernel(const __grid_constant__ ReconRgbaParams params) {
	__shared__ __align__(16) uint8_t stage[(RGBA_THREADS / 32) * WARP_STAGE];
	__shared__ __align__(16) uint8_t chroma[2][8][RGBA_MBS * 8];
	reconstruct_rgba_block(params.p, params.out[blockIdx.z], blockIdx.z, blockIdx.y, blockIdx.x * RGBA_MBS, threadIdx.x, stage, chroma);
}

// B pictures (the opt-in extension): the same two kernels instantiated for two references
__global__ void __launch_bounds__(THREADS, JSMPEG_RECON_MIN_CTAS)
reconstruct_b_kernel(const __grid_constant__ ReconParamsB params) {
	__shared__ __align__(16) uint8_t stage[(THREADS / 32) * WARP_STAGE];
	reconstruct_block<true>(params, blockIdx.y, blockIdx.x * THREADS, threadIdx.x, stage);
}

constexpr int MAX_TASKS_RGBA_B = 48;  // (48 * (56 + 16) B) + 16 < 4 KB
struct ReconRgbaParamsB {
	struct { CompactTaskB t[MAX_TASKS_RGBA_B]; int32_t n_tasks; } p;
	RgbaTarget out[MAX_TASKS_RGBA_B];
};
static_assert(sizeof(ReconParamsB) <= 4096 && sizeof(ReconRgbaParamsB) <= 4096, "kernel parameters");

__global__ void __launch_bounds__(RGBA_THREADS)
reconstruct_rgba_b_kernel(const __grid_constant__ ReconRgbaParamsB params) {
	__shared__ __align__(16) uint8_t stage[(RGBA_THREADS / 32) * WARP_STAGE];
	__shared__ __align__(16) uint8_t chroma[2][8][RGBA_MBS * 8];
	reconstruct_rgba_block<true>(params.p, params.out[blockIdx.z], blockIdx.z, blockIdx.y, blockIdx.x * RGBA_MBS, threadIdx.x, stage, chroma);
}

// OUT_RESIDUALS (DESIGN 3.15): the four kernels above, each block also storing its residual (reconstruct_at<..., RES>),
// with the tables of ReconResParamsT (recon.cuh)
constexpr int MAX_TASKS_RES = 72;         // (72 * (48 + 8) B) + 8 < 4 KB
constexpr int MAX_TASKS_RGBA_RES = 56;    // (56 * (48 + 8 + 16) B) + 8 < 4 KB
constexpr int MAX_TASKS_B_RES = 63;       // (63 * (56 + 8) B) + 8 < 4 KB
constexpr int MAX_TASKS_RGBA_B_RES = 51;  // (51 * (56 + 8 + 16) B) + 8 < 4 KB
using ReconResParams = ReconResParamsT<CompactTask, MAX_TASKS_RES>;
using ReconResParamsB = ReconResParamsT<CompactTaskB, MAX_TASKS_B_RES>;
struct ReconRgbaResParams {
	ReconResParamsT<CompactTask, MAX_TASKS_RGBA_RES> p;
	RgbaTarget out[MAX_TASKS_RGBA_RES];
};
struct ReconRgbaResParamsB {
	ReconResParamsT<CompactTaskB, MAX_TASKS_RGBA_B_RES> p;
	RgbaTarget out[MAX_TASKS_RGBA_B_RES];
};
static_assert(sizeof(ReconResParams) <= 4096 && sizeof(ReconResParamsB) <= 4096 && sizeof(ReconRgbaResParams) <= 4096 &&
              sizeof(ReconRgbaResParamsB) <= 4096, "kernel parameters");

__global__ void __launch_bounds__(THREADS, JSMPEG_RECON_MIN_CTAS)
reconstruct_res_kernel(const __grid_constant__ ReconResParams params) {
	__shared__ __align__(16) uint8_t stage[(THREADS / 32) * WARP_STAGE];
	reconstruct_block<false, true>(params, blockIdx.y, blockIdx.x * THREADS, threadIdx.x, stage);
}

__global__ void __launch_bounds__(RGBA_THREADS)
reconstruct_rgba_res_kernel(const __grid_constant__ ReconRgbaResParams params) {
	__shared__ __align__(16) uint8_t stage[(RGBA_THREADS / 32) * WARP_STAGE];
	__shared__ __align__(16) uint8_t chroma[2][8][RGBA_MBS * 8];
	reconstruct_rgba_block<false, true>(params.p, params.out[blockIdx.z], blockIdx.z, blockIdx.y, blockIdx.x * RGBA_MBS, threadIdx.x, stage, chroma);
}

// (at 5 resident CTAs, 96 registers, the B variant's residual store spills -- reconstruct_b_kernel spills there too, on
// its per-tap path; at 4, 128 registers, it does not)
#ifndef JSMPEG_RECON_RES_B_MIN_CTAS
#define JSMPEG_RECON_RES_B_MIN_CTAS 4
#endif
__global__ void __launch_bounds__(THREADS, JSMPEG_RECON_RES_B_MIN_CTAS)
reconstruct_res_b_kernel(const __grid_constant__ ReconResParamsB params) {
	__shared__ __align__(16) uint8_t stage[(THREADS / 32) * WARP_STAGE];
	reconstruct_block<true, true>(params, blockIdx.y, blockIdx.x * THREADS, threadIdx.x, stage);
}

__global__ void __launch_bounds__(RGBA_THREADS)
reconstruct_rgba_res_b_kernel(const __grid_constant__ ReconRgbaResParamsB params) {
	__shared__ __align__(16) uint8_t stage[(RGBA_THREADS / 32) * WARP_STAGE];
	__shared__ __align__(16) uint8_t chroma[2][8][RGBA_MBS * 8];
	reconstruct_rgba_block<true, true>(params.p, params.out[blockIdx.z], blockIdx.z, blockIdx.y, blockIdx.x * RGBA_MBS, threadIdx.x, stage, chroma);
}

// decode_frames (DESIGN 3.16): the four RES kernels, each block also storing its output rows to the task's planar frame
// (reconstruct_at<..., FRAME>), with the tables of ReconFrameParamsT (recon.cuh)
constexpr int MAX_TASKS_FRAME = 63;         // (63 * (48 + 8 + 8) B) + 8 < 4 KB
constexpr int MAX_TASKS_RGBA_FRAME = 51;    // (51 * (48 + 8 + 8 + 16) B) + 8 < 4 KB
constexpr int MAX_TASKS_B_FRAME = 56;       // (56 * (56 + 8 + 8) B) + 8 < 4 KB
constexpr int MAX_TASKS_RGBA_B_FRAME = 46;  // (46 * (56 + 8 + 8 + 16) B) + 8 < 4 KB
using ReconFrameParams = ReconFrameParamsT<CompactTask, MAX_TASKS_FRAME>;
using ReconFrameParamsB = ReconFrameParamsT<CompactTaskB, MAX_TASKS_B_FRAME>;
struct ReconRgbaFrameParams {
	ReconFrameParamsT<CompactTask, MAX_TASKS_RGBA_FRAME> p;
	RgbaTarget out[MAX_TASKS_RGBA_FRAME];
};
struct ReconRgbaFrameParamsB {
	ReconFrameParamsT<CompactTaskB, MAX_TASKS_RGBA_B_FRAME> p;
	RgbaTarget out[MAX_TASKS_RGBA_B_FRAME];
};
static_assert(sizeof(ReconFrameParams) <= 4096 && sizeof(ReconFrameParamsB) <= 4096 && sizeof(ReconRgbaFrameParams) <= 4096 &&
              sizeof(ReconRgbaFrameParamsB) <= 4096, "kernel parameters");

// (at 5 resident CTAs, 96 registers, the I/P variant spills 36 bytes; at 4, 126 registers, it does not.  The B variant
// uses 128 registers at 4, like reconstruct_res_b_kernel, and does not spill.)
#ifndef JSMPEG_RECON_FRAME_MIN_CTAS
#define JSMPEG_RECON_FRAME_MIN_CTAS 4
#endif
__global__ void __launch_bounds__(THREADS, JSMPEG_RECON_FRAME_MIN_CTAS)
reconstruct_frame_kernel(const __grid_constant__ ReconFrameParams params) {
	__shared__ __align__(16) uint8_t stage[(THREADS / 32) * WARP_STAGE];
	reconstruct_block<false, true, true>(params, blockIdx.y, blockIdx.x * THREADS, threadIdx.x, stage);
}

__global__ void __launch_bounds__(RGBA_THREADS)
reconstruct_rgba_frame_kernel(const __grid_constant__ ReconRgbaFrameParams params) {
	__shared__ __align__(16) uint8_t stage[(RGBA_THREADS / 32) * WARP_STAGE];
	__shared__ __align__(16) uint8_t chroma[2][8][RGBA_MBS * 8];
	reconstruct_rgba_block<false, true, true>(params.p, params.out[blockIdx.z], blockIdx.z, blockIdx.y, blockIdx.x * RGBA_MBS, threadIdx.x, stage, chroma);
}

__global__ void __launch_bounds__(THREADS, JSMPEG_RECON_FRAME_MIN_CTAS)
reconstruct_frame_b_kernel(const __grid_constant__ ReconFrameParamsB params) {
	__shared__ __align__(16) uint8_t stage[(THREADS / 32) * WARP_STAGE];
	reconstruct_block<true, true, true>(params, blockIdx.y, blockIdx.x * THREADS, threadIdx.x, stage);
}

__global__ void __launch_bounds__(RGBA_THREADS)
reconstruct_rgba_frame_b_kernel(const __grid_constant__ ReconRgbaFrameParamsB params) {
	__shared__ __align__(16) uint8_t stage[(RGBA_THREADS / 32) * WARP_STAGE];
	__shared__ __align__(16) uint8_t chroma[2][8][RGBA_MBS * 8];
	reconstruct_rgba_block<true, true, true>(params.p, params.out[blockIdx.z], blockIdx.z, blockIdx.y, blockIdx.x * RGBA_MBS, threadIdx.x, stage, chroma);
}

void fill_task(CompactTask &c, const ReconTask &t) {
	c.hdr = t.hdr;
	c.coef = t.coef;
	c.compact = t.compact;
	c.cur = t.cur.y;   // planes are contiguous: Y | Cr | Cb (engine.cu plane_set)
	c.fwd = t.fwd.y;
	c.mb_width = t.mb_width;
	c.mb_height = t.mb_size / t.mb_width;
	c.row_magic = (uint32_t)(0x100000000ull / (uint64_t)(6 * t.mb_width)) + 1u;
	c.flags = 0;
}

// One kernel's tasks, cut into launches of at most `per`: B = the kernel takes `bwd`, RGBA = it takes the fused
// conversion's target, RES = it takes the residual destinations, FRAME = also the planar frames.  The plain kernels'
// grid covers the largest picture's block slots, the RGBA kernels' its macroblock rows and columns.
template <bool B, bool RGBA, bool RES = false, bool FRAME = false, class Params>
int launch_kernel(void (*kernel)(Params), int per, const std::vector<const ReconTask *> &tasks, cudaStream_t stream) {
	int launches = 0;
	for (size_t first = 0; first < tasks.size(); first += per, launches++) {
		const int n = (int)std::min<size_t>(per, tasks.size() - first);
		Params p;
		auto &table = [&]() -> auto & { if constexpr (RGBA) return p.p; else return p; }();
		int max_slots = 0, max_w = 0, max_h = 0;
		for (int i = 0; i < n; i++) {
			const ReconTask &t = *tasks[first + i];
			fill_task(table.t[i], t);
			if constexpr (B) table.t[i].bwd = t.bwd.y;
			if constexpr (RGBA) p.out[i] = RgbaTarget{t.rgba, t.width, t.height};
			if constexpr (RES) table.res[i] = t.res;
			if constexpr (FRAME) table.frame[i] = t.frame;
			max_slots = std::max(max_slots, t.mb_size * 6);
			max_w = std::max(max_w, t.mb_width);
			max_h = std::max(max_h, t.mb_size / t.mb_width);
		}
		table.n_tasks = n;
		if constexpr (RGBA) kernel<<<dim3((max_w + RGBA_MBS - 1) / RGBA_MBS, max_h, n), RGBA_THREADS, 0, stream>>>(p);
		else kernel<<<dim3((max_slots + THREADS - 1) / THREADS, n), THREADS, 0, stream>>>(p);
	}
	return launches;
}

}  // namespace

int launch_reconstruct(const ReconTask *tasks_host, int n_tasks, cudaStream_t stream) {
	std::vector<const ReconTask *> by_kernel[4];  // I/P, I/P + RGBA, B, B + RGBA
	bool res[4] = {false, false, false, false};   // some task of the kernel has a residual destination: its RES variant
	bool frame[4] = {false, false, false, false}; // some task of the kernel has a planar frame: its FRAME variant
	for (int i = 0; i < n_tasks; i++) {
		const ReconTask &t = tasks_host[i];
		const int k = (t.bwd.y ? 2 : 0) + (t.rgba ? 1 : 0);
		by_kernel[k].push_back(&t);
		res[k] = res[k] || t.res;
		frame[k] = frame[k] || t.frame;
	}
	// (one statement per kernel: the launch order is the order above)
	int launches = frame[0] ? launch_kernel<false, false, true, true>(reconstruct_frame_kernel, MAX_TASKS_FRAME, by_kernel[0], stream)
	             : res[0]   ? launch_kernel<false, false, true>(reconstruct_res_kernel, MAX_TASKS_RES, by_kernel[0], stream)
	                        : launch_kernel<false, false>(reconstruct_kernel, MAX_TASKS, by_kernel[0], stream);
	launches += frame[1] ? launch_kernel<false, true, true, true>(reconstruct_rgba_frame_kernel, MAX_TASKS_RGBA_FRAME, by_kernel[1], stream)
	          : res[1]   ? launch_kernel<false, true, true>(reconstruct_rgba_res_kernel, MAX_TASKS_RGBA_RES, by_kernel[1], stream)
	                     : launch_kernel<false, true>(reconstruct_rgba_kernel, MAX_TASKS_RGBA, by_kernel[1], stream);
	launches += frame[2] ? launch_kernel<true, false, true, true>(reconstruct_frame_b_kernel, MAX_TASKS_B_FRAME, by_kernel[2], stream)
	          : res[2]   ? launch_kernel<true, false, true>(reconstruct_res_b_kernel, MAX_TASKS_B_RES, by_kernel[2], stream)
	                     : launch_kernel<true, false>(reconstruct_b_kernel, MAX_TASKS_B, by_kernel[2], stream);
	launches += frame[3] ? launch_kernel<true, true, true, true>(reconstruct_rgba_frame_b_kernel, MAX_TASKS_RGBA_B_FRAME, by_kernel[3], stream)
	          : res[3]   ? launch_kernel<true, true, true>(reconstruct_rgba_res_b_kernel, MAX_TASKS_RGBA_B_RES, by_kernel[3], stream)
	                     : launch_kernel<true, true>(reconstruct_rgba_b_kernel, MAX_TASKS_RGBA_B, by_kernel[3], stream);
	return launches;
}
