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

}  // namespace

int launch_reconstruct(const ReconTask *tasks_host, int n_tasks, cudaStream_t stream) {
	int launches = 0;
	for (int first = 0; first < n_tasks; first += MAX_TASKS, launches++) {
		const int n = n_tasks - first < MAX_TASKS ? n_tasks - first : MAX_TASKS;
		ReconParams p;
		int max_slots = 0;
		for (int i = 0; i < n; i++) {
			const ReconTask &t = tasks_host[first + i];
			fill_task(p.t[i], t);
			max_slots = max_slots > t.mb_size * 6 ? max_slots : t.mb_size * 6;
		}
		p.n_tasks = n;
		dim3 grid((max_slots + THREADS - 1) / THREADS, n);
		reconstruct_kernel<<<grid, THREADS, 0, stream>>>(p);
	}
	return launches;
}

int launch_reconstruct_rgba(const ReconTask *tasks_host, int n_tasks, cudaStream_t stream) {
	int launches = 0;
	for (int first = 0; first < n_tasks; first += MAX_TASKS_RGBA, launches++) {
		const int n = n_tasks - first < MAX_TASKS_RGBA ? n_tasks - first : MAX_TASKS_RGBA;
		ReconRgbaParams p;
		int max_w = 0, max_h = 0;
		for (int i = 0; i < n; i++) {
			const ReconTask &t = tasks_host[first + i];
			fill_task(p.p.t[i], t);
			p.out[i] = RgbaTarget{t.rgba, t.width, t.height};
			max_w = max_w > t.mb_width ? max_w : t.mb_width;
			const int h = t.mb_size / t.mb_width;
			max_h = max_h > h ? max_h : h;
		}
		p.p.n_tasks = n;
		dim3 grid((max_w + RGBA_MBS - 1) / RGBA_MBS, max_h, n);
		reconstruct_rgba_kernel<<<grid, RGBA_THREADS, 0, stream>>>(p);
	}
	return launches;
}

int launch_reconstruct_b(const ReconTask *tasks_host, int n_tasks, bool rgba, cudaStream_t stream) {
	int launches = 0;
	const int per = rgba ? MAX_TASKS_RGBA_B : MAX_TASKS_B;
	for (int first = 0; first < n_tasks; first += per, launches++) {
		const int n = n_tasks - first < per ? n_tasks - first : per;
		int max_slots = 0, max_w = 0, max_h = 0;
		for (int i = 0; i < n; i++) {
			const ReconTask &t = tasks_host[first + i];
			max_slots = max_slots > t.mb_size * 6 ? max_slots : t.mb_size * 6;
			max_w = max_w > t.mb_width ? max_w : t.mb_width;
			const int h = t.mb_size / t.mb_width;
			max_h = max_h > h ? max_h : h;
		}
		if (rgba) {
			ReconRgbaParamsB p;
			for (int i = 0; i < n; i++) {
				const ReconTask &t = tasks_host[first + i];
				fill_task(p.p.t[i], t);
				p.p.t[i].bwd = t.bwd.y;
				p.out[i] = RgbaTarget{t.rgba, t.width, t.height};
			}
			p.p.n_tasks = n;
			dim3 grid((max_w + RGBA_MBS - 1) / RGBA_MBS, max_h, n);
			reconstruct_rgba_b_kernel<<<grid, RGBA_THREADS, 0, stream>>>(p);
		} else {
			ReconParamsB p;
			for (int i = 0; i < n; i++) {
				const ReconTask &t = tasks_host[first + i];
				fill_task(p.t[i], t);
				p.t[i].bwd = t.bwd.y;
			}
			p.n_tasks = n;
			dim3 grid((max_slots + THREADS - 1) / THREADS, n);
			reconstruct_b_kernel<<<grid, THREADS, 0, stream>>>(p);
		}
	}
	return launches;
}
