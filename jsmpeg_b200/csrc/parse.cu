// parse.cu -- stage 1: bitstream / VLC parse (sm_90a), in two kernels.
//
// Replaces, for the bitstream half, the reference's decodePicture / decodeSlice / decodeMacroblock /
// decodeMotionVectors / decodeBlock (src/mpeg1.js:174-457, 698-811) and its bit reader
// (src/buffer.js:115-187).
//
// A picture is an inherently serial VLC walk: where symbol k+1 starts is only known once symbol k
// has been decoded.  Everything ELSE the reference does per symbol (run/level bookkeeping,
// zig-zag, dequantisation, oddification, clipping, the store) does not feed that chain.  So:
//
//   1a  walk_pictures_{lanes_,}kernel   one warp per PICTURE (every picture starts at a byte-aligned
//       start code and resets all predictor state in its slice headers, and nothing in the parse
//       depends on decoded pixels, so all buffered pictures of all streams are walked concurrently).
//       The walk does the minimum that is serial: macroblock headers (address increment, type,
//       quantiser, motion vectors with their predictors, coded block pattern), intra DC
//       differentials with their predictors, and for the AC coefficients only LUT -> code length
//       -> shift.  It emits the 16-byte macroblock record and, per coded block, the bit offset of
//       its first coefficient code (parked in the block's own 128-byte coefficient slot).
//       Default: the LANE-PARALLEL walk -- the 32 lanes take 32 sub-sequences of the picture's bits
//       and find the chain by VLC self-synchronisation (walk.cuh); the serial walk (all lanes on one
//       chain) is its in-kernel fall-back and, with JSMPEG_B200_WALK=serial, a kernel of its own.
//   1b  expand_blocks_kernel    one thread per coded BLOCK, all blocks of all pictures at once:
//       re-reads the block's codes from its bit offset, does run/level -> zig-zag -> dequantise ->
//       oddify -> clip (src/mpeg1.js:757-811) straight into its 32-byte compact record (coef_records.h) in
//       shared memory, which the warp stores with its neighbours' as whole 512-byte stretches; a block of more
//       than 12 values is decoded again into a 64 x int16 tile and leaves as the dense record, one TMA bulk store.
//
// VLCs are decoded with clz-indexed look-up tables in shared memory (tools/gen_tables.py; pinned
// to the reference's trees by tests/test_vlc_tables.py) instead of the reference's one-bit-per-step
// tree walk (src/mpeg1.js:66-72).  Bit window: 64-bit, MSB first, refilled one prefetched 32-bit
// word at a time.
// Output: mb_record_t per macroblock address + dequantised int16 coefficient blocks (records.h).
#include <string.h>

#include <mutex>
#include <vector>

#include "walk.cuh"
#include "walk_b.cuh"
#include "walk_slices.cuh"

namespace {

constexpr int CTA_THREADS = 128;       // expand kernel
constexpr uint32_t EXPAND_SMEM = EXP_OFF_TILES + CTA_THREADS * EXP_TILE_PITCH;

// ==================================================================================================
// 1a: one warp per picture (walk.cuh), serial or lane-parallel with serial fall-back

// the serial walk keeps the allocation it was tuned with (63 registers, no occupancy hint); the
// lane-parallel walk asks for 3 resident CTAs per SM.  Measured on an H100 (64 x 1080p x 60 pictures,
// tools/time_stages.py, two interleaved runs): walk 16.0 / 15.2 ms and step 49.6 / 51.0 ms with 3,
// against walk 19.6 / 19.7 ms and step 51.0 / 51.7 ms with 4 and walk 23.0 / 23.0 ms with 5.
#ifndef JSMPEG_LANES_MIN_CTAS
#define JSMPEG_LANES_MIN_CTAS 3
#endif
#define LANES_BOUNDS __launch_bounds__(WALK_THREADS, JSMPEG_LANES_MIN_CTAS)
#define WALK_KERNEL(NAME, LANES, BOUNDS)                                                                          \
	__global__ void BOUNDS NAME(const ParseTask *__restrict__ tasks, int n_tasks, const uint4 *__restrict__ ms_table) { \
		extern __shared__ __align__(128) uint8_t smem[];                                                          \
		walk_tables_init(smem, threadIdx.x, WALK_THREADS, ms_table, LANES);                                       \
		__syncthreads();                                                                                          \
		const int lane = threadIdx.x & 31;                                                                        \
		const int task_id = blockIdx.x * (WALK_THREADS / 32) + (threadIdx.x >> 5);                                \
		if (task_id >= n_tasks) return;                                                                           \
		const ParseTask t = tasks[task_id];                                                                       \
		const uint32_t sbase = smem_base(smem);                                                                   \
		walk_picture<LANES>(t, sbase, lane, LANES ? sbase + OFF_RING + threadIdx.x * RING_BYTES : 0u);            \
	}
WALK_KERNEL(walk_pictures_kernel, false, __launch_bounds__(WALK_THREADS))
WALK_KERNEL(walk_pictures_lanes_kernel, true, LANES_BOUNDS)

// B pictures (the opt-in extension, walk_b.cuh): the serial walk with the B-picture macroblock layer
__global__ void __launch_bounds__(WALK_THREADS)
walk_pictures_b_kernel(const ParseTask *__restrict__ tasks, int n_tasks, const uint4 *__restrict__ ms_table) {
	extern __shared__ __align__(128) uint8_t smem[];
	walk_tables_init(smem, threadIdx.x, WALK_THREADS, ms_table, false);
	__syncthreads();
	const int task_id = blockIdx.x * (WALK_THREADS / 32) + (threadIdx.x >> 5);
	if (task_id >= n_tasks) return;
	const ParseTask t = tasks[task_id];
	walk_picture_b(t, smem_base(smem), threadIdx.x & 31);
}

// pictures of many slices (opt-in, walk_slices.cuh): one lane per slice, serial walk as in-kernel fall-back
__global__ void LANES_BOUNDS
walk_pictures_slices_kernel(const ParseTask *__restrict__ tasks, int n_tasks, const uint4 *__restrict__ ms_table) {
	extern __shared__ __align__(128) uint8_t smem[];
	walk_tables_init(smem, threadIdx.x, WALK_THREADS, ms_table, true);
	__syncthreads();
	const int task_id = blockIdx.x * (WALK_THREADS / 32) + (threadIdx.x >> 5);
	if (task_id >= n_tasks) return;
	const ParseTask t = tasks[task_id];
	const uint32_t sbase = smem_base(smem);
	walk_picture_slices(t, sbase, threadIdx.x & 31, sbase + OFF_RING + threadIdx.x * RING_BYTES);
}

// ==================================================================================================
// 1b: expand every coded block (one thread per block slot, grid.y = picture)
//
// A CTA stages the tables once and then takes EXPAND_GROUPS runs of CTA_THREADS consecutive slots, one after
// the other: the warps go through their runs independently (staging areas are per warp, the tables read-only, so
// the one CTA barrier is the one after staging), and a thread asks for the next run's inputs before it expands
// the current block -- the staging, the barrier and the exposed load latency at the start of a CTA are paid
// once per EXPAND_GROUPS runs.
#ifndef JSMPEG_EXPAND_GROUPS
#define JSMPEG_EXPAND_GROUPS 4  // H100, step per 64 x 1080p x 60: 1 run 51.6 / 51.6 ms, 4 runs 51.0 / 51.7, 8 runs 51.9 / 52.2
#endif
constexpr int EXPAND_GROUPS = JSMPEG_EXPAND_GROUPS;

__global__ void __launch_bounds__(CTA_THREADS)
expand_blocks_kernel(const ParseTask *__restrict__ tasks) {
	extern __shared__ __align__(128) uint8_t smem[];
	const ParseTask &t = tasks[blockIdx.y];
	const int n_slots = t.mb_size * 6;
	// a thread's inputs: the macroblock record's second word and the pair the walk parked for the block.
	// (A picture that was not decoded has no present macroblock: the walk clears the records first.)
	auto fetch = [&](int slot_id, uint32_t &rec, uint2 &parked) {
		rec = 0;
		parked = make_uint2(0u, 0u);
		if (slot_id < n_slots) {
			rec = __ldg(reinterpret_cast<const uint32_t *>(t.hdr + slot_id / 6) + 1);
			parked = __ldg(t.park + slot_id);
		}
	};
	int slot_id = blockIdx.x * (CTA_THREADS * EXPAND_GROUPS) + threadIdx.x;  // mb * 6 + block
	uint32_t rec;
	uint2 parked;
	fetch(slot_id, rec, parked);  // requested before the tables are staged: one exposed latency, not two
	{
		// tables: the two DCT code tables of stage 1b (1536 + 1024 B, 16 bytes per thread each) and the picture's
		// two quantiser tables in zig-zag order (256 B, one entry per thread)
		static_assert(CTA_THREADS >= (VLC_DCT_MAX_Z + 1) * 8 && CTA_THREADS >= 128, "one pass stages the tables");
		if (threadIdx.x < (VLC_DCT_MAX_Z + 1) * 8)
			reinterpret_cast<uint4 *>(smem + EXP_OFF_DCT)[threadIdx.x] = __ldg(reinterpret_cast<const uint4 *>(VLC_DCT_EXPAND) + threadIdx.x);
		if (threadIdx.x < 64)
			reinterpret_cast<uint4 *>(smem + EXP_OFF_TOP8)[threadIdx.x] = __ldg(reinterpret_cast<const uint4 *>(VLC_DCT_EXPAND_TOP8) + threadIdx.x);
		if (threadIdx.x < 128)
			reinterpret_cast<uint16_t *>(smem + EXP_OFF_XQ)[threadIdx.x] = __ldg(&t.seq->xq[0][0] + threadIdx.x);
	}
	__syncthreads();
	const uint32_t sbase = smem_base(smem);
	// the warp's staging area (walk.cuh): its lanes' compact rows, or their 64 x int16 tiles
	const int lane = threadIdx.x & 31;
	const uint32_t wstage = sbase + EXP_OFF_TILES + (threadIdx.x - lane) * EXP_TILE_PITCH;
#pragma unroll 1
	for (int g = 0; g < EXPAND_GROUPS; g++) {
		const uint32_t rec_now = rec;
		const uint2 parked_now = parked;
		const int slot_now = slot_id;
		slot_id += CTA_THREADS;
		if (g + 1 < EXPAND_GROUPS) fetch(slot_id, rec, parked);  // the next run's, while this block is expanded
		const int block = slot_now % 6;
		const bool coded = slot_now < n_slots && (rec_now & MBF_PRESENT) && ((rec_now >> 8) & (0x20u >> block));
		if (!__any_sync(0xffffffffu, coded)) continue;
		expand_warp_run(t, coded, rec_now, parked_now, slot_now, lane, sbase, wstage);
	}
}

// Stage 1b of n_tasks pictures of up to max_mb_size macroblocks on `stream`
void launch_expand(const ParseTask *tasks, int n_tasks, int max_mb_size, cudaStream_t stream) {
	dim3 grid((max_mb_size * 6 + CTA_THREADS * EXPAND_GROUPS - 1) / (CTA_THREADS * EXPAND_GROUPS), n_tasks);
	expand_blocks_kernel<<<grid, CTA_THREADS, EXPAND_SMEM, stream>>>(tasks);
}

// The walk kernel of each WalkKind and its dynamic shared memory.  The lane-parallel walk is the default for WALK_LANES;
// JSMPEG_B200_WALK=serial selects the one-chain-per-warp walk instead.
struct WalkKernel {
	void (*fn)(const ParseTask *, int, const uint4 *);
	size_t smem;
};
const WalkKernel *walk_kernels() {
	static const bool serial = [] {
		const char *e = getenv("JSMPEG_B200_WALK");
		return e && !strcmp(e, "serial");
	}();
	static const WalkKernel table[N_WALK_KINDS] = {
	    serial ? WalkKernel{walk_pictures_kernel, WALK_SMEM_SERIAL} : WalkKernel{walk_pictures_lanes_kernel, WALK_SMEM_LANES},
	    {walk_pictures_slices_kernel, WALK_SMEM_LANES},
	    {walk_pictures_b_kernel, WALK_SMEM_SERIAL},
	};
	return table;
}

}  // namespace

// The multi-symbol walk table (walk.cuh: build_ms_table), built once per device from the generated DCT table.
static const uint16_t *ms_table_for_current_device() {
	static uint16_t *tables[64] = {};
	static std::mutex lock;  // decoders may be driven from several host threads
	std::lock_guard<std::mutex> guard(lock);
	int dev = 0;
	CUDA_CHECK(cudaGetDevice(&dev));
	if (tables[dev]) return tables[dev];
	for (int k = 0; k < N_WALK_KINDS; k++)  // per device, once
		CUDA_CHECK(cudaFuncSetAttribute(walk_kernels()[k].fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)walk_kernels()[k].smem));
	std::vector<uint16_t> dct((VLC_DCT_MAX_Z + 1) * 32);
	CUDA_CHECK(cudaMemcpyFromSymbol(dct.data(), VLC_DCT_COEFF, dct.size() * sizeof(uint16_t)));
	std::vector<uint16_t> ms(MS_TABLE_ENTRIES);
	build_ms_table(dct.data(), ms.data());
	uint16_t *d = nullptr;
	CUDA_CHECK(cudaMalloc(&d, ms.size() * sizeof(uint16_t)));
	CUDA_CHECK(cudaMemcpy(d, ms.data(), ms.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
	tables[dev] = d;
	return d;
}

int launch_parse_pictures(WalkKind kind, const ParseTask *tasks, int n_tasks, int max_mb_size, bool expand,
                          cudaStream_t stream, const ParseFork *fork, cudaStream_t after_walks) {
	if (n_tasks <= 0) return 0;
	const uint4 *ms = reinterpret_cast<const uint4 *>(ms_table_for_current_device());
	const WalkKernel walk = walk_kernels()[kind];
	const int per_cta = WALK_THREADS / 32;
	// The wave arrives sorted by picture size, largest first.  A lane-parallel wave of at least 64 pictures per group
	// is cut into PARSE_GROUPS equal groups: group 0 (largest pictures) stays on `stream`, the others go to side
	// streams, each walk followed by its own expand, so that the expand of the smaller pictures runs while the walk of
	// the bigger ones is still going.  On an H100 this takes 3 ms off stage 1 of a 3840-picture 1080p wave (DESIGN 8).
	// A walk-only wave has no expand to overlap: one group.  The slice and B walks take one group: B pictures are the
	// small ones of a stream.
	const int groups = (kind == WALK_LANES && expand && fork && n_tasks >= 64 * PARSE_GROUPS) ? PARSE_GROUPS : 1;
	if (groups > 1) CUDA_CHECK(cudaEventRecord(fork->fork, stream));
	for (int g = 0; g < groups; g++) {
		const int lo = (int)((long)n_tasks * g / groups), hi = (int)((long)n_tasks * (g + 1) / groups);
		const int n = hi - lo;
		cudaStream_t st = g == 0 ? stream : fork->side[g];
		if (g > 0) CUDA_CHECK(cudaStreamWaitEvent(st, fork->fork, 0));
		walk.fn<<<(n + per_cta - 1) / per_cta, WALK_THREADS, walk.smem, st>>>(tasks + lo, n, ms);
		if (after_walks) {
			CUDA_CHECK(cudaEventRecord(fork->walked[g], st));
			CUDA_CHECK(cudaStreamWaitEvent(after_walks, fork->walked[g], 0));
		}
		if (expand) launch_expand(tasks + lo, n, max_mb_size, st);
		if (g > 0) {
			CUDA_CHECK(cudaEventRecord(fork->join[g], st));
			CUDA_CHECK(cudaStreamWaitEvent(stream, fork->join[g], 0));
		}
	}
	return (expand ? 2 : 1) * groups;
}
