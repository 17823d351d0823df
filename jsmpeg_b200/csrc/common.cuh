// common.cuh -- task descriptors shared by the kernels and the host engine (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <stdexcept>
#include <string>

#include "coef_records.h"
#include "records.h"

// A failed CUDA call never takes the host process down (the reference "never fails": a decoder that
// cannot work answers decode() == false).  CUDA_CHECK throws; every C-ABI entry point catches, marks
// its decoder dead (jsmpeg_b200_batch_last_error) and returns its failure value (engine.cu).
struct CudaFailure : std::runtime_error {
	cudaError_t code;
	CudaFailure(cudaError_t c, const std::string &what) : std::runtime_error(what), code(c) {}
};
[[noreturn]] inline void throw_cuda_failure(cudaError_t e, const char *file, int line) {
	char msg[512];
	snprintf(msg, sizeof msg, "jsmpeg_b200: CUDA error %s at %s:%d: %s", cudaGetErrorName(e), file, line, cudaGetErrorString(e));
	throw CudaFailure(e, msg);
}
#define CUDA_CHECK(expr)                                                  \
	do {                                                                  \
		cudaError_t _e = (expr);                                          \
		if (_e != cudaSuccess) throw_cuda_failure(_e, __FILE__, __LINE__); \
	} while (0)

// Per-stream sequence parameters as the kernels need them (reference mpeg1.js:78-153).
struct SeqParams {
	int32_t mb_width, mb_height, mb_size;
	int32_t coded_width, coded_height;
	uint8_t intra_q[64];     // de-zigzagged (mpeg1.js:100-116)
	uint8_t non_intra_q[64];
	// the same two matrices in COEFFICIENT (zig-zag) order, as stage 1b wants them: entry n of table k
	// (0 intra, 1 non-intra) = (raster index of coefficient n) * 2 | Q[raster index] << 8 (seq_fill_xq)
	uint16_t xq[2][64];
};

// host helper: derive SeqParams::xq from the de-zigzagged matrices (ZIG_ZAG, mpeg1.js:996-1005)
inline void seq_fill_xq(SeqParams &sp) {
	static const uint8_t zz[64] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48,
	                               41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22,
	                               15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
	for (int n = 0; n < 64; n++) {
		sp.xq[0][n] = (uint16_t)(zz[n] * 2 | sp.intra_q[zz[n]] << 8);
		sp.xq[1][n] = (uint16_t)(zz[n] * 2 | sp.non_intra_q[zz[n]] << 8);
	}
}

// Stage 1: one warp parses one picture.
struct ParseTask {
	const uint8_t *es;     // 16-byte aligned base of the stream's ES mirror in HBM, >= 64 readable bytes past es_len
	uint32_t es_len;       // valid bytes (bytes past it read as zero, like a JS typed array)
	uint32_t start_byte;   // first byte after the 00 00 01 00 picture start code
	const SeqParams *seq;  // device pointer
	mb_record_t *hdr;      // [mb_size]
	int16_t *coef;         // [mb_size][6][64]
	picture_info_t *info;  // out
	uint2 *park;           // [mb_size][6]: per coded block {bit offset of its first coefficient code, intra dc},
	                       // the walk's hand-over to stage 1b (a dense side array, written and read as a stream)
	int32_t mb_width, mb_size;  // copies of the sequence parameters (no dependent load in front of the walk)
	// lane-parallel walk: staging area for relative macroblock records (walk.cuh, WALK_STAGE): stage_entries
	// entries of 64 bytes, shared out among the lanes; nullptr = no staging (the walk then makes a second,
	// storing pass over the bits).  Once the picture's walk has finished the area is dead, and stage 1b reuses it
	// as the picture's compact coefficient plane (compact_plane); nullptr = stage 1b writes dense records only.
	uint4 *stage;
	int32_t stage_entries;
	// the stream's start-code prefixes (byte positions of 00 00 01, sorted, all of them up to es_len) and the
	// index of this picture's own start code in that list: a slice ends at the first prefix at or after its
	// first macroblock, so the walk looks the position up instead of searching the bytes.  nullptr = search.
	const uint32_t *codes;
	uint32_t n_codes, code_hint;
};

// staging entries per picture: three per macroblock (a lane keeps its macroblocks in its own stretch and a
// sub-sequence of small macroblocks holds more than the average; a lane that runs out falls back to the
// second pass) + one per lane for rounding
constexpr int stage_entries_for(int mb_size) { return 3 * mb_size + 64; }

// The compact coefficient plane of a picture (coef_records.h): one 32-byte record per block slot mb * 6 + b, in the
// picture's staging area.  6 * 32 * mb_size bytes fit the stage_entries_for(mb_size) * 64 = 192 * mb_size + 4096
// bytes of the area; the walk is done with it before stage 1b of the same picture runs (same stream), and a slot is
// walked again only after the reconstruction of its last picture (ev_round, engine.cu), the rule that already
// guards the dense coefficient plane.
static_assert(6 * sizeof(coef_record_t) <= 3 * 64, "the compact plane fits the staging area");
__host__ __device__ inline coef_record_t *compact_plane(uint4 *stage) { return reinterpret_cast<coef_record_t *>(stage); }

struct PlaneSet {
	uint8_t *y, *cr, *cb;
};

// PREDICTION_INSIDE: whether every tap an 8x8 block's prediction USES lies inside its plane of plane_size samples: the block's first tap
// at flat index src (origin + (mv >> 1) * stride + (mh >> 1), mpeg1.js:479, 567), oh / ov its horizontal / vertical
// half-sample flags.  A flat-index rule: a vector past a row's end wraps into the next row.  Stage 2 predicts 0 for a
// block outside (recon.cuh), and the accumulated map ends its trace there (accumulate.cuh).  A macro: stage 2's machine
// code is the same as with the expression written out (an inline function reorders it).
#define PREDICTION_INSIDE(src, stride, plane_size, oh, ov) \
	((src) >= 0 && (src) + 7 * (stride) + 7 + ((ov) ? (stride) : 0) + ((oh) ? 1 : 0) < (plane_size))

// Stage 2: one task per (stream, picture); blockIdx.y selects the task.
struct ReconTask {
	const mb_record_t *hdr;
	const int16_t *coef;            // dense records: the blocks the compact plane marks COEF_RECORD_DENSE
	const coef_record_t *compact;   // compact records (coef_records.h), or nullptr: every coded block is dense
	PlaneSet cur;   // written
	PlaneSet fwd;   // read (previous I/P picture; B picture: the older of the two most recent I/P pictures)
	int32_t mb_width, mb_size;
	int32_t coded_width, coded_height;
	uint8_t *rgba;  // optional fused epilogue target (display size, RGBA8888) or nullptr
	int32_t width, height;
	PlaneSet bwd;   // B picture (the opt-in extension): the newer of the two most recent I/P pictures
	int16_t *res;   // OUT_RESIDUALS: the picture's residual, coded_size * 3 / 2 int16 in the planes' layout, or nullptr
	uint8_t *frame; // decode_frames: a second copy of the picture's planes (coded_size * 3 / 2 bytes), or nullptr
};

// kernel launchers (defined in scan.cu / parse.cu / recon.cu)
// Stage 0, all streams of a batch in one launch: span k = bytes [from, len) of the ES mirror `es`; its hits
// (byte positions of 00 00 01, unsorted) go to positions[k * capacity ...], their number to counts[k] (it keeps
// counting past `capacity`: the host sees an overflow and repeats the scan with room).
struct ScanSpan {
	const uint8_t *es;
	uint32_t from, len;
};
void launch_scan_start_codes(const ScanSpan *spans, int n_spans, uint32_t longest_span, uint32_t *positions,
                             uint32_t capacity, uint32_t *counts, cudaStream_t stream);
// Helper streams/events with which stage 1 forks a (size-sorted) wave of I/P pictures into groups: the expand of
// a group of small pictures runs while the walk of the bigger pictures is still going.
constexpr int PARSE_GROUPS = 8;
struct ParseFork {
	cudaStream_t side[PARSE_GROUPS];
	cudaEvent_t fork, join[PARSE_GROUPS];
	cudaEvent_t walked[PARSE_GROUPS];  // behind each group's walk, before its expand (launch_parse_pictures: after_walks)
};
// The walk kernels of stage 1a, in the order a wave launches them:
//   WALK_LANES   I/P pictures: the lane-parallel walk (walk.cuh), or with JSMPEG_B200_WALK=serial the serial walk
//   WALK_SLICES  I/P pictures of many slices (opt-in "slice_walk", walk_slices.cuh): a lane per slice
//   WALK_B       B pictures (opt-in "decode_b", walk_b.cuh): the serial walk with the B-picture macroblock layer
enum WalkKind { WALK_LANES, WALK_SLICES, WALK_B, N_WALK_KINDS };
// the host routes an I/P picture to the slice walk when it has at least this many slices
constexpr int SLICE_WALK_MIN_SLICES = 4;
// Stage 1 of n_tasks pictures of walk kernel `kind`: the walk + the expand, or with expand = false the walk alone
// (macroblock records without coefficients).  A WALK_LANES wave with expand and `fork` is cut into size groups, a walk
// + an expand launch per group; every other call is one group.  after_walks, unless nullptr (it needs `fork`), is a stream
// that is made to wait for every group's walk and for none of the expands: what is queued on it next finds the walks'
// output, the picture infos among it, while stage 1b is still running.  Returns the number of kernels launched.
int launch_parse_pictures(WalkKind kind, const ParseTask *tasks, int n_tasks, int max_mb_size, bool expand,
                          cudaStream_t stream, const ParseFork *fork = nullptr, cudaStream_t after_walks = nullptr);
// Stage 2 of n_tasks pictures, by kernel: I/P pictures, then I/P pictures with the planar -> RGBA conversion fused in
// (tasks with `rgba`), then B pictures (tasks with `bwd`: prediction from two references), then B pictures with the
// conversion; each kernel's tasks in their order.  `tasks_host` is read on the host at launch time: the table travels
// in the kernel parameters.  When any task of a kernel has `res`, all that kernel's tasks go to its RES variant, which
// also stores the residual of every task with `res` (the others ride along with none); when any has `frame`, they go to
// its FRAME variant instead, which stores both the residual and the planar frame of every task that has one.  Returns
// the number of kernels launched.
int launch_reconstruct(const ReconTask *tasks_host, int n_tasks, cudaStream_t stream);

// Macroblock export (macroblocks.cu): request i converts the records of one picture (`mb_size` of them at `src`, a
// picture of picture_coding_type `picture_type`) into the public jsmpeg_b200_macroblock_t layout at `dst`; `first` is
// the number of macroblocks of requests 0 .. i-1.  One thread per macroblock of all requests, one launch.
struct MbExportTask {
	const mb_record_t *src;
	void *dst;
	uint32_t first;
	int32_t mb_size;
	int32_t picture_type;
	int32_t pad;
};
void launch_export_macroblocks(const MbExportTask *tasks, int n_tasks, uint32_t total_mb, cudaStream_t stream);

// Coefficient export (coefficients.cu): request i writes the dequantised coefficients of one picture (`mb_size`
// macroblocks; records at `hdr`, stage 1b's compact plane at `compact` and dense records at `coef`, as stage 2 reads
// them) to `dst` in the public layout of jsmpeg_b200_batch_decode_coefficients: per macroblock 6 blocks of 64 int16 in
// raster order, 0 for uncoded blocks and absent macroblocks.  `first` is the number of macroblocks of requests
// 0 .. i-1.  One thread per 16-byte output row (48 per macroblock) of all requests, one launch.
struct CoefExportTask {
	const mb_record_t *hdr;
	const int16_t *coef;
	const coef_record_t *compact;
	void *dst;
	uint32_t first;
	int32_t mb_size;
};
void launch_export_coefficients(const CoefExportTask *tasks, int n_tasks, uint32_t total_mb, cudaStream_t stream);

// Residual export (residuals.cu): request i writes the inverse transform of every block of one picture (`mb_width` x
// `mb_height` macroblocks; records as CoefExportTask's) to `dst` in the public layout of
// jsmpeg_b200_batch_decode_residuals: int16 planes Y | Cr | Cb of the coded size, 0 for uncoded blocks and absent
// macroblocks.  One thread per block, a warp per 32 blocks of one request (6 * mb_size block slots rounded up to
// whole warps); `first` is the number of warps of requests 0 .. i-1.  One launch for all requests.
// (A type of its own: CoefExportTask, and so export_coefficients_kernel, stay as they are.)
struct ResExportTask {
	const mb_record_t *hdr;
	const int16_t *coef;
	const coef_record_t *compact;
	int16_t *dst;
	uint32_t first;
	int32_t mb_width, mb_height;
	int32_t pad;
};
// the warps of a request of mb_size macroblocks
constexpr uint32_t res_export_warps(int mb_size) { return ((uint32_t)mb_size * 6 + 31) / 32; }
void launch_export_residuals(const ResExportTask *tasks, int n_tasks, uint32_t total_warps, cudaStream_t stream);

// Accumulated map (accumulate.cu, DESIGN 3.11): task i writes the map of one reference picture of a chain (records as
// ResExportTask's) to `dst` from `prev`, the map of the chain's previous reference picture (nullptr: the chain's first
// picture, which traces nothing back).  A map is one 8-byte record {dx, dy, residual, back} (int16 each, the public
// jsmpeg_b200_accumulated_t) per sample of the planes Y | Cr | Cb.  The geometry of ResExportTask: a thread per block,
// `first` warps before task i; one launch per chain depth.
struct AccTask {
	const mb_record_t *hdr;
	const int16_t *coef;
	const coef_record_t *compact;
	const uint2 *prev;
	uint2 *dst;
	uint32_t first;
	int32_t mb_width, mb_height;
};
void launch_accumulate(const AccTask *tasks, int n_tasks, uint32_t total_warps, cudaStream_t stream);
