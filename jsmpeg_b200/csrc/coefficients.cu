// coefficients.cu -- export of stage 1b's coefficient records into the public layout (sm_90a), for
// jsmpeg_b200_batch_decode_coefficients (engine.cu, DESIGN 3.9).
//
// One thread per 16-byte output row: 8 coefficients, one raster row of one block; 48 threads per macroblock, a CTA
// takes EXPORT_MBS consecutive macroblocks of the flattened index over all requests of a wave (request i owns
// [first_i, first_i + mb_size_i)).  A warp finds its requests by a 32-ary search over `first` (a warp covers at most two
// macroblocks), then a thread loads its macroblock record's flags / cbp word, and for a coded block its 32-byte compact
// record (one sector for the block's 8 threads) -- plus, for a block marked dense, its 16-byte row of the dense
// record.  Uncoded blocks and absent macroblocks load nothing more and store zeros.  Every row leaves as one 16-byte
// streaming store: nothing rereads it.
//
// Index width: the macroblock index is 32-bit (total_mb, the macroblocks of one wave, is far below 2^32 for any slot
// pool); the row number 48 * macroblock, which passes 2^32 for a few thousand 1080p slots, is never formed: the grid
// runs over macroblocks (EXPORT_MBS per CTA) and a thread's row within its macroblock is threadIdx.x % 48.
#include <string.h>

#include "common.cuh"

namespace {

constexpr int ROWS_PER_MB = 6 * 8;
constexpr int EXPORT_MBS = 8;  // macroblocks per CTA: 384 threads
constexpr int EXPORT_THREADS = EXPORT_MBS * ROWS_PER_MB;

__global__ void __launch_bounds__(EXPORT_THREADS)
export_coefficients_kernel(const CoefExportTask *__restrict__ tasks, int n_tasks, uint32_t total_mb) {
	const uint32_t g = blockIdx.x * EXPORT_MBS + threadIdx.x / ROWS_PER_MB;  // macroblock of the flattened index
	const uint32_t g0 = __shfl_sync(~0u, g, 0);                             // the warp's first: g is g0 or g0 + 1
	if (g0 >= total_mb) return;                                              // (the whole warp)
	const int r = threadIdx.x % ROWS_PER_MB;  // block * 8 + raster row
	const int block = r >> 3, row = r & 7;
	// The last request with first <= g0, by a 32-ary search of the warp: each round the lanes probe 32 evenly spaced
	// requests of the range and keep the stretch behind the last probe at or below g0 -- two rounds of dependent loads
	// for up to 1024 requests, where a binary search takes ten.
	const int lane = threadIdx.x & 31;
	int lo = 0, len = n_tasks;
	while (len > 1) {
		const int step = (len + 31) >> 5;
		const int at = lo + lane * step;
		const unsigned below = __ballot_sync(~0u, lane * step < len && __ldg(&tasks[at].first) <= g0);
		const int j = 31 - __clz(below);  // (lane 0's probe, first[lo] <= g0, always holds)
		lo += j * step;
		len = min(step, len - j * step);
	}
	// the warp's second macroblock may open the next request (every request has at least one macroblock)
	if (g != g0 && lo + 1 < n_tasks && __ldg(&tasks[lo + 1].first) <= g) lo++;
	if (g >= total_mb) return;
	const CoefExportTask t = tasks[lo];
	const uint32_t mb = g - t.first;
	// flags (byte 0) and cbp (byte 1) of the record's second word
	const uint32_t rec = __ldg(reinterpret_cast<const uint32_t *>(t.hdr + mb) + 1);
	uint4 out = make_uint4(0u, 0u, 0u, 0u);
	if ((rec & MBF_PRESENT) && ((rec >> 8) & (0x20u >> block))) {
		const uint4 *crec = reinterpret_cast<const uint4 *>(t.compact + (size_t)mb * 6 + block);
		const uint4 c0 = __ldg(crec), c1 = __ldg(crec + 1);
		coef_record_t cr;
		memcpy(&cr, &c0, 16);
		memcpy(reinterpret_cast<uint8_t *>(&cr) + 16, &c1, 16);
		if (cr.mask == COEF_RECORD_DENSE) {  // (rare) the dense record: its row as it is
			out = __ldg(reinterpret_cast<const uint4 *>(t.coef) + (size_t)mb * ROWS_PER_MB + r);
		} else {
			int16_t v[8];
			coef_record_row(cr, row, v);
			memcpy(&out, v, sizeof out);
		}
		if (row == 0 && (rec & MBF_INTRA)) {  // an intra DC leaves in its public form, sat16(8 * dc) (records.h)
			const int dc8 = max(-32768, min(32767, 8 * (int)(int16_t)(out.x & 0xffffu)));
			out.x = (out.x & 0xffff0000u) | ((uint32_t)dc8 & 0xffffu);
		}
	}
	__stcs(reinterpret_cast<uint4 *>(t.dst) + (size_t)mb * ROWS_PER_MB + r, out);
}

}  // namespace

void launch_export_coefficients(const CoefExportTask *tasks, int n_tasks, uint32_t total_mb, cudaStream_t stream) {
	if (n_tasks <= 0 || total_mb == 0) return;
	export_coefficients_kernel<<<(total_mb + EXPORT_MBS - 1) / EXPORT_MBS, EXPORT_THREADS, 0, stream>>>(tasks, n_tasks, total_mb);
	CUDA_CHECK(cudaGetLastError());
}
