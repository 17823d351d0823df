// macroblocks.cu -- export of the walks' macroblock records into the public layout (sm_90a), for
// jsmpeg_b200_batch_decode_macroblocks (engine.cu, DESIGN 3.8).
//
// One thread per macroblock of every request of a wave, over a flattened index: request i owns the
// range [first_i, first_i + mb_size_i), so pictures of mixed sizes share the grid evenly.  A thread
// finds its request by binary search over `first` (the task table is small and stays in L1/L2), then
// moves one 16-byte record to one 16-byte entry through export_macroblock (macroblocks.cuh).
#include <string.h>

#include "common.cuh"
#include "macroblocks.cuh"

namespace {

constexpr int EXPORT_THREADS = 256;

__global__ void __launch_bounds__(EXPORT_THREADS)
export_macroblocks_kernel(const MbExportTask *__restrict__ tasks, int n_tasks, uint32_t total_mb) {
	const uint32_t i = blockIdx.x * EXPORT_THREADS + threadIdx.x;
	if (i >= total_mb) return;
	int lo = 0, hi = n_tasks - 1;  // the last request with first <= i
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (__ldg(&tasks[mid].first) <= i) lo = mid;
		else hi = mid - 1;
	}
	const MbExportTask t = tasks[lo];
	const uint32_t mb = i - t.first;
	const uint4 raw = __ldg(reinterpret_cast<const uint4 *>(t.src) + mb);
	mb_record_t r;
	memcpy(&r, &raw, sizeof r);
	const jsmpeg_b200_macroblock_t m = export_macroblock(r, t.picture_type);
	uint4 out;
	memcpy(&out, &m, sizeof out);
	reinterpret_cast<uint4 *>(t.dst)[mb] = out;
}

}  // namespace

void launch_export_macroblocks(const MbExportTask *tasks, int n_tasks, uint32_t total_mb, cudaStream_t stream) {
	if (n_tasks <= 0 || total_mb == 0) return;
	export_macroblocks_kernel<<<(total_mb + EXPORT_THREADS - 1) / EXPORT_THREADS, EXPORT_THREADS, 0, stream>>>(tasks, n_tasks, total_mb);
	CUDA_CHECK(cudaGetLastError());
}
