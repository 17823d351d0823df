// conceal.cu -- the copy of the opt-in `conceal` option (sm_90a, DESIGN 3.19): every macroblock a damaged picture
// lacks gets the co-located samples of its forward plane set, before the picture's reconstruct step.
//
// One warp per macroblock of every request of a step, over a flattened index as in macroblocks.cu: request i owns the
// range [first_i, first_i + mb_size_i).  A warp finds its request by binary search over `first`, reads the
// macroblock's flags and, when MBF_PRESENT is clear, copies its rows (conceal_macroblock, conceal.cuh).
#include "common.cuh"
#include "conceal.cuh"

namespace {

constexpr int CONCEAL_THREADS = 256;
constexpr int CONCEAL_WARPS = CONCEAL_THREADS / 32;

__global__ void __launch_bounds__(CONCEAL_THREADS)
conceal_kernel(const ConcealTask *__restrict__ tasks, int n_tasks, uint32_t total_mb) {
	const uint32_t i = blockIdx.x * CONCEAL_WARPS + (threadIdx.x >> 5);
	if (i >= total_mb) return;
	int lo = 0, hi = n_tasks - 1;  // the last request with first <= i
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (__ldg(&tasks[mid].first) <= i) lo = mid;
		else hi = mid - 1;
	}
	const ConcealTask t = tasks[lo];
	conceal_macroblock(t, (int)(i - t.first), threadIdx.x & 31);
}

}  // namespace

void launch_conceal(const ConcealTask *tasks, int n_tasks, uint32_t total_mb, cudaStream_t stream) {
	if (n_tasks <= 0 || total_mb == 0) return;
	conceal_kernel<<<(total_mb + CONCEAL_WARPS - 1) / CONCEAL_WARPS, CONCEAL_THREADS, 0, stream>>>(tasks, n_tasks, total_mb);
	CUDA_CHECK(cudaGetLastError());
}
