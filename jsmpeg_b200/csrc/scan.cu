// scan.cu -- stage 0: byte-parallel search for start-code prefixes (00 00 01) in an elementary
// stream resident in HBM.
//
// The reference finds the next picture with a serial byte scan on every decode()
// (src/buffer.js:115-139 findNextStartCode / findStartCode), and ends a slice where the next bytes
// are a start code (buffer.js:141-150).  Here the scan runs once per written span: each thread tests
// 16 byte positions (one 16-byte load plus a look-ahead word) and appends hits to the stream's
// position list; the host sorts the (short) list, picks the picture start codes (fourth byte 00) out
// of it and hands the whole list back to the device: knowing every picture start up front is what
// lets stage 1 parse all buffered pictures concurrently, and knowing every prefix is what tells the
// lane-parallel walk where a slice ends without reading the slice (instead of a 128-bytes-per-step
// search over every picture's bytes once more).
#include "common.cuh"

namespace {

__global__ void scan_start_codes_kernel(const ScanSpan *__restrict__ spans, uint32_t *__restrict__ positions, uint32_t capacity,
                                        uint32_t *__restrict__ counts) {
	// blockIdx.y = the span; `es` is 16-byte aligned; a thread handles byte positions [base, base + 16)
	const ScanSpan sp = spans[blockIdx.y];
	const uint8_t *__restrict__ es = sp.es;
	const uint32_t from = sp.from, len = sp.len;
	const uint32_t first = from & ~15u;
	const uint32_t base = first + (blockIdx.x * blockDim.x + threadIdx.x) * 16u;
	if (base >= len) return;
	const uint4 v = __ldg(reinterpret_cast<const uint4 *>(es + base));
	uint32_t w[5] = {v.x, v.y, v.z, v.w, 0u};
	if (base + 16u < len) w[4] = __ldg(reinterpret_cast<const uint32_t *>(es + base + 16u));
#pragma unroll
	for (int i = 0; i < 16; i++) {
		// four bytes starting at position base + i, byte 0 in the low bits
		const uint32_t q = __funnelshift_r(w[i >> 2], w[(i >> 2) + 1], (i & 3) * 8);
		const uint32_t pos = base + i;
		// 00 00 01 -> low three bytes 0x010000; all three bytes must be inside the buffer (the fourth, the code,
		// is looked at by the host once it is there)
		if ((q & 0x00ffffffu) == 0x00010000u && pos >= from && pos + 2u < len) {
			const uint32_t slot = atomicAdd(counts + blockIdx.y, 1u);
			if (slot < capacity) positions[(size_t)blockIdx.y * capacity + slot] = pos;
		}
	}
}

}  // namespace

// longest_span = the largest len - (from & ~15) of the spans: the grid covers it, shorter spans' surplus threads leave at once
void launch_scan_start_codes(const ScanSpan *spans, int n_spans, uint32_t longest_span, uint32_t *positions,
                             uint32_t capacity, uint32_t *counts, cudaStream_t stream) {
	if (n_spans <= 0 || longest_span == 0) return;
	const uint32_t n_threads = (longest_span + 15u) / 16u;
	const int block = 256;
	const dim3 grid((n_threads + block - 1) / block, (unsigned)n_spans);
	scan_start_codes_kernel<<<grid, block, 0, stream>>>(spans, positions, capacity, counts);
}
