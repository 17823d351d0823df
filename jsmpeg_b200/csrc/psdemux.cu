// psdemux.cu -- MPEG program stream demultiplexing on the device, many streams in one pass (ISO 11172-1
// system streams, .mpg; ISO 13818-1 program streams, .vob).  The item, link and place rules are in
// psdemux.cuh; the Python model is tools/mini_ps.py; DESIGN section 3.5 has the why.
//
// A call demultiplexes many requests (psdemux.cuh: a stream's left-over bytes and new bytes, each at its own
// 16-byte aligned offset of one staging buffer).  Where the items ARE is a chain of variable lengths: item k + 1
// starts where item k ends.  Walking it is ~6,000 dependent steps for a 12 MB clip of 2 KB packets, so it is
// resolved in parallel over CANDIDATES instead:
//   candidates  one thread per 16 staged bytes keeps every 00 00 01 that lies inside one request and has a code
//               >= B9 and counts it for its request; one sort of the call-wide positions groups them by request
//   link        per candidate: its SUCCESSOR, the candidate at pos + len of its request (binary search) -- or,
//               after a break (no item where one should start), the request's next valid pack header (a
//               suffix minimum over the candidates) -- or a terminal: END (exactly at the request's end),
//               INCOMPLETE (needs bytes of the stream's next write), NOHEAD (no pack header left); a terminal
//               points to itself.  Successors lie strictly later in the same request.
//   chain       pointer doubling J(k+1)(x) = Jk(Jk(x)) up to the largest request's candidate count; one head per
//               request; marking from all heads top down: S = {heads}, for k = K .. 0 add Jk(x) for every x in
//               S.  What ends up marked is exactly what the heads reach; J_K(head) is the request's terminal.
//   place       one thread per marked candidate: PES packet of the request's stream -> payload span, PTS; one
//               exclusive scan of (payload length << 32 | PES table entry) over all candidates gives every payload
//               its ES offset within its request and every entry its index in (request, offset) order; after the
//               host has made room in the streams, one CTA per packet copies its payload to its stream.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "demux.h"
#include "psdemux.cuh"

namespace {

constexpr uint32_t NONE = PS_NONE;

struct MinOp {
	__device__ uint32_t operator()(uint32_t a, uint32_t b) const { return a < b ? a : b; }
};

// the request owning staging byte g: the last one whose base is <= g; NONE if g lies in the padding behind it
__device__ __forceinline__ uint32_t request_at(const PsReq *__restrict__ req, uint32_t n_req, uint32_t g) {
	uint32_t lo = 0, hi = n_req;
	while (lo < hi) {
		const uint32_t mid = (lo + hi) >> 1;
		if (req[mid].base <= g) lo = mid + 1; else hi = mid;
	}
	return lo > 0 && g - req[lo - 1].base < req[lo - 1].n ? lo - 1 : NONE;
}

__device__ __forceinline__ PsCands cands_of(const PsReq &rq, const PsReqOut &o, const uint32_t *pos, const uint32_t *npr, uint32_t m) {
	return PsCands{pos, npr, m, o.c0, o.c0 + o.count, rq.base};
}

// candidates: a thread tests 16 staged byte positions (one 16-byte load plus a look-ahead word, as scan.cu does);
// ctl[0] = candidates, ctl[1] = the largest request's count
__global__ void ps_candidates_kernel(const uint8_t *__restrict__ stage, uint32_t staged, const PsReq *__restrict__ req, uint32_t n_req,
                                     PsReqOut *__restrict__ out, uint32_t *__restrict__ sel, uint32_t *__restrict__ ctl) {
	const uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) * 16u;
	if (base >= staged) return;
	const uint4 v = __ldg(reinterpret_cast<const uint4 *>(stage + base));
	uint32_t w[5] = {v.x, v.y, v.z, v.w, 0u};
	if (base + 16u < staged) w[4] = __ldg(reinterpret_cast<const uint32_t *>(stage + base + 16u));
#pragma unroll
	for (int i = 0; i < 16; i++) {
		const uint32_t q = __funnelshift_r(w[i >> 2], w[(i >> 2) + 1], (i & 3) * 8);
		if ((q & 0x00ffffffu) != 0x00010000u) continue;
		const uint32_t g = base + i, r = request_at(req, n_req, g);
		if (r == NONE || !ps_keep(stage + req[r].base, req[r].n, g - req[r].base)) continue;
		sel[atomicAdd(ctl, 1u)] = g;
		atomicMax(ctl + 1, atomicAdd(&out[r].count, 1u) + 1u);
	}
}

// per candidate: rev[m - 1 - i] = i if a valid pack header starts there; per request: its first candidate
__global__ void ps_pack_kernel(const uint8_t *__restrict__ stage, const PsReq *__restrict__ req, uint32_t n_req, const uint32_t *__restrict__ pos,
                               uint32_t m, PsReqOut *__restrict__ out, uint32_t *__restrict__ rev) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < m) {
		const uint32_t r = request_at(req, n_req, pos[i]);
		rev[m - 1 - i] = ps_is_pack(stage + req[r].base, req[r].n, pos[i] - req[r].base) ? i : NONE;
	}
	if (i < n_req) out[i].c0 = ps_lower(pos, 0, m, req[i].base);
}

// per candidate: successor (J0) and terminal record
__global__ void ps_link_kernel(const uint8_t *__restrict__ stage, const PsReq *__restrict__ req, uint32_t n_req, const PsReqOut *__restrict__ out,
                               const uint32_t *__restrict__ pos, const uint32_t *__restrict__ npr, uint32_t m, uint32_t *__restrict__ j0,
                               uint2 *__restrict__ term) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= m) return;
	const uint32_t r = request_at(req, n_req, pos[i]);
	const PsStep s = ps_link(stage + req[r].base, req[r].n, cands_of(req[r], out[r], pos, npr, m), i);
	j0[i] = s.kind == PS_T_LINK ? s.next : i;
	term[i] = make_uint2(s.kind, s.stop);
}

__global__ void ps_double_kernel(const uint32_t *__restrict__ jk, uint32_t *__restrict__ jk1, uint32_t m) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < m) jk1[i] = jk[jk[i]];
}

// one thread per request: the head of its chain (marked), or its terminal if it has none
__global__ void ps_head_kernel(const uint8_t *__restrict__ stage, const PsReq *__restrict__ req, uint32_t n_req, PsReqOut *__restrict__ out,
                               const uint32_t *__restrict__ pos, const uint32_t *__restrict__ npr, uint32_t m, uint8_t *__restrict__ marked) {
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= n_req) return;
	const PsStep s = ps_head(stage + req[r].base, req[r].n, cands_of(req[r], out[r], pos, npr, m), req[r].in_sync != 0);
	if (s.kind == PS_T_LINK) {
		out[r].head = s.next;
		marked[s.next] = 1;
	} else {
		out[r].head = NONE;
		out[r].kind = s.kind;
		out[r].stop = s.stop;
	}
}

// one level of the top-down marking.  A node marked during this launch may or may not pass its mark on:
// either way only nodes a head reaches get marked, and every one of them is marked after level 0.
__global__ void ps_mark_kernel(const uint32_t *__restrict__ jk, uint32_t m, uint8_t *marked) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < m && marked[i]) marked[jk[i]] = 1;
}

// classify: place key, payload start (staging position) and PTS of every candidate; key[m] = 0 for the scan's total
__global__ void ps_classify_kernel(const uint8_t *__restrict__ stage, const PsReq *__restrict__ req, uint32_t n_req,
                                   const uint32_t *__restrict__ pos, uint32_t m, const uint8_t *__restrict__ marked,
                                   uint64_t *__restrict__ key, uint32_t *__restrict__ src, uint64_t *__restrict__ pts) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > m) return;
	uint64_t k = 0;
	if (i < m && marked[i]) {
		const uint32_t r = request_at(req, n_req, pos[i]);
		uint32_t start;
		uint64_t t;
		k = ps_place_key(stage + req[r].base, req[r].n, pos[i] - req[r].base, req[r].stream_id, &start, &t);
		src[i] = req[r].base + start;
		pts[i] = t;
	}
	key[i] = k;
}

// per request: its terminal, what it consumed, its ES bytes and PES table entries
__global__ void ps_totals_kernel(const PsReq *__restrict__ req, uint32_t n_req, const uint32_t *__restrict__ jtop, const uint2 *__restrict__ term,
                                 const uint64_t *__restrict__ scan, PsReqOut *__restrict__ out) {
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= n_req) return;
	PsReqOut o = out[r];
	if (o.head != NONE) {
		const uint2 t = term[jtop[o.head]];
		o.kind = t.x;
		o.stop = t.y;
	}
	ps_finish(o.kind, o.stop, req[r].n, &o.consumed, &o.in_sync);
	const uint64_t a = scan[o.c0], b = scan[o.c0 + o.count];
	o.total = (uint32_t)(b >> 32) - (uint32_t)(a >> 32);
	o.pes = (uint32_t)b - (uint32_t)a;
	o.pes_first = (uint32_t)a;
	out[r] = o;
}

// place: CTA i < m copies candidate i's payload to its stream and lists its PES table entry; CTAs m + r then zero
// the `pad` bytes behind request r's new ES bytes (the kernels read zeros there)
__global__ void ps_gather_kernel(const uint8_t *__restrict__ stage, const PsReq *__restrict__ req, uint32_t n_req, const PsReqOut *__restrict__ out,
                                 const uint32_t *__restrict__ pos, uint32_t m, const uint64_t *__restrict__ key, const uint32_t *__restrict__ src,
                                 const uint64_t *__restrict__ pts, const uint64_t *__restrict__ scan, uint32_t pad,
                                 uint32_t *__restrict__ pes_offset, uint64_t *__restrict__ pes_pts) {
	const uint32_t i = blockIdx.x;
	if (i >= m) {
		const uint32_t r = i - m;
		if (req[r].dst)
			for (uint32_t k = threadIdx.x; k < pad; k += blockDim.x) req[r].dst[out[r].total + k] = 0;
		return;
	}
	const uint64_t kk = key[i];
	const uint32_t len = (uint32_t)(kk >> 32);
	if (len == 0) return;
	const uint32_t r = request_at(req, n_req, pos[i]);
	if (!req[r].dst) return;
	const uint64_t at = scan[i];
	const uint32_t off = (uint32_t)(at >> 32) - (uint32_t)(scan[out[r].c0] >> 32);
	if (threadIdx.x == 0 && (kk & 1)) {
		pes_offset[(uint32_t)at] = req[r].es_base + off;
		pes_pts[(uint32_t)at] = pts[i];
	}
	const uint8_t *s = stage + src[i];
	uint8_t *d = req[r].dst + off;
	for (uint32_t k = threadIdx.x; k < len; k += blockDim.x) d[k] = s[k];
}

constexpr int BLOCK = 256;
int blocks(uint64_t threads) { return (int)std::max<uint64_t>((threads + BLOCK - 1) / BLOCK, 1); }

}  // namespace

struct PsScratch {
	DeviceBuffer<uint8_t> marked;
	DeviceBuffer<uint32_t> ctl, sel, pos;
	PinnedBuffer<uint32_t> h_ctl;
	DeviceBuffer<uint32_t> jump;  // (levels + 1) x cap
	DeviceBuffer<uint2> term;
	DeviceBuffer<uint32_t> rev, next_pack_rev, src;
	DeviceBuffer<uint64_t> key, scan, pts;
	size_t cap = 0;  // candidates the per-candidate arrays have room for
	int levels = 0;
	uint32_t n_req = 0, staged = 0, m = 0;
};

PsScratch *ps_scratch_create() { return new PsScratch(); }
void ps_scratch_destroy(PsScratch *s) { delete s; }

void ps_call_begin(PsScratch *s, uint32_t n_req, uint32_t staged) {
	s->n_req = n_req;
	s->staged = staged;
	s->m = 0;
	s->ctl.reserve(2);
	s->h_ctl.reserve(2);
	// candidates lie >= 4 bytes apart (the byte behind 00 00 01 is >= B9, so no prefix starts there) except one
	// cut by a request's end: room for every one the staged bytes can hold
	const size_t most = staged / 4 + n_req + 1;
	if (most > s->sel.size()) s->sel.reserve(most + most / 4);
}

uint32_t ps_call_candidates(PsScratch *s, PsIo &io, cudaStream_t st) {
	CUDA_CHECK(cudaMemsetAsync(io.out.data(), 0, s->n_req * sizeof(PsReqOut), st));
	CUDA_CHECK(cudaMemsetAsync(s->ctl.data(), 0, 2 * sizeof(uint32_t), st));
	ps_candidates_kernel<<<blocks((s->staged + 15) / 16), BLOCK, 0, st>>>(io.stage.data(), s->staged, io.req.data(), s->n_req, io.out.data(),
	                                                                      s->sel.data(), s->ctl.data());
	CUDA_CHECK(cudaMemcpyAsync(s->h_ctl.data(), s->ctl.data(), 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	return 1;
}

uint32_t ps_call_measure(PsScratch *s, PsIo &io, cudaStream_t st) {
	const uint32_t n = s->n_req, m = s->h_ctl[0], most = s->h_ctl[1];
	s->m = m;
	// doubling levels: 2^levels >= the largest request's candidate count bounds every chain
	int levels = 1;
	while ((1u << levels) < most) levels++;
	if (m > s->cap || levels > s->levels) {
		const size_t cap = std::max<size_t>(m + m / 4 + 64, s->cap);
		const int lv = std::max(levels + 1, s->levels);
		s->pos.reserve(cap);
		s->jump.reserve((size_t)(lv + 1) * cap);
		s->term.reserve(cap);
		s->rev.reserve(cap);
		s->next_pack_rev.reserve(cap);
		s->marked.reserve(cap);
		s->src.reserve(cap);
		s->pts.reserve(cap);
		s->key.reserve(cap + 1);
		s->scan.reserve(cap + 1);
		s->cap = cap;
		s->levels = lv;
	}
	io.reserve_pes(m);  // (a PES table entry per candidate at most)
	uint32_t launches = 0;
	const uint8_t *stage = io.stage.data();
	const PsReq *req = io.req.data();
	PsReqOut *out = io.out.data();
	const uint32_t *pos = s->pos.data(), *npr = s->next_pack_rev.data();
	size_t bytes = 0;
	if (m) {
		int bits = 1;
		while (bits < 32 && (1ull << bits) <= s->staged) bits++;
		cub::DeviceRadixSort::SortKeys(nullptr, bytes, s->sel.data(), s->pos.data(), (int)m, 0, bits, st);
		cub::DeviceRadixSort::SortKeys(io.temp_storage(bytes), bytes, s->sel.data(), s->pos.data(), (int)m, 0, bits, st);
		launches++;
	}
	ps_pack_kernel<<<blocks(std::max(m, n)), BLOCK, 0, st>>>(stage, req, n, pos, m, out, s->rev.data());
	launches++;
	if (m) {
		bytes = 0;
		cub::DeviceScan::InclusiveScan(nullptr, bytes, s->rev.data(), s->next_pack_rev.data(), MinOp(), (int)m, st);
		cub::DeviceScan::InclusiveScan(io.temp_storage(bytes), bytes, s->rev.data(), s->next_pack_rev.data(), MinOp(), (int)m, st);
		launches++;
	}
	uint32_t *jump = s->jump.data();
	ps_link_kernel<<<blocks(m), BLOCK, 0, st>>>(stage, req, n, out, pos, npr, m, jump, s->term.data());
	for (int k = 0; k < levels; k++) ps_double_kernel<<<blocks(m), BLOCK, 0, st>>>(jump + (size_t)k * s->cap, jump + (size_t)(k + 1) * s->cap, m);
	if (m) CUDA_CHECK(cudaMemsetAsync(s->marked.data(), 0, m, st));
	ps_head_kernel<<<blocks(n), BLOCK, 0, st>>>(stage, req, n, out, pos, npr, m, s->marked.data());
	for (int k = levels; k >= 0; k--) ps_mark_kernel<<<blocks(m), BLOCK, 0, st>>>(jump + (size_t)k * s->cap, m, s->marked.data());
	ps_classify_kernel<<<blocks((uint64_t)m + 1), BLOCK, 0, st>>>(stage, req, n, pos, m, s->marked.data(), s->key.data(), s->src.data(), s->pts.data());
	bytes = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, bytes, s->key.data(), s->scan.data(), (int)(m + 1), st);
	cub::DeviceScan::ExclusiveSum(io.temp_storage(bytes), bytes, s->key.data(), s->scan.data(), (int)(m + 1), st);
	ps_totals_kernel<<<blocks(n), BLOCK, 0, st>>>(req, n, jump + (size_t)levels * s->cap, s->term.data(), s->scan.data(), out);
	launches += 2 * levels + 6;  // link, doubling, head, marking, classify, scan, totals (a cub algorithm counts as one)
	CUDA_CHECK(cudaMemcpyAsync(io.h_out.data(), out, n * sizeof(PsReqOut), cudaMemcpyDeviceToHost, st));
	return launches;
}

uint32_t ps_call_gather(PsScratch *s, PsIo &io, uint32_t pad, cudaStream_t st) {
	const uint32_t n = s->n_req, m = s->m;
	ps_gather_kernel<<<m + n, 128, 0, st>>>(io.stage.data(), io.req.data(), n, io.out.data(), s->pos.data(), m, s->key.data(), s->src.data(),
	                                        s->pts.data(), s->scan.data(), pad, io.pes_offset.data(), io.pes_pts.data());
	return 1;
}
