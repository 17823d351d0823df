// psdemux.cu -- MPEG program stream demultiplexing on the device (ISO 11172-1 system streams, .mpg;
// ISO 13818-1 program streams, .vob).  The item rules are in psdemux.cuh; the Python model is
// tools/mini_ps.py; DESIGN section 3.5 has the why.
//
// Decomposition.  Where the items ARE is a chain of variable lengths: item k + 1 starts where item k
// ends.  Walking it is ~6,000 dependent steps for a 12 MB clip of 2 KB packets, so it is resolved in
// parallel over CANDIDATES instead:
//   candidates  every 00 00 01 of the buffer (scan.cu's kernel), those with a code >= B9 kept, sorted;
//               per candidate: its item length and its SUCCESSOR, the candidate at pos + len (binary
//               search) -- or a terminal: END (exactly at the buffer end), INCOMPLETE (needs bytes of the
//               next call), BREAK (no item where one should start); a terminal points to itself
//   chain       pointer doubling J(k+1)(x) = Jk(Jk(x)), then marking from the head top down: S = {head},
//               for k = K .. 0 add Jk(x) for every x in S.  What ends up marked is exactly what the head
//               reaches, after 2 (K + 1) launches.  A BREAK restarts from the next valid pack header
//               after it (a suffix minimum over the candidates), one round per break.
//   classify    one thread per marked candidate: PES packet of the selected stream -> payload span, PTS
//   place       exclusive scan of the payload lengths; one CTA copies one packet's payload to its place;
//               PES starts with a PTS are appended to a list for the host's PTS table.
#include <algorithm>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include "buffers.h"
#include "common.cuh"
#include "psdemux.cuh"

namespace {

constexpr uint32_t NONE = 0xffffffffu;
constexpr uint64_t NONE_PTS = ~0ull;  // (a PTS has 33 bits)
enum : uint32_t { T_LINK = 0, T_END = 1, T_INCOMPLETE = 2, T_BREAK = 3, T_NOHEAD = 4 };

struct KeepCode {  // start-code prefixes that can begin an item (video ES has none of these)
	const uint8_t *buf;
	uint32_t n;
	__device__ bool operator()(uint32_t p) const { return p + 3 >= n || buf[p + 3] >= 0xB9; }
};

struct MinOp {
	__device__ uint32_t operator()(uint32_t a, uint32_t b) const { return a < b ? a : b; }
};

// first index with pos[index] >= want (m if none)
__device__ uint32_t lower_bound(const uint32_t *__restrict__ pos, uint32_t m, uint32_t want) {
	uint32_t lo = 0, hi = m;
	while (lo < hi) {
		const uint32_t mid = (lo + hi) >> 1;
		if (pos[mid] < want) lo = mid + 1; else hi = mid;
	}
	return lo;
}

// What follows when the chain reaches byte t: the candidate there, or a terminal.
__device__ uint2 follow(const uint8_t *__restrict__ buf, uint32_t n, const uint32_t *__restrict__ pos, uint32_t m, uint32_t t) {
	if (t == n) return make_uint2(T_END, n);
	const uint32_t j = lower_bound(pos, m, t);
	if (j < m && pos[j] == t) return make_uint2(T_LINK, j);
	// no candidate: only the head of a start-code prefix cut by the buffer end can still become an item
	return make_uint2(ps_item_at(buf, n, t).kind == PS_NEED_MORE ? T_INCOMPLETE : T_BREAK, t);
}

// per candidate: successor (J0) and terminal record; rev[m - 1 - i] = i if a valid pack header starts there
__global__ void ps_link_kernel(const uint8_t *__restrict__ buf, uint32_t n, const uint32_t *__restrict__ pos, uint32_t m,
                               uint32_t *__restrict__ j0, uint2 *__restrict__ term, uint32_t *__restrict__ rev) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= m) return;
	const uint32_t p = pos[i];
	const PsItem it = ps_item_at(buf, n, p);
	uint2 r;
	if (it.kind == PS_NEED_MORE) r = make_uint2(T_INCOMPLETE, p);
	else if (it.kind == PS_BAD) r = make_uint2(T_BREAK, p);
	else r = follow(buf, n, pos, m, p + it.len);
	j0[i] = r.x == T_LINK ? r.y : i;
	term[i] = r;
	rev[m - 1 - i] = ps_is_pack(buf, n, p) ? i : NONE;
}

__global__ void ps_double_kernel(const uint32_t *__restrict__ jk, uint32_t *__restrict__ jk1, uint32_t m) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < m) jk1[i] = jk[jk[i]];
}

// Head of a round (one thread).  ctl: [0] head, [1] terminal type, [2] stop position.  from == NONE: the chain
// continues from the previous call at byte 0; otherwise it starts at the first valid pack header at or after `from`.
__global__ void ps_head_kernel(const uint8_t *__restrict__ buf, uint32_t n, const uint32_t *__restrict__ pos, uint32_t m,
                               const uint32_t *__restrict__ next_pack_rev, uint32_t from, uint32_t *__restrict__ ctl,
                               uint8_t *__restrict__ marked) {
	uint32_t head = NONE;
	if (from == NONE) {
		const uint2 r = follow(buf, n, pos, m, 0);
		if (r.x == T_LINK) head = r.y;
		else if (r.x == T_BREAK) from = 1;
		else { ctl[0] = NONE; ctl[1] = r.x; ctl[2] = r.y; return; }
	}
	if (head == NONE) {
		const uint32_t i = lower_bound(pos, m, from);
		if (i < m) head = next_pack_rev[m - 1 - i];
	}
	ctl[0] = head;
	ctl[1] = T_NOHEAD;
	ctl[2] = from;
	if (head != NONE) marked[head] = 1;
}

// one level of the top-down marking.  A node marked during this launch may or may not pass its mark on:
// either way only nodes the head reaches get marked, and every one of them is marked after level 0.
__global__ void ps_mark_kernel(const uint32_t *__restrict__ jk, uint32_t m, uint8_t *marked) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < m && marked[i]) marked[jk[i]] = 1;
}

__global__ void ps_end_kernel(const uint32_t *__restrict__ jtop, const uint2 *__restrict__ term, uint32_t *__restrict__ ctl) {
	const uint32_t head = ctl[0];
	if (head == NONE) return;
	const uint2 r = term[jtop[head]];
	ctl[1] = r.x;
	ctl[2] = r.y;
}

// classify: payload span of every marked PES packet of `stream_id`
__global__ void ps_classify_kernel(const uint8_t *__restrict__ buf, uint32_t n, const uint32_t *__restrict__ pos, uint32_t m,
                                   const uint8_t *__restrict__ marked, int stream_id, uint32_t *__restrict__ src,
                                   uint32_t *__restrict__ lens, uint64_t *__restrict__ pts) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= m) return;
	uint32_t len = 0, start = 0;
	uint64_t t = NONE_PTS;
	const uint32_t p = pos[i];
	if (marked[i] && p + 3 < n && buf[p + 3] == (uint32_t)stream_id) {
		const PsItem it = ps_item_at(buf, n, p);
		if (it.kind == PS_ITEM) {
			const PsPayload pl = ps_payload(buf + p, it.len);
			start = p + pl.start;
			len = pl.len;
			if (pl.has_pts && len) t = pl.pts;
		}
	}
	src[i] = start;
	lens[i] = len;
	pts[i] = t;
}

// place: one CTA per candidate copies its payload; a PES start with a PTS is appended to the list
__global__ void ps_gather_kernel(const uint8_t *__restrict__ buf, uint32_t m, const uint32_t *__restrict__ src,
                                 const uint32_t *__restrict__ lens, const uint32_t *__restrict__ offsets,
                                 const uint64_t *__restrict__ pts, uint8_t *__restrict__ es, uint32_t es_base,
                                 uint32_t *__restrict__ pes_count, uint32_t *__restrict__ pes_offset, uint64_t *__restrict__ pes_pts) {
	const uint32_t i = blockIdx.x;
	const uint32_t len = lens[i];
	if (len == 0) return;
	const uint32_t off = offsets[i];
	if (threadIdx.x == 0 && pts[i] != NONE_PTS) {
		const uint32_t k = atomicAdd(pes_count, 1u);
		pes_offset[k] = es_base + off;
		pes_pts[k] = pts[i];
	}
	const uint8_t *s = buf + src[i];
	uint8_t *d = es + es_base + off;
	for (uint32_t k = threadIdx.x; k < len; k += blockDim.x) d[k] = s[k];
}

}  // namespace

struct PsScratch {
	DeviceBuffer<uint8_t> buf, marked;
	DeviceBuffer<uint32_t> scan_pos, scan_count, sel, sel_count, pos;
	DeviceBuffer<ScanSpan> span;
	DeviceBuffer<uint32_t> jump;  // (levels + 1) x cap
	DeviceBuffer<uint2> term;
	DeviceBuffer<uint32_t> rev, next_pack_rev, ctl;
	DeviceBuffer<uint32_t> src, lens, offsets;
	DeviceBuffer<uint64_t> pts;
	DeviceBuffer<uint32_t> pes_count, pes_offset;
	DeviceBuffer<uint64_t> pes_pts;
	DeviceBuffer<uint8_t> temp;  // cub's temporary storage
	size_t cap = 0;  // candidates the per-candidate arrays have room for
	int levels = 0;
	uint32_t m = 0, launches = 0;
};

// room for `need` bytes of cub's temporary storage
static void *ps_temp(PsScratch &s, size_t need) {
	s.temp.reserve(need);
	return s.temp.data();
}

static void ps_reserve_scan(PsScratch &s, uint32_t n) {
	if (n <= s.scan_pos.size()) return;
	const uint32_t cap = n + n / 4 + 64;
	s.scan_pos.reserve(cap);
	s.sel.reserve(cap);
}

static void ps_reserve(PsScratch &s, size_t m) {
	int levels = 1;
	while ((size_t(1) << levels) < m) levels++;
	if (m <= s.cap && levels <= s.levels) return;
	const size_t cap = m + m / 4 + 64;
	while ((size_t(1) << levels) < cap) levels++;
	s.pos.reserve(cap);
	s.jump.reserve((size_t)(levels + 1) * cap);
	s.term.reserve(cap);
	s.rev.reserve(cap);
	s.next_pack_rev.reserve(cap);
	s.marked.reserve(cap);
	s.src.reserve(cap);
	s.lens.reserve(cap + 1);
	s.offsets.reserve(cap + 1);
	s.pts.reserve(cap);
	s.pes_offset.reserve(cap);
	s.pes_pts.reserve(cap);
	s.cap = cap;
	s.levels = levels;
}

PsScratch *ps_scratch_create() { return new PsScratch(); }
void ps_scratch_destroy(PsScratch *s) { delete s; }

// Phase 1: upload, candidates, chain, classify, scan.  *in_sync in/out: does the buffer continue the chain of
// the previous call at its first byte?  Returns the ES byte count; *consumed = the bytes of the buffer the
// demuxer is done with (the rest is the caller's leftover).
long ps_demux_measure(PsScratch *s, const uint8_t *host, size_t n_bytes, int stream_id, bool *in_sync, size_t *consumed, cudaStream_t st) {
	*consumed = 0;
	s->m = 0;
	s->launches = 0;
	if (n_bytes == 0) return 0;
	if (n_bytes > 0xfffff000ull) throw std::runtime_error("jsmpeg_b200: program stream buffer of 4 GiB or more");
	const uint32_t n = (uint32_t)n_bytes;
	// the scan reads 16-byte vectors and a look-ahead word
	if (n_bytes + 32 > s->buf.size()) s->buf.reserve(n_bytes + n_bytes / 4 + 32);
	s->span.reserve(1);
	s->scan_count.reserve(1);
	s->sel_count.reserve(1);
	s->ctl.reserve(3);
	s->pes_count.reserve(1);
	CUDA_CHECK(cudaMemcpyAsync(s->buf.data(), host, n_bytes, cudaMemcpyHostToDevice, st));
	CUDA_CHECK(cudaMemsetAsync(s->buf.data() + n_bytes, 0, 32, st));
	const ScanSpan span{s->buf.data(), 0, n};
	CUDA_CHECK(cudaMemcpyAsync(s->span.data(), &span, sizeof(span), cudaMemcpyHostToDevice, st));
	// candidates: every 00 00 01 (a scan that ran out of room counts on: rescan with room for all)
	ps_reserve_scan(*s, n / 256 + 1024);
	uint32_t hits = 0;
	for (;;) {
		CUDA_CHECK(cudaMemsetAsync(s->scan_count.data(), 0, sizeof(uint32_t), st));
		launch_scan_start_codes(s->span.data(), 1, n, s->scan_pos.data(), (uint32_t)s->scan_pos.size(), s->scan_count.data(), st);
		s->launches++;
		CUDA_CHECK(cudaMemcpyAsync(&hits, s->scan_count.data(), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
		CUDA_CHECK(cudaStreamSynchronize(st));
		if (hits <= s->scan_pos.size()) break;
		ps_reserve_scan(*s, hits);
	}
	ps_reserve(*s, hits);
	uint32_t m = 0;
	if (hits) {
		const KeepCode keep{s->buf.data(), n};
		size_t bytes = 0;
		cub::DeviceSelect::If(nullptr, bytes, s->scan_pos.data(), s->sel.data(), s->sel_count.data(), (int)hits, keep, st);
		cub::DeviceSelect::If(ps_temp(*s, bytes), bytes, s->scan_pos.data(), s->sel.data(), s->sel_count.data(), (int)hits, keep, st);
		CUDA_CHECK(cudaMemcpyAsync(&m, s->sel_count.data(), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
		CUDA_CHECK(cudaStreamSynchronize(st));
		s->launches++;
	}
	if (m) {
		int bits = 1;
		while (bits < 32 && (1ull << bits) <= n) bits++;
		size_t bytes = 0;
		cub::DeviceRadixSort::SortKeys(nullptr, bytes, s->sel.data(), s->pos.data(), (int)m, 0, bits, st);
		cub::DeviceRadixSort::SortKeys(ps_temp(*s, bytes), bytes, s->sel.data(), s->pos.data(), (int)m, 0, bits, st);
		s->launches++;
	}
	const int block = 256;
	const int grid = (int)((m + block - 1) / block);
	int levels = 1;
	while ((1u << levels) < m) levels++;
	uint32_t *jtop = s->jump.data() + (size_t)levels * s->cap;
	if (m) {
		ps_link_kernel<<<grid, block, 0, st>>>(s->buf.data(), n, s->pos.data(), m, s->jump.data(), s->term.data(), s->rev.data());
		size_t bytes = 0;
		cub::DeviceScan::InclusiveScan(nullptr, bytes, s->rev.data(), s->next_pack_rev.data(), MinOp(), (int)m, st);
		cub::DeviceScan::InclusiveScan(ps_temp(*s, bytes), bytes, s->rev.data(), s->next_pack_rev.data(), MinOp(), (int)m, st);
		for (int k = 0; k < levels; k++)
			ps_double_kernel<<<grid, block, 0, st>>>(s->jump.data() + (size_t)k * s->cap, s->jump.data() + (size_t)(k + 1) * s->cap, m);
		CUDA_CHECK(cudaMemsetAsync(s->marked.data(), 0, m, st));
		s->launches += 2 + levels;
	}
	// the chain, one round per break
	uint32_t from = *in_sync ? NONE : 0;
	uint32_t ctl[3] = {NONE, T_NOHEAD, 0};
	for (;;) {
		ps_head_kernel<<<1, 1, 0, st>>>(s->buf.data(), n, s->pos.data(), m, s->next_pack_rev.data(), from, s->ctl.data(), s->marked.data());
		if (m) {
			for (int k = levels; k >= 0; k--) ps_mark_kernel<<<grid, block, 0, st>>>(s->jump.data() + (size_t)k * s->cap, m, s->marked.data());
			ps_end_kernel<<<1, 1, 0, st>>>(jtop, s->term.data(), s->ctl.data());
			s->launches += levels + 2;
		}
		s->launches++;
		CUDA_CHECK(cudaMemcpyAsync(ctl, s->ctl.data(), sizeof(ctl), cudaMemcpyDeviceToHost, st));
		CUDA_CHECK(cudaStreamSynchronize(st));
		if (ctl[1] != T_BREAK) break;
		from = ctl[2] + 1;
	}
	switch (ctl[1]) {
		case T_END: *consumed = n; *in_sync = true; break;
		case T_INCOMPLETE: *consumed = ctl[2]; *in_sync = true; break;
		default:  // no valid pack header at or after ctl[2]: keep what could still begin one
			*consumed = std::max<size_t>(ctl[2], n >= 4 ? n - 4 : 0);
			*in_sync = false;
	}
	if (m == 0) return 0;
	ps_classify_kernel<<<grid, block, 0, st>>>(s->buf.data(), n, s->pos.data(), m, s->marked.data(), stream_id, s->src.data(), s->lens.data(), s->pts.data());
	CUDA_CHECK(cudaMemsetAsync(s->lens.data() + m, 0, sizeof(uint32_t), st));
	size_t bytes = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, bytes, s->lens.data(), s->offsets.data(), (int)(m + 1), st);
	cub::DeviceScan::ExclusiveSum(ps_temp(*s, bytes), bytes, s->lens.data(), s->offsets.data(), (int)(m + 1), st);
	s->launches += 2;
	uint32_t total = 0;
	CUDA_CHECK(cudaMemcpyAsync(&total, s->offsets.data() + m, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	CUDA_CHECK(cudaStreamSynchronize(st));
	s->m = m;
	return (long)total;
}

// Phase 2: gather into es[es_base ...]; returns the PES count, lists copied to the host arrays.
int ps_demux_gather(PsScratch *s, uint8_t *es, uint32_t es_base, uint64_t *pts_out, uint32_t *offset_out, int n_max, cudaStream_t st) {
	if (s->m == 0) return 0;
	CUDA_CHECK(cudaMemsetAsync(s->pes_count.data(), 0, sizeof(uint32_t), st));
	ps_gather_kernel<<<s->m, 128, 0, st>>>(s->buf.data(), s->m, s->src.data(), s->lens.data(), s->offsets.data(), s->pts.data(), es, es_base, s->pes_count.data(),
	                                       s->pes_offset.data(), s->pes_pts.data());
	s->launches++;
	uint32_t count = 0;
	CUDA_CHECK(cudaMemcpyAsync(&count, s->pes_count.data(), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	CUDA_CHECK(cudaStreamSynchronize(st));
	if (pts_out && offset_out && n_max > 0) {
		const uint32_t k = count < (uint32_t)n_max ? count : (uint32_t)n_max;
		CUDA_CHECK(cudaMemcpyAsync(pts_out, s->pes_pts.data(), k * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
		CUDA_CHECK(cudaMemcpyAsync(offset_out, s->pes_offset.data(), k * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
		CUDA_CHECK(cudaStreamSynchronize(st));
	}
	return (int)count;
}

uint32_t ps_demux_launches(const PsScratch *s) { return s->launches; }
