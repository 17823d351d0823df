// tsdemux.cu -- MPEG-TS demultiplexing on the device, many streams in one pass (SURVEY.md section 8f, rank 1;
// DESIGN 3.3).
//
// Mirror of the reference's JSMpeg.Demuxer.TS (src/ts.js:25-210): sync byte 0x47 and RESYNC on a
// byte that is not one (:45-50, :155-189), payload_unit_start / PID / adaptation_field_control
// (:52-58), adaptation field skip (:73-77), PES header on a payload start whose next bytes are
// 00 00 01 (:79-126: stream id, PES header length, 33-bit PTS), PID -> stream id binding that EVERY
// PES header of a PID renews (:81-83: a PID re-bound to another stream id stops feeding ours),
// payload bytes appended in packet order (:191-197).  Bytes a write() leaves over (a partial packet,
// a resync that needs more data) are kept for the next one by the caller (engine.cu), like
// leftoverBytes (:25-41).
// What "packet complete" means in the reference (:65-70, :143-146, :201) only decides how the
// payload is CHUNKED into destination.write() calls; the decoder concatenates the chunks, so the
// elementary stream is the concatenation of the accepted payloads.  The host mirror
// (jsmpeg_b200/ts.py) reproduces the chunking too; both are pinned by tests/fixtures/ts_cases.json.
//
// A call demultiplexes many requests (tsdemux.cuh: a stream's left-over bytes and new bytes, its packet
// slots).  The only serial thing in a transport stream is where the packets ARE once sync was lost;
// everything else is per packet:
//   grid     every request's packets lie on its 188-byte grid (checked in parallel, one thread per slot) --
//            or, after a bad sync byte, one warp per such request walks its bytes: 32 grid positions per
//            step, the resync search (187 candidates x 5 sync bytes, ts.js:165-181) spread over the lanes
//   classify one thread per slot: header fields, PES header, payload span; a PES header is the EVENT
//            (request, PID, slot) -> stream id
//   bind     the events are sorted once; a packet's stream id is that of the last event of its (request,
//            PID) at or before it (binary search) -- or the binding the stream carried over, its PID table
//            in HBM, which the last event of each (request, PID) then updates in place
//   place    one exclusive scan of (payload length << 32 | PES start) over all slots gives every packet its
//            ES offset and every PES start its place in the call's list, in (request, offset) order; after
//            the host has made room in the streams, one warp per packet copies the payload to its stream
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "demux.h"
#include "tsdemux.cuh"

namespace {

// the request owning `slot`: the last one whose first slot is <= slot (requests without slots own none)
__device__ __forceinline__ uint32_t request_of(const TsReq *__restrict__ req, uint32_t n_req, uint32_t slot) {
	uint32_t lo = 0, hi = n_req;
	while (lo < hi) {
		const uint32_t mid = (lo + hi) >> 1;
		if (req[mid].slot0 <= slot) lo = mid + 1; else hi = mid;
	}
	return lo - 1;
}

__device__ __forceinline__ uint32_t packet_pos(const TsReqOut &o, const uint32_t *__restrict__ grid, uint32_t slot, uint32_t k) {
	return o.misaligned ? grid[slot] : k * 188u;  // the packet's sync byte, relative to the request
}

// grid, aligned case: is every 188th byte of every request a sync byte?
__global__ void ts_check_grid_kernel(const uint8_t *__restrict__ stage, const TsReq *__restrict__ req, uint32_t n_req,
                                     TsReqOut *__restrict__ out) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= req[n_req].slot0) return;
	const uint32_t r = request_of(req, n_req, i);
	if (stage[req[r].base + (i - req[r].slot0) * 188u] != 0x47) out[r].misaligned = 1;
}

// grid, general case (ts.js:25-50, 155-189): one warp per request.  out.count = packets, out.stop = where parsing stopped.
__global__ void ts_walk_grid_kernel(const uint8_t *__restrict__ stage, const TsReq *__restrict__ req, uint32_t n_req,
                                    uint32_t *__restrict__ grid, TsReqOut *__restrict__ out) {
	const uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int lane = threadIdx.x & 31;
	if (r >= n_req) return;
	const uint32_t n = req[r].n, cap = req[r + 1].slot0 - req[r].slot0;
	if (!out[r].misaligned) {
		if (lane == 0) { out[r].count = cap; out[r].stop = cap * 188u; }
		return;
	}
	const uint8_t *ts = stage + req[r].base;
	uint32_t *g = grid + req[r].slot0;
	uint32_t pos = 0, count = 0;
	while (n - pos >= 188u) {  // bits.has(188 << 3)
		// 32 grid positions at once
		const uint32_t p = pos + 188u * (uint32_t)lane;
		const bool whole = p <= n && n - p >= 188u;
		const bool ok = whole && ts[p] == 0x47;
		const unsigned good = __ballot_sync(0xffffffffu, ok);
		const int m = good == 0xffffffffu ? 32 : __ffs((int)~good) - 1;  // leading packets in sync
		if (lane < m) g[count + lane] = p;
		count += (uint32_t)m;
		pos += 188u * (uint32_t)m;
		if (m == 32 || n - pos < 188u) continue;
		// the byte at pos is not a sync byte: it is consumed (bits.read(8)), then resync() looks at what follows
		pos += 1;
		if (n - pos < TS_RESYNC_BYTES) break;  // not enough data to attempt a resync: maybe next time
		int found = -1;
		for (int base = 0; base < 187 && found < 0; base += 32) {
			const int i = base + lane;
			const unsigned any = __ballot_sync(0xffffffffu, i < 187 && ts_resync_at(ts, pos, (uint32_t)i));
			if (any) found = base + __ffs((int)any) - 1;
		}
		if (found < 0) { pos += 187; break; }  // garbage: skip it, give up for this write()
		if (lane == 0) g[count] = pos + (uint32_t)found;
		count++;
		pos = pos + (uint32_t)found + 188u;
	}
	if (lane == 0) { out[r].count = count; out[r].stop = pos; }
}

// classify: one thread per slot (ts.js:52-58, 73-126)
__global__ void ts_classify_kernel(const uint8_t *__restrict__ stage, const TsReq *__restrict__ req, uint32_t n_req,
                                   const uint32_t *__restrict__ grid, const TsReqOut *__restrict__ out, TsPacketInfo *__restrict__ info,
                                   uint64_t *__restrict__ pts, uint64_t *__restrict__ ev_key, uint32_t *__restrict__ ev_val) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= req[n_req].slot0) return;
	const uint32_t r = request_of(req, n_req, i), k = i - req[r].slot0;
	const TsReqOut o = out[r];
	TsPacketInfo pi{0, 0, 0, 188, 0};
	uint64_t t = 0;
	if (k < o.count) pi = ts_classify(stage + req[r].base, req[r].n, packet_pos(o, grid, i, k), &t);
	info[i] = pi;
	pts[i] = t;
	ev_key[i] = (pi.flags & 2) ? ts_event_key(r, pi.pid, i) : TS_NO_EVENT;
	ev_val[i] = pi.sid;
}

// bind: stream id in force for every packet; payload span of ours (ts.js:128-150, 191-197).  lenpes[i] =
// payload length << 32 | PES start, with a 0 behind the last slot for the scan's total.
__global__ void ts_bind_kernel(const TsReq *__restrict__ req, uint32_t n_req, const TsPacketInfo *__restrict__ info,
                               const uint64_t *__restrict__ ev_key, const uint32_t *__restrict__ ev_val, TsPacketUse *__restrict__ use,
                               uint64_t *__restrict__ lenpes) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, n_slots = req[n_req].slot0;
	if (i > n_slots) return;
	TsPacketUse u{0, 0};
	int pes = 0;
	if (i < n_slots) {
		const TsPacketInfo pi = info[i];
		if (pi.flags & 1) {
			const uint32_t r = request_of(req, n_req, i);
			const int sid = ts_binding(ev_key, ev_val, n_slots, r, pi.pid, i, req[r].bound);
			u = ts_use(pi, sid, req[r].stream_id, &pes);
		}
		use[i] = u;
	}
	lenpes[i] = (uint64_t)u.len << 32 | (uint64_t)pes;
}

// what the PIDs of each stream are bound to after this call: the stream id of the last event of each (request, PID)
__global__ void ts_carry_kernel(const TsReq *__restrict__ req, uint32_t n_req, const uint64_t *__restrict__ ev_key,
                                const uint32_t *__restrict__ ev_val) {
	const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x, n_slots = req[n_req].slot0;
	if (e >= n_slots || ev_key[e] == TS_NO_EVENT) return;
	const uint64_t group = ev_key[e] >> TS_SLOT_BITS;
	if (e + 1 == n_slots || (ev_key[e + 1] >> TS_SLOT_BITS) != group) {
		const uint32_t r = (uint32_t)(group >> TS_PID_BITS), pid = (uint32_t)(group & 8191u);
		req[r].bound[pid] = (int16_t)ev_val[e];
	}
}

// per request: ES bytes, PES starts and where its PES starts begin in the call's list
__global__ void ts_totals_kernel(const TsReq *__restrict__ req, uint32_t n_req, const uint64_t *__restrict__ scan, TsReqOut *__restrict__ out) {
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= n_req) return;
	const uint64_t a = scan[req[r].slot0], b = scan[req[r + 1].slot0];
	out[r].total = (uint32_t)(b >> 32) - (uint32_t)(a >> 32);
	out[r].pes = (uint32_t)b - (uint32_t)a;
	out[r].pes_first = (uint32_t)a;
}

// place: one warp copies one packet's payload to its stream and lists a PES start; warps n_slots + r then zero the
// `pad` bytes behind request r's new ES bytes (the kernels read zeros there)
__global__ void ts_gather_kernel(const uint8_t *__restrict__ stage, const TsReq *__restrict__ req, uint32_t n_req,
                                 const uint32_t *__restrict__ grid, const TsReqOut *__restrict__ out, const TsPacketUse *__restrict__ use,
                                 const uint64_t *__restrict__ scan, const uint64_t *__restrict__ pts, uint32_t pad,
                                 uint32_t *__restrict__ pes_offset, uint64_t *__restrict__ pes_pts) {
	const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_slots = req[n_req].slot0;
	const int lane = threadIdx.x & 31;
	if (w >= n_slots) {
		const uint32_t r = w - n_slots;
		if (r < n_req && req[r].dst)
			for (uint32_t k = lane; k < pad; k += 32) req[r].dst[out[r].total + k] = 0;
		return;
	}
	const uint32_t r = request_of(req, n_req, w), k = w - req[r].slot0;
	const TsReqOut o = out[r];
	if (k >= o.count || !req[r].dst) return;
	const uint64_t at = scan[w];
	const uint32_t off = (uint32_t)(at >> 32) - (uint32_t)(scan[req[r].slot0] >> 32);
	const TsPacketUse u = use[w];
	if (lane == 0 && (uint32_t)scan[w + 1] != (uint32_t)at) {  // a PES start
		pes_offset[(uint32_t)at] = req[r].es_base + off;
		pes_pts[(uint32_t)at] = pts[w];
	}
	const uint8_t *src = stage + req[r].base + packet_pos(o, grid, w, k) + u.start;
	uint8_t *dst = req[r].dst + off;
	for (int b = lane; b < u.len; b += 32) dst[b] = src[b];
}

constexpr int BLOCK = 256;
int blocks(uint64_t threads) { return (int)((threads + BLOCK - 1) / BLOCK); }

}  // namespace

struct TsScratch {
	DeviceBuffer<uint32_t> grid;
	DeviceBuffer<TsPacketInfo> info;
	DeviceBuffer<TsPacketUse> use;
	DeviceBuffer<uint64_t> pts, lenpes, scan;
	DeviceBuffer<uint64_t> ev_key, ev_key2;
	DeviceBuffer<uint32_t> ev_val, ev_val2;
	uint32_t n_req = 0, n_slots = 0;
	int key_bits = 0;
};

TsScratch *ts_scratch_create() { return new TsScratch(); }
void ts_scratch_destroy(TsScratch *s) { delete s; }

void ts_call_begin(TsScratch *s, TsIo &io, uint32_t n_req, uint32_t n_slots, uint32_t max_req) {
	const uint32_t m = n_slots;
	s->n_req = n_req;
	s->n_slots = n_slots;
	s->key_bits = TS_PID_BITS + TS_SLOT_BITS;
	while (s->key_bits < 64 && (1ull << (s->key_bits - TS_PID_BITS - TS_SLOT_BITS)) < max_req) s->key_bits++;
	if (m + 1 > s->grid.size()) {
		const size_t cap = m + 1 + m / 4 + 8;
		s->grid.reserve(cap);
		s->info.reserve(cap);
		s->use.reserve(cap);
		s->pts.reserve(cap);
		s->lenpes.reserve(cap);
		s->scan.reserve(cap);
		s->ev_key.reserve(cap);
		s->ev_key2.reserve(cap);
		s->ev_val.reserve(cap);
		s->ev_val2.reserve(cap);
	}
	io.reserve_pes(m);  // (a PES start per packet at most)
}

uint32_t ts_call_measure(TsScratch *s, TsIo &io, cudaStream_t st) {
	const uint32_t n = s->n_req, m = s->n_slots;
	CUDA_CHECK(cudaMemsetAsync(io.out.data(), 0, n * sizeof(TsReqOut), st));
	ts_check_grid_kernel<<<blocks(m), BLOCK, 0, st>>>(io.stage.data(), io.req.data(), n, io.out.data());
	ts_walk_grid_kernel<<<blocks((uint64_t)n * 32), BLOCK, 0, st>>>(io.stage.data(), io.req.data(), n, s->grid.data(), io.out.data());
	ts_classify_kernel<<<blocks(m), BLOCK, 0, st>>>(io.stage.data(), io.req.data(), n, s->grid.data(), io.out.data(), s->info.data(),
	                                                 s->pts.data(), s->ev_key.data(), s->ev_val.data());
	size_t bytes = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, bytes, s->ev_key.data(), s->ev_key2.data(), s->ev_val.data(), s->ev_val2.data(), (int)m, 0,
	                                s->key_bits, st);
	cub::DeviceRadixSort::SortPairs(io.temp_storage(bytes), bytes, s->ev_key.data(), s->ev_key2.data(), s->ev_val.data(),
	                                s->ev_val2.data(), (int)m, 0, s->key_bits, st);
	ts_bind_kernel<<<blocks((uint64_t)m + 1), BLOCK, 0, st>>>(io.req.data(), n, s->info.data(), s->ev_key2.data(), s->ev_val2.data(),
	                                                          s->use.data(), s->lenpes.data());
	ts_carry_kernel<<<blocks(m), BLOCK, 0, st>>>(io.req.data(), n, s->ev_key2.data(), s->ev_val2.data());
	bytes = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, bytes, s->lenpes.data(), s->scan.data(), (int)(m + 1), st);
	cub::DeviceScan::ExclusiveSum(io.temp_storage(bytes), bytes, s->lenpes.data(), s->scan.data(), (int)(m + 1), st);
	ts_totals_kernel<<<blocks(n), BLOCK, 0, st>>>(io.req.data(), n, s->scan.data(), io.out.data());
	CUDA_CHECK(cudaMemcpyAsync(io.h_out.data(), io.out.data(), n * sizeof(TsReqOut), cudaMemcpyDeviceToHost, st));
	return 8;  // (a cub algorithm counts as one launch)
}

uint32_t ts_call_gather(TsScratch *s, TsIo &io, uint32_t pad, cudaStream_t st) {
	const uint32_t n = s->n_req, m = s->n_slots;
	ts_gather_kernel<<<blocks(((uint64_t)m + n) * 32), BLOCK, 0, st>>>(io.stage.data(), io.req.data(), n, s->grid.data(), io.out.data(),
	                                                                    s->use.data(), s->scan.data(), s->pts.data(), pad,
	                                                                    io.pes_offset.data(), io.pes_pts.data());
	return 1;
}
