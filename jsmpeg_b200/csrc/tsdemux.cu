// tsdemux.cu -- MPEG-TS demultiplexing on the device (SURVEY.md section 8f, rank 1).
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
// Decomposition.  The only serial thing in a transport stream is where the packets ARE once sync was
// lost; everything else is per packet:
//   grid     packets lie on the 188-byte grid (checked in parallel) -- or, after a bad sync byte, one
//            warp walks the buffer: 32 grid positions per step, the resync search (187 candidates x
//            5 sync bytes, ts.js:165-181) spread over the lanes
//   classify one thread per packet: header fields, PES header, payload span; PES headers become
//            (PID, packet index) -> stream id EVENTS
//   bind     the events are sorted by (PID, packet index); a packet's stream id is that of the last
//            event of its PID at or before it (binary search) -- or the binding carried over from the
//            previous write()
//   place    exclusive scan of the payload lengths, one warp copies a packet's payload to its place;
//            PES starts (offset in the ES, PTS) are appended to a list for the host's PTS table
//            (src/decoder.js:36-47).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "buffers.h"
#include "common.cuh"

namespace {

struct PacketUse {
	uint16_t start;  // first payload byte inside the packet (may be >= 188: nothing to copy)
	uint16_t len;    // payload bytes that go to the elementary stream (0 = none)
};

struct PacketInfo {      // classify -> bind
	uint16_t pid;
	uint8_t flags;       // 1 payload present (adaptation_field_control & 1), 2 PES header here
	uint8_t sid;         // PES header: its stream id
	uint16_t at;         // first byte after the adaptation field; PES header: first byte after the PES header
	uint16_t pad;
};

__device__ __forceinline__ uint32_t rd(const uint8_t *__restrict__ ts, uint32_t n, uint32_t i) {
	return i < n ? ts[i] : 0u;  // a read past the buffer yields 0 in the reference's bit reader (undefined & mask)
}

__device__ __forceinline__ uint32_t packet_pos(const uint32_t *__restrict__ grid, uint32_t i) {
	return grid ? grid[i] : i * 188u;  // position of the packet's sync byte
}

// grid, aligned case: every 188th byte is a sync byte?
__global__ void ts_check_grid_kernel(const uint8_t *__restrict__ ts, uint32_t n_packets, int *__restrict__ misaligned) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n_packets && ts[(size_t)i * 188] != 0x47) *misaligned = 1;
}

// grid, general case (ts.js:25-50, 155-189): ONE warp.  out[0] = packet count, out[1] = where parsing stopped.
__global__ void ts_walk_grid_kernel(const uint8_t *__restrict__ ts, uint32_t n, uint32_t *__restrict__ grid, uint32_t *__restrict__ out) {
	const int lane = threadIdx.x;
	uint32_t pos = 0, count = 0;
	while (n - pos >= 188u) {  // bits.has(188 << 3)
		// 32 grid positions at once
		const uint32_t p = pos + 188u * (uint32_t)lane;
		const bool whole = p <= n && n - p >= 188u;
		const bool ok = whole && ts[p] == 0x47;
		const unsigned good = __ballot_sync(0xffffffffu, ok);
		const int m = good == 0xffffffffu ? 32 : __ffs((int)~good) - 1;  // leading packets in sync
		if (lane < m) grid[count + lane] = p;
		count += (uint32_t)m;
		pos += 188u * (uint32_t)m;
		if (m == 32 || n - pos < 188u) continue;
		// the byte at pos is not a sync byte: it is consumed (bits.read(8)), then resync() looks at what follows
		pos += 1;
		if (n - pos < 188u * 6u) break;  // not enough data to attempt a resync: maybe next time
		int found = -1;
		for (int base = 0; base < 187 && found < 0; base += 32) {
			const int i = base + lane;
			bool hit = false;
			if (i < 187 && ts[pos + i] == 0x47) {
				hit = true;
				for (int j = 1; j < 5; j++) hit = hit && ts[pos + i + 188 * j] == 0x47;
			}
			const unsigned any = __ballot_sync(0xffffffffu, hit);
			if (any) found = base + __ffs((int)any) - 1;
		}
		if (found < 0) { pos += 187; break; }  // garbage: skip it, give up for this write()
		if (lane == 0) grid[count] = pos + (uint32_t)found;
		count++;
		pos = pos + (uint32_t)found + 188u;
	}
	if (lane == 0) { out[0] = count; out[1] = pos; }
}

// classify: one thread per packet (ts.js:52-58, 73-126)
__global__ void ts_classify_kernel(const uint8_t *__restrict__ ts, uint32_t n, const uint32_t *__restrict__ grid, uint32_t n_packets,
                                   PacketInfo *__restrict__ info, uint64_t *__restrict__ pts, uint64_t *__restrict__ ev_key,
                                   uint32_t *__restrict__ ev_val, uint32_t *__restrict__ ev_count) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_packets) return;
	const uint32_t p0 = packet_pos(grid, i);  // sync byte; the packet is wholly inside the buffer
	const uint32_t b1 = ts[p0 + 1], b2 = ts[p0 + 2], b3 = ts[p0 + 3];
	const int pusi = (b1 >> 6) & 1;
	const int pid = ((b1 & 0x1f) << 8) | b2;
	const int afc = (b3 >> 4) & 3;
	PacketInfo pi{(uint16_t)pid, 0, 0, 188, 0};
	uint64_t t = 0;
	if (afc & 1) {
		uint32_t at = 4;
		if (afc & 2) at += 1 + ts[p0 + 4];  // adaptation_field_length may point past the packet: `at` is then > 188
		pi.flags = 1;
		// nextBytesAreStartCode (buffer.js:141-150) looks at the BUFFER, not the packet: true at its very end
		const uint32_t q = p0 + at;
		if (pusi && (q >= n || (rd(ts, n, q) == 0 && rd(ts, n, q + 1) == 0 && rd(ts, n, q + 2) == 1))) {
			pi.flags = 3;
			pi.sid = (uint8_t)rd(ts, n, q + 3);
			if (rd(ts, n, q + 7) & 0x80) {  // PTS present (ts.js:94-116)
				const uint32_t c0 = rd(ts, n, q + 9), c1 = rd(ts, n, q + 10), c2 = rd(ts, n, q + 11), c3 = rd(ts, n, q + 12), c4 = rd(ts, n, q + 13);
				t = ((uint64_t)((c0 >> 1) & 7) << 30) | ((uint64_t)((c1 << 7) | (c2 >> 1)) << 15) | (uint64_t)((c3 << 7) | (c4 >> 1));
			}
			at += 9 + rd(ts, n, q + 8);
			const uint32_t k = atomicAdd(ev_count, 1u);
			ev_key[k] = ((uint64_t)pid << 32) | (uint64_t)(i + 1u);  // index 0 is the binding carried over from earlier writes
			ev_val[k] = pi.sid;
		}
		pi.at = (uint16_t)(at > 0xffffu ? 0xffffu : at);
	}
	info[i] = pi;
	pts[i] = t;
}

// bind: stream id in force for every packet; payload span of ours (ts.js:128-150, 191-197)
__global__ void ts_bind_kernel(uint32_t n_packets, const PacketInfo *__restrict__ info, const uint64_t *__restrict__ ev_key,
                               const uint32_t *__restrict__ ev_val, uint32_t n_events, int stream_id, PacketUse *__restrict__ use,
                               uint32_t *__restrict__ lens, uint8_t *__restrict__ is_pes) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_packets) return;
	const PacketInfo pi = info[i];
	PacketUse u{0, 0};
	uint8_t pes = 0;
	if (pi.flags & 1) {
		// last event with key <= (pid, i + 1): upper bound - 1
		const uint64_t want = ((uint64_t)pi.pid << 32) | (uint64_t)(i + 1u);
		uint32_t lo = 0, hi = n_events;
		while (lo < hi) {
			const uint32_t mid = (lo + hi) >> 1;
			if (ev_key[mid] <= want) lo = mid + 1; else hi = mid;
		}
		int sid = 0;  // unbound (undefined in the reference) and stream id 0 both mean "nobody" (ts.js:128)
		if (lo > 0 && (uint32_t)(ev_key[lo - 1] >> 32) == pi.pid) sid = (int)ev_val[lo - 1];
		if (sid != 0 && sid == stream_id) {
			pes = (pi.flags & 2) ? 1 : 0;
			if (pi.at < 188) { u.start = pi.at; u.len = (uint16_t)(188 - pi.at); }
		}
	}
	use[i] = u;
	lens[i] = u.len;
	is_pes[i] = pes;
}

// what the PIDs are bound to after this buffer: the stream id of each PID's last event
__global__ void ts_carry_kernel(const uint64_t *__restrict__ ev_key, const uint32_t *__restrict__ ev_val, uint32_t n_events,
                                int16_t *__restrict__ bound) {
	const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= n_events) return;
	const uint32_t pid = (uint32_t)(ev_key[e] >> 32);
	if (e + 1 == n_events || (uint32_t)(ev_key[e + 1] >> 32) != pid) bound[pid] = (int16_t)ev_val[e];
}

// place: one warp copies one packet's payload to its place; PES starts are appended to a list
__global__ void ts_gather_kernel(const uint8_t *__restrict__ ts, const uint32_t *__restrict__ grid, uint32_t n_packets,
                                 const PacketUse *__restrict__ use, const uint32_t *__restrict__ offsets, const uint8_t *__restrict__ is_pes,
                                 const uint64_t *__restrict__ pts, uint8_t *__restrict__ es, uint32_t es_base,
                                 uint32_t *__restrict__ pes_count, uint32_t pes_cap, uint32_t *__restrict__ pes_offset,
                                 uint64_t *__restrict__ pes_pts) {
	const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int lane = threadIdx.x & 31;
	if (i >= n_packets) return;
	const PacketUse u = use[i];
	const uint32_t off = offsets[i];
	if (lane == 0 && is_pes[i]) {
		const uint32_t k = atomicAdd(pes_count, 1u);
		if (k < pes_cap) { pes_offset[k] = es_base + off; pes_pts[k] = pts[i]; }
	}
	const uint8_t *src = ts + packet_pos(grid, i) + u.start;
	uint8_t *dst = es + es_base + off;
	for (int k = lane; k < u.len; k += 32) dst[k] = src[k];
}

}  // namespace

struct TsScratch {
	DeviceBuffer<uint8_t> ts;  // 16 bytes of slack past the packets
	DeviceBuffer<uint32_t> grid, grid_out;
	DeviceBuffer<PacketInfo> info;
	DeviceBuffer<PacketUse> use;
	DeviceBuffer<uint32_t> lens, offsets;
	DeviceBuffer<uint8_t> is_pes;
	DeviceBuffer<uint64_t> pts;
	DeviceBuffer<uint64_t> ev_key, ev_key2;
	DeviceBuffer<uint32_t> ev_val, ev_val2, ev_count;
	DeviceBuffer<int16_t> bound;
	DeviceBuffer<uint32_t> pes_count, pes_offset;
	DeviceBuffer<uint64_t> pes_pts;
	DeviceBuffer<int> misaligned;
	DeviceBuffer<uint8_t> scan_temp, sort_temp;  // cub's temporary storage
	size_t n_cap = 0;  // packets the per-packet arrays have room for
	bool grid_in_use = false;
	uint32_t n_packets = 0;
};

static void ts_reserve(TsScratch &s, size_t ts_bytes, size_t n) {
	if (ts_bytes + 16 > s.ts.size()) s.ts.reserve(ts_bytes + ts_bytes / 4 + 16);
	s.bound.reserve(8192);
	s.misaligned.reserve(1);
	s.pes_count.reserve(1);
	s.ev_count.reserve(1);
	s.grid_out.reserve(2);
	if (n > s.n_cap) {
		const size_t cap = n + n / 4 + 8;
		const size_t ev_cap = cap + 8192;  // one event per packet at most, plus the carried bindings
		s.grid.reserve(cap);
		s.info.reserve(cap);
		s.use.reserve(cap);
		s.lens.reserve(cap + 1);
		s.offsets.reserve(cap + 1);
		s.is_pes.reserve(cap);
		s.pts.reserve(cap);
		s.ev_key.reserve(ev_cap);
		s.ev_key2.reserve(ev_cap);
		s.ev_val.reserve(ev_cap);
		s.ev_val2.reserve(ev_cap);
		s.pes_offset.reserve(cap);
		s.pes_pts.reserve(cap);
		size_t bytes = 0;
		cub::DeviceScan::ExclusiveSum(nullptr, bytes, s.lens.data(), s.offsets.data(), (int)(cap + 1));
		s.scan_temp.reserve(bytes);
		bytes = 0;
		cub::DeviceRadixSort::SortPairs(nullptr, bytes, s.ev_key.data(), s.ev_key2.data(), s.ev_val.data(), s.ev_val2.data(), (int)ev_cap,
		                                0, 45);
		s.sort_temp.reserve(bytes);
		s.n_cap = cap;
	}
}

TsScratch *ts_scratch_create() { return new TsScratch(); }
void ts_scratch_destroy(TsScratch *s) { delete s; }

// Phase 1: upload + grid + classify + bind + scan.  `bound` [8192]: the stream id every PID is bound to
// (0 = none), in/out (pidsToStreamIds lives across write() calls, ts.js:9).  Returns the ES byte count;
// *consumed = bytes of the buffer the demuxer is done with (the rest is the caller's leftover).
long ts_demux_measure(TsScratch *s, const uint8_t *ts_host, size_t ts_bytes, int stream_id, int16_t *bound, size_t *consumed, cudaStream_t st) {
	*consumed = 0;
	s->n_packets = 0;
	if (ts_bytes < 188) return 0;  // not a whole packet yet: everything stays with the caller
	if (ts_bytes > 0xfffff000ull) throw std::runtime_error("jsmpeg_b200: transport stream buffer of 4 GiB or more");
	const size_t n_max = ts_bytes / 188;
	ts_reserve(*s, ts_bytes, n_max);
	const uint32_t n = (uint32_t)ts_bytes;
	CUDA_CHECK(cudaMemcpyAsync(s->ts.data(), ts_host, ts_bytes, cudaMemcpyHostToDevice, st));
	CUDA_CHECK(cudaMemsetAsync(s->misaligned.data(), 0, sizeof(int), st));
	CUDA_CHECK(cudaMemsetAsync(s->pes_count.data(), 0, sizeof(uint32_t), st));
	const int block = 256;
	int grid_n = (int)((n_max + block - 1) / block);
	ts_check_grid_kernel<<<grid_n, block, 0, st>>>(s->ts.data(), (uint32_t)n_max, s->misaligned.data());
	int misaligned = 0;
	CUDA_CHECK(cudaMemcpyAsync(&misaligned, s->misaligned.data(), sizeof(int), cudaMemcpyDeviceToHost, st));
	CUDA_CHECK(cudaStreamSynchronize(st));
	uint32_t n_packets = (uint32_t)n_max, stop = (uint32_t)(n_max * 188);
	s->grid_in_use = misaligned != 0;
	if (misaligned) {  // sync was lost somewhere: one warp walks the buffer the way the reference does
		ts_walk_grid_kernel<<<1, 32, 0, st>>>(s->ts.data(), n, s->grid.data(), s->grid_out.data());
		uint32_t out[2] = {0, 0};
		CUDA_CHECK(cudaMemcpyAsync(out, s->grid_out.data(), sizeof(out), cudaMemcpyDeviceToHost, st));
		CUDA_CHECK(cudaStreamSynchronize(st));
		n_packets = out[0];
		stop = out[1];
	}
	*consumed = stop;
	s->n_packets = n_packets;
	if (n_packets == 0) return 0;
	const uint32_t *grid = s->grid_in_use ? s->grid.data() : nullptr;
	// events: the carried bindings first (index 0 of their PID), then the PES headers of this buffer
	static thread_local uint64_t carry_key[8192];
	static thread_local uint32_t carry_val[8192];
	uint32_t n_carry = 0;
	for (uint32_t pid = 0; pid < 8192; pid++)
		if (bound[pid]) { carry_key[n_carry] = (uint64_t)pid << 32; carry_val[n_carry] = (uint32_t)(uint16_t)bound[pid]; n_carry++; }
	if (n_carry) {
		CUDA_CHECK(cudaMemcpyAsync(s->ev_key.data(), carry_key, n_carry * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
		CUDA_CHECK(cudaMemcpyAsync(s->ev_val.data(), carry_val, n_carry * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
	}
	CUDA_CHECK(cudaMemcpyAsync(s->ev_count.data(), &n_carry, sizeof(uint32_t), cudaMemcpyHostToDevice, st));
	grid_n = (int)((n_packets + block - 1) / block);
	ts_classify_kernel<<<grid_n, block, 0, st>>>(s->ts.data(), n, grid, n_packets, s->info.data(), s->pts.data(), s->ev_key.data(),
	                                             s->ev_val.data(), s->ev_count.data());
	uint32_t n_events = 0;
	CUDA_CHECK(cudaMemcpyAsync(&n_events, s->ev_count.data(), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	CUDA_CHECK(cudaStreamSynchronize(st));  // (also: carry_key / carry_val / n_carry have been read)
	const uint64_t *keys = s->ev_key.data();
	const uint32_t *vals = s->ev_val.data();
	if (n_events > 1) {
		size_t bytes = s->sort_temp.size();
		cub::DeviceRadixSort::SortPairs(s->sort_temp.data(), bytes, s->ev_key.data(), s->ev_key2.data(), s->ev_val.data(), s->ev_val2.data(),
		                                (int)n_events, 0, 45, st);
		keys = s->ev_key2.data();
		vals = s->ev_val2.data();
	}
	ts_bind_kernel<<<grid_n, block, 0, st>>>(n_packets, s->info.data(), keys, vals, n_events, stream_id, s->use.data(), s->lens.data(),
	                                         s->is_pes.data());
	if (n_events) {
		static thread_local int16_t host_bound[8192];
		memcpy(host_bound, bound, sizeof(host_bound));
		CUDA_CHECK(cudaMemcpyAsync(s->bound.data(), host_bound, sizeof(host_bound), cudaMemcpyHostToDevice, st));
		ts_carry_kernel<<<(int)((n_events + block - 1) / block), block, 0, st>>>(keys, vals, n_events, s->bound.data());
		CUDA_CHECK(cudaMemcpyAsync(host_bound, s->bound.data(), sizeof(host_bound), cudaMemcpyDeviceToHost, st));
		CUDA_CHECK(cudaStreamSynchronize(st));
		memcpy(bound, host_bound, sizeof(host_bound));
	}
	CUDA_CHECK(cudaMemsetAsync(s->lens.data() + n_packets, 0, sizeof(uint32_t), st));
	size_t bytes = s->scan_temp.size();
	cub::DeviceScan::ExclusiveSum(s->scan_temp.data(), bytes, s->lens.data(), s->offsets.data(), (int)(n_packets + 1), st);
	uint32_t total = 0;
	CUDA_CHECK(cudaMemcpyAsync(&total, s->offsets.data() + n_packets, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	CUDA_CHECK(cudaStreamSynchronize(st));
	return (long)total;
}

// Phase 2: gather into es[es_base ...]; returns the PES count, lists copied to the host arrays.
int ts_demux_gather(TsScratch *s, uint8_t *es, uint32_t es_base, uint64_t *pts_out, uint32_t *offset_out, int n_max, cudaStream_t st) {
	const size_t n = s->n_packets;
	if (n == 0) return 0;
	const int block = 256;
	const int grid = (int)((n * 32 + block - 1) / block);
	ts_gather_kernel<<<grid, block, 0, st>>>(s->ts.data(), s->grid_in_use ? s->grid.data() : nullptr, (uint32_t)n, s->use.data(),
	                                         s->offsets.data(), s->is_pes.data(), s->pts.data(), es, es_base, s->pes_count.data(),
	                                         (uint32_t)s->n_cap, s->pes_offset.data(), s->pes_pts.data());
	uint32_t count = 0;
	CUDA_CHECK(cudaMemcpyAsync(&count, s->pes_count.data(), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	CUDA_CHECK(cudaStreamSynchronize(st));
	if (pts_out && offset_out && n_max > 0) {
		const uint32_t m = count < (uint32_t)n_max ? count : (uint32_t)n_max;
		CUDA_CHECK(cudaMemcpyAsync(pts_out, s->pes_pts.data(), m * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
		CUDA_CHECK(cudaMemcpyAsync(offset_out, s->pes_offset.data(), m * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
		CUDA_CHECK(cudaStreamSynchronize(st));
	}
	return (int)count;
}
