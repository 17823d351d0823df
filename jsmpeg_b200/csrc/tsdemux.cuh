// tsdemux.cuh -- per-packet arithmetic of the MPEG-TS demuxer (tsdemux.cu), kept apart so that the host
// compiler can build it too (tests/emu/ts_many_check.cpp runs the segmented pass with it against the host
// mirror of src/ts.js, jsmpeg_b200/ts.py).
//
// One call demultiplexes many REQUESTS (a stream's left-over bytes followed by the new ones).  Their bytes
// lie one after another in a staging buffer and every request owns a run of packet SLOTS, one per 188
// bytes it holds (the most packets it can have); a slot past the request's packet count is idle.
// Positions handed to the functions here are relative to the request's first byte, and `n` is the
// request's length: a read past it is 0 and its end counts as a start code, as in the reference
// (src/buffer.js:141-150, 152-170).
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

constexpr uint32_t TS_PACKET = 188;
constexpr uint32_t TS_RESYNC_BYTES = 188 * 6;  // a resync needs this many bytes after the bad sync byte (ts.js:155-189)
// event keys (request, PID, slot + 1): a call's slots number < 2^32 / 188 < 2^25
constexpr int TS_SLOT_BITS = 25;
constexpr int TS_PID_BITS = 13;
constexpr uint64_t TS_NO_EVENT = ~0ull;  // the key of a slot without a PES header; sorts behind every event

struct TsReq {  // one request of a call, the host fills it
	uint32_t base;       // first byte in the staging buffer
	uint32_t n;          // bytes: the stream's left-over bytes, then the new ones
	uint32_t slot0;      // first packet slot; the request owns n / 188 of them (entry [n_req]: the call's slot count)
	int stream_id;       // PES stream id that feeds the stream
	int16_t *bound;      // the stream's PID -> stream id table (8192 entries, in HBM), read and updated in place
	uint8_t *dst;        // where its ES bytes go (the stream's ES mirror at es_base); set after the totals are known
	uint32_t es_base;    // the stream's ES length before this write
	uint32_t pad;
};

struct TsReqOut {  // per request, the device fills it
	uint32_t misaligned;  // a 188-byte grid position is not a sync byte
	uint32_t count;       // packets
	uint32_t stop;        // bytes consumed (the rest stays for the stream's next write)
	uint32_t total;       // ES bytes
	uint32_t pes;         // PES starts of the stream
	uint32_t pes_first;   // index of its first PES start in the call's list
};

struct TsPacketInfo {  // classify -> bind
	uint16_t pid;
	uint8_t flags;  // 1 payload present (adaptation_field_control & 1), 2 PES header here
	uint8_t sid;    // PES header: its stream id
	uint16_t at;    // first byte after the adaptation field; PES header: first byte after the PES header
	uint16_t pad;
};

struct TsPacketUse {
	uint16_t start;  // first payload byte inside the packet
	uint16_t len;    // payload bytes that go to the elementary stream (0 = none)
};

__host__ __device__ inline uint32_t ts_rd(const uint8_t *ts, uint32_t n, uint32_t i) {
	return i < n ? ts[i] : 0u;  // a read past the request yields 0 in the reference's bit reader (undefined & mask)
}

// Header fields, PES header and PTS of the packet whose sync byte is at p0 (ts.js:52-58, 73-126); the packet is
// wholly inside the request.  *pts = the PES header's 90 kHz PTS, 0 if absent.
__host__ __device__ inline TsPacketInfo ts_classify(const uint8_t *ts, uint32_t n, uint32_t p0, uint64_t *pts) {
	const uint32_t b1 = ts[p0 + 1], b2 = ts[p0 + 2], b3 = ts[p0 + 3];
	const int pusi = (b1 >> 6) & 1;
	const uint32_t pid = ((b1 & 0x1f) << 8) | b2;
	const int afc = (b3 >> 4) & 3;
	TsPacketInfo pi{(uint16_t)pid, 0, 0, 188, 0};
	*pts = 0;
	if (afc & 1) {
		uint32_t at = 4;
		if (afc & 2) at += 1 + ts[p0 + 4];  // adaptation_field_length may point past the packet: `at` is then > 188
		pi.flags = 1;
		// nextBytesAreStartCode looks at the BUFFER, not the packet: true at its very end
		const uint32_t q = p0 + at;
		if (pusi && (q >= n || (ts_rd(ts, n, q) == 0 && ts_rd(ts, n, q + 1) == 0 && ts_rd(ts, n, q + 2) == 1))) {
			pi.flags = 3;
			pi.sid = (uint8_t)ts_rd(ts, n, q + 3);
			if (ts_rd(ts, n, q + 7) & 0x80) {  // PTS present (ts.js:94-116)
				const uint32_t c0 = ts_rd(ts, n, q + 9), c1 = ts_rd(ts, n, q + 10), c2 = ts_rd(ts, n, q + 11);
				const uint32_t c3 = ts_rd(ts, n, q + 12), c4 = ts_rd(ts, n, q + 13);
				*pts = ((uint64_t)((c0 >> 1) & 7) << 30) | ((uint64_t)((c1 << 7) | (c2 >> 1)) << 15) | (uint64_t)((c3 << 7) | (c4 >> 1));
			}
			at += 9 + ts_rd(ts, n, q + 8);
		}
		pi.at = (uint16_t)(at > 0xffffu ? 0xffffu : at);
	}
	return pi;
}

// One candidate of a resync after the byte before `pos` was not a sync byte: does a packet start at pos + i
// (i < 187), i.e. are there sync bytes at pos + i + 188 j for j = 0..4 (ts.js:165-181)?  The caller has
// made sure that n - pos >= TS_RESYNC_BYTES.
__host__ __device__ inline bool ts_resync_at(const uint8_t *ts, uint32_t pos, uint32_t i) {
	bool hit = ts[pos + i] == 0x47;
	for (uint32_t j = 1; j < 5; j++) hit = hit && ts[pos + i + 188 * j] == 0x47;
	return hit;
}

// The event of a PES header of `pid` in `slot` of request r
__host__ __device__ inline uint64_t ts_event_key(uint32_t r, uint32_t pid, uint32_t slot) {
	return ((uint64_t)r << (TS_PID_BITS + TS_SLOT_BITS)) | ((uint64_t)pid << TS_SLOT_BITS) | (uint64_t)(slot + 1u);
}

// The stream id `pid` is bound to in `slot` of request r: that of the last event of (r, pid) at or before the
// slot among the sorted keys[0 .. n_keys) -- or, without one, the binding carried over from the stream's earlier
// writes, bound[pid] (ts.js:81-83; 0 = nobody)
__host__ __device__ inline int ts_binding(const uint64_t *keys, const uint32_t *vals, uint32_t n_keys, uint32_t r, uint32_t pid,
                                          uint32_t slot, const int16_t *bound) {
	const uint64_t want = ts_event_key(r, pid, slot);
	uint32_t lo = 0, hi = n_keys;
	while (lo < hi) {  // upper bound
		const uint32_t mid = (lo + hi) >> 1;
		if (keys[mid] <= want) lo = mid + 1; else hi = mid;
	}
	if (lo > 0 && (keys[lo - 1] >> TS_SLOT_BITS) == (want >> TS_SLOT_BITS)) return (int)vals[lo - 1];
	return bound[pid];
}

// What of the packet goes to a stream fed by `stream_id` when its PID is bound to `sid` (ts.js:128-150, 191-197);
// *pes = 1 if a PES packet of the stream starts here
__host__ __device__ inline TsPacketUse ts_use(TsPacketInfo pi, int sid, int stream_id, int *pes) {
	TsPacketUse u{0, 0};
	*pes = 0;
	if ((pi.flags & 1) && sid != 0 && sid == stream_id) {  // unbound (undefined in the reference) and 0 both mean nobody
		*pes = (pi.flags & 2) ? 1 : 0;
		if (pi.at < 188) { u.start = pi.at; u.len = (uint16_t)(188 - pi.at); }
	}
	return u;
}
