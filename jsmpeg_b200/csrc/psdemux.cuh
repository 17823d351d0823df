// psdemux.cuh -- per-item, per-candidate and per-request arithmetic of the MPEG program stream demuxer
// (psdemux.cu), kept apart so that the host compiler can build it too (tests/emu/ps_item_check.cpp checks
// the item rules against the Python model, tools/mini_ps.py; tests/emu/ps_many_check.cpp runs the whole
// many-request pass with the step functions below).
//
// A program stream (ISO 11172-1 system stream, ISO 13818-1 program stream) is a chain of items with
// no gaps between them; an item starting at `p` is, by the bytes there:
//   00 00 01 BA, next byte 0010xxxx   ISO 11172-1 pack header          12 bytes
//   00 00 01 BA, next byte 01xxxxxx   ISO 13818-1 pack header          14 + (byte 13 & 7)
//   00 00 01 B9                       end code                          4
//   00 00 01 BB..FF                   system header, PSM, PES packet    6 + packet_length (bytes 4-5)
// Anything else where an item should start is a break in the chain (lost sync).
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

enum : int {
	PS_ITEM = 0,       // a whole item: len bytes starting at p
	PS_NEED_MORE = 1,  // could be an item, but the bytes that decide it (or its body) are behind the buffer end
	PS_BAD = 2,        // no item starts here
};

struct PsItem {
	int kind;
	uint32_t len;  // PS_ITEM: the item's length
};

// What starts at byte p of buf[0 .. n)?
__host__ __device__ inline PsItem ps_item_at(const uint8_t *buf, uint32_t n, uint32_t p) {
	const uint32_t have = n - p;
	const uint8_t prefix[3] = {0, 0, 1};
	for (uint32_t k = 0; k < 3; k++) {
		if (k >= have) return PsItem{PS_NEED_MORE, 0};
		if (buf[p + k] != prefix[k]) return PsItem{PS_BAD, 0};
	}
	if (have < 4) return PsItem{PS_NEED_MORE, 0};
	const uint32_t code = buf[p + 3];
	uint32_t len;
	if (code == 0xBA) {
		if (have < 5) return PsItem{PS_NEED_MORE, 0};
		const uint32_t b4 = buf[p + 4];
		if ((b4 >> 4) == 2) len = 12;
		else if ((b4 >> 6) == 1) {
			if (have < 14) return PsItem{PS_NEED_MORE, 0};
			len = 14 + (buf[p + 13] & 7u);
		} else return PsItem{PS_BAD, 0};
	} else if (code == 0xB9) {
		len = 4;
	} else if (code > 0xB9) {
		if (have < 6) return PsItem{PS_NEED_MORE, 0};
		len = 6 + ((uint32_t)buf[p + 4] << 8 | buf[p + 5]);
	} else {
		return PsItem{PS_BAD, 0};
	}
	if (len > have) return PsItem{PS_NEED_MORE, 0};
	return PsItem{PS_ITEM, len};
}

// 00 00 01 BA and a next byte of either form: where parsing (re)starts when out of sync
__host__ __device__ inline bool ps_is_pack(const uint8_t *buf, uint32_t n, uint32_t p) {
	if (n - p < 5 || buf[p] != 0 || buf[p + 1] != 0 || buf[p + 2] != 1 || buf[p + 3] != 0xBA) return false;
	const uint32_t b4 = buf[p + 4];
	return (b4 >> 4) == 2 || (b4 >> 6) == 1;
}

// 33-bit PTS of the 5 bytes at q (ISO 11172-1 2.4.4.2 / ISO 13818-1 2.4.3.7)
__host__ __device__ inline uint64_t ps_read_pts(const uint8_t *q) {
	return ((uint64_t)((q[0] >> 1) & 7u) << 30) | ((uint64_t)(((uint32_t)q[1] << 7) | (q[2] >> 1)) << 15) |
	       (uint64_t)(((uint32_t)q[3] << 7) | (q[4] >> 1));
}

struct PsPayload {
	uint32_t start;  // offset of the first payload byte inside the packet
	uint32_t len;    // payload bytes (0: none, or a header that runs past the packet end)
	int has_pts;
	uint64_t pts;
};

// Payload of the PES packet pkt[0 .. len) (len = 6 + packet_length, the whole packet is readable).
__host__ __device__ inline PsPayload ps_payload(const uint8_t *pkt, uint32_t len) {
	PsPayload r{len, 0, 0, 0};
	uint32_t i = 6;
	int pts_at = -1;
	if (i < len && (pkt[i] >> 6) == 2) {  // ISO 13818-1 PES header
		if (len < 9) return r;
		if (pkt[7] & 0x80) pts_at = 9;
		i = 9 + pkt[8];
		if (pts_at >= 0 && 14 > len) return r;
	} else {  // ISO 11172-1 packet header
		while (i < len && pkt[i] == 0xFF) i++;  // stuffing
		if (i >= len) return r;
		if ((pkt[i] >> 6) == 1) {  // STD buffer scale and size
			i += 2;
			if (i >= len) return r;
		}
		const uint32_t c = pkt[i] >> 4;
		if (c == 2) { pts_at = (int)i; i += 5; }
		else if (c == 3) { pts_at = (int)i; i += 10; }
		else i += 1;  // 0000 1111: neither PTS nor DTS
	}
	if (i > len) return r;
	r.start = i;
	r.len = len - i;
	if (pts_at >= 0) { r.has_pts = 1; r.pts = ps_read_pts(pkt + pts_at); }
	return r;
}

// ---- the many-request pass --------------------------------------------------------------------------
// One call demultiplexes many REQUESTS (a stream's left-over bytes followed by its new ones), each at its own
// 16-byte aligned offset of one staging buffer.  A CANDIDATE is a 00 00 01 whose three bytes lie inside one
// request and whose code is >= B9 (or behind the request's end); the candidates of all requests are sorted by
// staging position, so those of request r are the run [c0, c1) of the list.  Positions handed to the
// functions below are relative to the request's first byte unless they say otherwise, and `n` is the
// request's length: the request's end is the buffer end for every item rule.

constexpr uint32_t PS_NONE = 0xffffffffu;
enum : uint32_t {  // what the chain reaches next
	PS_T_LINK = 0,        // a candidate (PsStep::next)
	PS_T_END = 1,         // exactly the request's end
	PS_T_INCOMPLETE = 2,  // an item that needs bytes of the stream's next write, at PsStep::stop
	PS_T_NOHEAD = 3,      // no valid pack header at or after PsStep::stop: out of sync
};

struct PsReq {  // one request of a call, the host fills it
	uint32_t base;     // first byte in the staging buffer (a multiple of 16)
	uint32_t n;        // bytes: the stream's left-over bytes, then the new ones
	int stream_id;     // the PES stream id that feeds the stream
	uint32_t in_sync;  // does byte 0 continue the stream's item chain?
	uint8_t *dst;      // where its ES bytes go (the stream's ES mirror at es_base); set once the totals are known
	uint32_t es_base;  // the stream's ES length before this write
	uint32_t pad;
};

struct PsReqOut {  // per request, the device fills it
	uint32_t count;      // candidates
	uint32_t c0;         // its first candidate in the call's sorted list
	uint32_t head;       // the candidate its chain starts at (PS_NONE: none)
	uint32_t kind;       // the chain's terminal (PS_T_END, PS_T_INCOMPLETE, PS_T_NOHEAD) ...
	uint32_t stop;       // ... and where it stopped
	uint32_t consumed;   // bytes the demuxer is done with (the rest stays for the stream's next write)
	uint32_t in_sync;    // the stream's state after it
	uint32_t total;      // ES bytes
	uint32_t pes;        // PES table entries
	uint32_t pes_first;  // index of its first entry in the call's list
};

struct PsStep {
	uint32_t next;  // PS_T_LINK: the candidate (a global index)
	uint32_t kind;
	uint32_t stop;  // a terminal: where the chain stopped
};

// The candidates of one request: pos[c0 .. c1) are their staging positions (the request starts at `base`);
// next_pack_rev[m - 1 - i] = the first candidate at or after i that is a valid pack header (a suffix minimum
// over the whole list, PS_NONE if none).
struct PsCands {
	const uint32_t *pos;
	const uint32_t *next_pack_rev;
	uint32_t m, c0, c1, base;
};

// Is there a candidate at p?  (p + 2 < n: all three bytes of the prefix inside the request.)
__host__ __device__ inline bool ps_keep(const uint8_t *buf, uint32_t n, uint32_t p) {
	return p + 2 < n && buf[p] == 0 && buf[p + 1] == 0 && buf[p + 2] == 1 && (p + 3 >= n || buf[p + 3] >= 0xB9);
}

// first index in [lo, hi) with pos[index] >= want (hi if none)
__host__ __device__ inline uint32_t ps_lower(const uint32_t *pos, uint32_t lo, uint32_t hi, uint32_t want) {
	while (lo < hi) {
		const uint32_t mid = (lo + hi) >> 1;
		if (pos[mid] < want) lo = mid + 1; else hi = mid;
	}
	return lo;
}

// Out of sync from byte `from` on: the chain resumes at the request's first valid pack header at or after it
// (mini_ps.find_pack), or stops there.
__host__ __device__ inline PsStep ps_resync(const PsCands &c, uint32_t from) {
	const uint32_t k = ps_lower(c.pos, c.c0, c.c1, c.base + from);
	const uint32_t j = k < c.c1 ? c.next_pack_rev[c.m - 1 - k] : PS_NONE;
	if (j < c.c1) return PsStep{j, PS_T_LINK, 0};
	return PsStep{PS_NONE, PS_T_NOHEAD, from};
}

// What follows when the chain reaches byte t: the candidate there, the end, an item cut by the end -- or, where
// no item starts (a break), the next valid pack header after t.
__host__ __device__ inline PsStep ps_follow(const uint8_t *buf, uint32_t n, const PsCands &c, uint32_t t) {
	if (t == n) return PsStep{PS_NONE, PS_T_END, n};
	const uint32_t j = ps_lower(c.pos, c.c0, c.c1, c.base + t);
	if (j < c.c1 && c.pos[j] == c.base + t) return PsStep{j, PS_T_LINK, 0};
	// no candidate: only the head of a start-code prefix cut by the request's end can still become an item
	if (ps_item_at(buf, n, t).kind == PS_NEED_MORE) return PsStep{PS_NONE, PS_T_INCOMPLETE, t};
	return ps_resync(c, t + 1);
}

// Successor of candidate i (global index), always a later candidate of the same request -- or a terminal.
__host__ __device__ inline PsStep ps_link(const uint8_t *buf, uint32_t n, const PsCands &c, uint32_t i) {
	const uint32_t p = c.pos[i] - c.base;
	const PsItem it = ps_item_at(buf, n, p);
	if (it.kind == PS_NEED_MORE) return PsStep{PS_NONE, PS_T_INCOMPLETE, p};
	if (it.kind == PS_BAD) return ps_resync(c, p + 1);
	return ps_follow(buf, n, c, p + it.len);
}

// Where the request's chain starts: at byte 0 if it continues the stream's chain, else at its first valid
// pack header.  A terminal if it has no head.
__host__ __device__ inline PsStep ps_head(const uint8_t *buf, uint32_t n, const PsCands &c, bool in_sync) {
	return in_sync ? ps_follow(buf, n, c, 0) : ps_resync(c, 0);
}

// The request's outcome from its chain's terminal: bytes consumed and the stream's in-sync state after it
__host__ __device__ inline void ps_finish(uint32_t kind, uint32_t stop, uint32_t n, uint32_t *consumed, uint32_t *in_sync) {
	if (kind == PS_T_END) { *consumed = n; *in_sync = 1; }
	else if (kind == PS_T_INCOMPLETE) { *consumed = stop; *in_sync = 1; }
	else {  // no valid pack header at or after stop: keep what could still begin one
		const uint32_t tail = n >= 4 ? n - 4 : 0;
		*consumed = stop > tail ? stop : tail;
		*in_sync = 0;
	}
}

// The payload of the candidate at p if the chain reaches it and it is a PES packet of `stream_id`: returns the
// place key, payload length << 32 | 1 if it gives a PES table entry (a PTS and a non-empty payload); *start =
// its first payload byte, *pts its PTS.
__host__ __device__ inline uint64_t ps_place_key(const uint8_t *buf, uint32_t n, uint32_t p, int stream_id, uint32_t *start,
                                                 uint64_t *pts) {
	*start = 0;
	*pts = 0;
	if (p + 3 >= n || buf[p + 3] != (uint32_t)stream_id) return 0;
	const PsItem it = ps_item_at(buf, n, p);
	if (it.kind != PS_ITEM) return 0;
	const PsPayload pl = ps_payload(buf + p, it.len);
	*start = p + pl.start;
	*pts = pl.pts;
	return (uint64_t)pl.len << 32 | (uint64_t)(pl.has_pts && pl.len ? 1 : 0);
}
