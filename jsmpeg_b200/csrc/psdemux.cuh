// psdemux.cuh -- per-item arithmetic of the MPEG program stream demuxer (psdemux.cu), kept apart so
// that the host compiler can build it too (tests/emu/ps_item_check.cpp checks it against the Python
// model, tools/mini_ps.py).
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
