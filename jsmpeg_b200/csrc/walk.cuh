// walk.cuh -- stage 1 device code: the walk of one picture's bitstream (1a) and the per-block expansion
// (1b) (sm_90a).
//
// Included by parse.cu (the kernels, the tables' upload and the launcher live there).  The same text
// compiles for the host when JSMPEG_WALK_EMU is defined and the including file supplies the few CUDA
// intrinsics it uses (tests/emu/walk_emu.cpp runs a "warp" as 32 coroutines): that is how the
// lane-parallel walk is checked against the serial one, and both plus stage 1b against the oracle, on
// machines without a GPU.  Nothing in the product library is built that way.
//
// (Three candidates were measured and deleted: staged relative records + fix-up instead of the second
// semantic pass (a faster walk, the same stage 1); the storing pass writing the block records itself, no
// stage 1b (slower stage 1); 16-byte register-cached refills (slower walk).)
#pragma once
#include "common.cuh"

#ifndef VLC_TABLE_QUALIFIER
#define VLC_TABLE_QUALIFIER alignas(16) static __device__ const
#endif
#include "vlc_tables.h"

namespace {

#ifndef JSMPEG_MS_BITS
#define JSMPEG_MS_BITS 13
#endif
#ifndef JSMPEG_WALK_THREADS
#define JSMPEG_WALK_THREADS 256
#endif
constexpr int WALK_THREADS = JSMPEG_WALK_THREADS;  // walk kernel: the pictures of a CTA share one multi-symbol table
constexpr int MS_BITS = JSMPEG_MS_BITS;            // multi-symbol table is indexed by the next MS_BITS bits (2 << MS_BITS bytes)
constexpr uint32_t OFF_MS = 4096;      // uint16[1 << MS_BITS], after the per-symbol tables
constexpr uint32_t OFF_MS_FIRST = OFF_MS + (2u << MS_BITS);  // uint16[1 << (MS_BITS - 1)]: dct_coeff_first variant, prefixes with a leading 1 (lane-parallel walk only)
constexpr uint32_t MS_TABLE_ENTRIES = (1u << MS_BITS) + (1u << (MS_BITS - 1));
constexpr uint32_t WALK_SMEM_SERIAL = OFF_MS + (2u << MS_BITS), WALK_SMEM_LANES_TABLES = OFF_MS + 2u * MS_TABLE_ENTRIES;
// lane-parallel walk: after the tables, one 64-byte bitstream ring per lane (BitReaderT<true>)
constexpr uint32_t OFF_RING = (WALK_SMEM_LANES_TABLES + 15u) & ~15u, RING_BYTES = 64;
constexpr uint32_t WALK_SMEM_LANES = OFF_RING + (uint32_t)JSMPEG_WALK_THREADS * RING_BYTES;

// shared-memory layout (byte offsets from the dynamic shared base)
constexpr uint32_t OFF_DCT = 0;                                        // uint16[384]
constexpr uint32_t OFF_MBA = OFF_DCT + (VLC_DCT_MAX_Z + 1) * 64;       // uint16[256]
constexpr uint32_t OFF_CBP = OFF_MBA + (VLC_MBA_MAX_Z + 1) * 64;       // uint16[256]
constexpr uint32_t OFF_MOTION = OFF_CBP + (VLC_CBP_MAX_Z + 1) * 64;    // uint16[224]
constexpr uint32_t OFF_DC_LUMA = OFF_MOTION + (VLC_MOTION_MAX_Z + 1) * 64;  // uint16[128]
constexpr uint32_t OFF_DC_CHROMA = OFF_DC_LUMA + 256;                  // uint16[256]
constexpr uint32_t OFF_TYPE_I = OFF_DC_CHROMA + 512;                   // uint16[4]
constexpr uint32_t OFF_TYPE_P = OFF_TYPE_I + 8;                        // uint16[64]
static_assert(OFF_TYPE_P + 128 <= OFF_MS, "the per-symbol tables end before the multi-symbol table");
// stage 1b (its own kernel, its own shared memory): the DCT table with values, the two quantiser tables
// in zig-zag order (SeqParams::xq), and per warp a staging area: the lanes' compact rows, or their 64 x int16 tiles
constexpr uint32_t EXP_OFF_DCT = 0;                                     // uint32[384]: VLC_DCT_EXPAND (clz-indexed)
constexpr uint32_t EXP_OFF_TOP8 = EXP_OFF_DCT + (VLC_DCT_MAX_Z + 1) * 128;  // uint32[256]: VLC_DCT_EXPAND_TOP8 (next 8 bits)
constexpr uint32_t EXP_OFF_XQ = EXP_OFF_TOP8 + 1024;                    // uint16[2][64]
constexpr uint32_t EXP_OFF_TILES = (EXP_OFF_XQ + 256 + 127) & ~127u;
constexpr uint32_t EXP_TABLE_BYTES = EXP_OFF_XQ;                        // the two code tables, contiguous

#ifndef JSMPEG_WALK_EMU
__device__ __forceinline__ uint32_t lds_u16(uint32_t addr) {
	uint16_t v;
	asm("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
	return v;
}
__device__ __forceinline__ uint32_t lds_u8(uint32_t addr) {
	uint32_t v;
	asm("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
	return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
	uint32_t v;
	asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
	return v;
}
__device__ __forceinline__ void sts_s16(uint32_t addr, int v) {
	asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"((uint16_t)v) : "memory");
}
__device__ __forceinline__ void sts_u64(uint32_t addr, uint64_t v) {
	asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(addr), "r"((uint32_t)v), "r"((uint32_t)(v >> 32)) : "memory");
}
#else
// host emulation (tests only): `emu_smem` stands in for the CTA's shared memory, addresses are offsets into it
constexpr uint32_t EMU_EXPAND_BASE = (WALK_SMEM_LANES + 127u) & ~127u;  // a second "CTA": stage 1b's own tables and tile
static uint8_t emu_smem[EMU_EXPAND_BASE + 8192];
static inline uint32_t lds_u16(uint32_t addr) { uint16_t v; memcpy(&v, emu_smem + addr, 2); return v; }
static inline uint32_t lds_u8(uint32_t addr) { return emu_smem[addr]; }
static inline uint32_t lds_u32(uint32_t addr) { uint32_t v; memcpy(&v, emu_smem + addr, 4); return v; }
static inline void sts_s16(uint32_t addr, int v) { const int16_t x = (int16_t)v; memcpy(emu_smem + addr, &x, 2); }
static inline void sts_u64(uint32_t addr, uint64_t v) { memcpy(emu_smem + addr, &v, 8); }
#endif
// MSB-first bit window over a byte span (src/buffer.js:152-187); one copy per thread.
//
// RING (the lane-parallel walk): the bytes reach the lane through its own 64-byte ring in shared memory,
// filled by asynchronous 16-byte global -> shared copies (cp.async, SASS LDGSTS) issued three chunks
// (48 bytes, some forty look-ups) ahead of the read position.  Refilling with one 4-byte global load per
// lane, a single word ahead, left the load's latency exposed: with 1024 lanes per SM each on its own stream
// L1 thrashes.  A 16-byte register cache per lane (loads still on demand) was slower too; what was missing
// was distance, not width.
// PADDED: the bytes behind the data are known to be zero (the product's ES mirror: ES_PAD zeroed bytes)
// and no reader runs further than a few words past the end, so neither the test against len nor the mask
// of the last word is needed.  (Host emulation: exact-size buffers under AddressSanitizer, so never.)
#ifdef JSMPEG_WALK_EMU
constexpr bool ES_IS_PADDED = false;
#else
constexpr bool ES_IS_PADDED = true;
#endif
template <bool RING, bool PADDED = false>
struct BitReaderT {
	const uint32_t *words;  // 16-byte aligned base of the ES mirror (cudaMalloc), ES_PAD readable bytes past len
	const uint8_t *bytes;
	uint32_t len;    // valid bytes; everything past it reads as zero (JS typed-array semantics)
	uint32_t wpos;   // index of the word held in `nextw` (the next one to enter the window)
	uint32_t nextw;  // prefetched
	uint64_t win;    // left-aligned window
	int nbits;       // valid bits in win, >= 32 between calls
	uint32_t ring;   // RING: shared-window address of this lane's ring (4 chunks of 16 bytes, chunk q in slot q & 3).
	                 // Invariant between calls: the chunks up to (chunk of word wpos) + 3 have been requested.

	__device__ __forceinline__ uint32_t finish_word(uint32_t raw, uint32_t byte) const {
		uint32_t v = __byte_perm(raw, 0, 0x0123);  // first byte -> MSB
		const uint32_t left = len - byte;
		if (left < 4u) v &= 0xffffffffu << (8u * (4u - left));
		return v;
	}
	// any word, straight from global memory (random access: the slice-end search)
	__device__ __forceinline__ uint32_t load_word_direct(uint32_t w) const {
		const uint32_t byte = w * 4u;
		if (byte >= len) return 0u;
		return finish_word(__ldg(words + w), byte);
	}
#if !defined(JSMPEG_WALK_EMU)
	// one commit group per chunk.  No branch: a chunk past the data is fetched from the zeroed pad behind
	// it (clamped to the pad's first chunk, which is all zero and inside the allocation)
	__device__ __forceinline__ void ring_request(uint32_t q) {
		const uint32_t off = min(q << 4, (len + 15u) & ~15u);
		asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(ring + ((q & 3u) << 4)), "l"(bytes + off) : "memory");
		asm volatile("cp.async.commit_group;" ::: "memory");
	}
	__device__ __forceinline__ uint32_t ring_word(uint32_t w) const {
		uint32_t v;
		asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(ring + ((w & 15u) << 2)) : "memory");
		return v;
	}
#endif
	// the next word of a sequential read (w only grows between seeks)
	// (Rejected for the global-load refill: a branch-free variant relying on the zero pad after the data, and a
	// software prefetch 256 B ahead at every refill; both were slower.)
	__device__ __forceinline__ uint32_t load_word(uint32_t w) {
#if !defined(JSMPEG_WALK_EMU)
		if (RING) {
			// No test against len and no tail mask here: the mirror is followed by zeroed bytes (ES_PAD), a chunk
			// past them is fetched from the pad too (ring_request), and no walk runs more than a macroblock
			// header past the end of the data before it stops.
			if ((w & 3u) == 0u) {  // first word of chunk q: chunk q - 1 is consumed, its slot takes chunk q + 3
				ring_request((w >> 2) + 3u);
				asm volatile("cp.async.wait_group 3;" ::: "memory");  // everything but the three newest chunks has landed
			}
			return __byte_perm(ring_word(w), 0, 0x0123);  // first byte -> MSB
		}
#endif
		if (PADDED) return __byte_perm(__ldg(words + w), 0, 0x0123);
		const uint32_t byte = w * 4u;
		if (byte >= len) return 0u;
		return finish_word(__ldg(words + w), byte);
	}
	__device__ __forceinline__ void seek_byte(uint32_t byte_pos) {
		const uint32_t w = byte_pos >> 2;
#if !defined(JSMPEG_WALK_EMU)
		if (RING) {
			asm volatile("cp.async.wait_all;" ::: "memory");  // nothing requested for the old position may still be landing
			const uint32_t q0 = w >> 2;
			ring_request(q0); ring_request(q0 + 1u); ring_request(q0 + 2u); ring_request(q0 + 3u);
			asm volatile("cp.async.wait_all;" ::: "memory");
			auto raw = [&](uint32_t x) { return __byte_perm(ring_word(x), 0, 0x0123); };
			win = ((uint64_t)raw(w) << 32) | raw(w + 1);
			wpos = w + 2;
			nextw = raw(wpos);
			// w .. w + 2 lie in chunks q0, q0 + 1.  If they reach into q0 + 1, chunk q0 is consumed and that
			// chunk's turn to extend the ring (load_word, first word of a chunk) is taken here -- after the
			// reads, the new chunk goes into q0's slot -- so that the invariant holds
			if (((w + 2u) >> 2) != q0) ring_request(q0 + 4u);
		} else
#endif
		{
			win = ((uint64_t)load_word(w) << 32) | load_word(w + 1);
			wpos = w + 2;
			nextw = load_word(wpos);
		}
		nbits = 64;
		const int drop = (int)(byte_pos & 3u) * 8;
		if (drop) consume(drop);
	}
	__device__ __forceinline__ void seek_bit(uint32_t bit_pos) {
		seek_byte(bit_pos >> 3);
		if (bit_pos & 7u) consume((int)(bit_pos & 7u));
	}
	__device__ __forceinline__ uint32_t peek32() const { return (uint32_t)(win >> 32); }
	__device__ __forceinline__ void consume(int n) {  // 0 <= n <= 32
		win <<= n;
		nbits -= n;
		if (nbits < 32) {
			win |= (uint64_t)nextw << (32 - nbits);
			nbits += 32;
			wpos++;
			nextw = load_word(wpos);
		}
	}
	__device__ __forceinline__ uint32_t read(int n) {  // 1 <= n <= 32
		const uint32_t v = peek32() >> (32 - n);
		consume(n);
		return v;
	}
	__device__ __forceinline__ uint32_t bitpos() const { return wpos * 32u - (uint32_t)nbits; }

	// src/buffer.js:141-150 nextBytesAreStartCode
	__device__ __forceinline__ bool next_bytes_are_start_code() const {
		const uint32_t bp = bitpos();
		const uint32_t i = (bp + 7u) >> 3;
		if (i >= len) return true;
		const int skip = (int)((8u - (bp & 7u)) & 7u);
		// bytes past `len` are zero in the window, so a code straddling the end cannot match
		return (uint32_t)((win << skip) >> 40) == 0x000001u && i + 2u < len;
	}
	// src/buffer.js:115-128 findNextStartCode.  Returns the code (reader left just after it) or -1
	// (reader parked at the end of the data).  A start code needs its 4 bytes inside the buffer.
	__device__ int find_next_start_code() {
		uint32_t i = (bitpos() + 7u) >> 3;
		for (; i + 3u < len; i++) {
			if (bytes[i + 2] > 1) { i += 2; continue; }  // 00 00 01 cannot end at i+2, i+3 or i+4
			if (bytes[i] == 0 && bytes[i + 1] == 0 && bytes[i + 2] == 1) {
				const int code = bytes[i + 3];
				seek_byte(i + 4u);
				return code;
			}
		}
		seek_byte(len);
		return -1;
	}
};
using BitReader = BitReaderT<false>;  // stage 1b and the serial-walk kernel: plain global loads


struct PictureState {
	int picture_type, full_pel, r_size, f;
	int qscale, mb_addr;
	bool slice_begin;
	int mv_h, mv_v, mv_h_prev, mv_v_prev;
	int dc_y, dc_b4, dc_b5;  // block 4 / block 5 predictors (the reference's "Cr"/"Cb", mpeg1.js:717)
	int n_present, n_coded, error;
	int n_fixup;  // slices of the lane-parallel walk that needed no second pass (staged records + fix-up)
	// lane-parallel walk only: which parts of a RELATIVE state no longer depend on the state the lane
	// started from, and whether a case outside the lane-parallel walk's domain was met
	bool qs_set, dc_abs, mv_abs, anomaly;
};

#ifndef JSMPEG_WALK_EMU
// The shared-window address of the dynamic shared memory, made opaque so that the compiler keeps
// it in a register instead of re-deriving it (S2R + LEA) at every table access.
__device__ __forceinline__ uint32_t smem_base(const void *p) {
	uint32_t a = (uint32_t)__cvta_generic_to_shared(p), r;
	asm volatile("mov.u32 %0, %1;" : "=r"(r) : "r"(a));
	return r;
}
#else
static inline uint32_t smem_base(const void *) { return 0; }
#endif

__device__ __forceinline__ uint32_t clz_lut(uint32_t table_addr, uint32_t w, int max_z) {
	const int z = __clz((int)w);
	if (z > max_z) return 0;
	return lds_u16(table_addr + (((uint32_t)z << 5) | ((w << (z + 1)) >> 27)) * 2u);
}

// ==================================================================================================
// 1a: the serial walk

// walk-table entry derived from the DCT table: bits 0..4 = bits to consume (code + sign),
// bits 5..10 = run + 1, bits 11..12 = 1 end_of_block / 2 escape; 0 = invalid code.
__device__ __forceinline__ uint16_t walk_entry(uint16_t e) {
	const int len = e & 31, run = (e >> 5) & 31, level = e >> 10;
	if (len == 0) return 0;
	if (level == 0) return run ? (uint16_t)(2 | (1 << 11)) : (uint16_t)(6 | (2 << 11));
	return (uint16_t)((len + 1) | ((run + 1) << 5));
}

// One coded block (bitstream side of src/mpeg1.js:698-811): intra DC with its predictor, then only
// code lengths.  Leaves {bit offset of the first coefficient code, intra dc clamped as records.h says} in the block's slot.
// head: DC size VLC + differential + predictor (mpeg1.js:705-751), the parked pair, dct_coeff_first
// RAW_DC (staging): the pair holds the DC predictor's value itself (possibly relative), not yet clamped
template <bool DEFER, bool RAW_DC = false, class BR>
__device__ __forceinline__ bool walk_block_head(BR &br, uint32_t sbase, PictureState &ps, bool intra, int block,
                                                uint2 *__restrict__ park, bool store, int &n, bool &defer_first) {
	n = 0;
	int dc_rec = 0, dc_raw = 0;
	if (intra) {
		const uint32_t w = br.peek32();
		const uint32_t e = block < 4 ? lds_u16(sbase + OFF_DC_LUMA + (w >> 25) * 2u)
		                             : lds_u16(sbase + OFF_DC_CHROMA + (w >> 24) * 2u);
		const int len = e & 31, size = e >> 5;
		if (len == 0) return false;
		// (The pointer sends the three predictors to local memory.  Selects instead were slower: the state then
		// competes for the 64 registers and spills far more.)
		int *pred = block < 4 ? &ps.dc_y : (block == 4 ? &ps.dc_b4 : &ps.dc_b5);
		int dc = *pred;
		if (DEFER) {  // code and differential (at most 8 + 8 bits) sit in the same 32-bit peek: the window moves once
			if (size > 0) {
				const int diff = (int)((w << len) >> (32 - size));
				dc += (diff & (1 << (size - 1))) ? diff : (int)((0xffffffffu << size) | (uint32_t)(diff + 1));
			}
			br.consume(len + size);
		} else {
			br.consume(len);
			if (size > 0) {
				const int diff = (int)br.read(size);
				dc += (diff & (1 << (size - 1))) ? diff : (int)((0xffffffffu << size) | (uint32_t)(diff + 1));
			}
		}
		*pred = dc;
		dc_raw = dc;
		dc_rec = max(-INTRA_DC_BOUND, min(255 + INTRA_DC_BOUND, dc));  // x 256 = dc << 8 in stage 2 (mpeg1.js:747)
		n = 1;
	}
	if (store) *park = make_uint2(br.bitpos(), RAW_DC ? (uint32_t)dc_raw : (uint32_t)dc_rec & 0xffffu);
	if (DEFER) {
		defer_first = !intra;  // the caller's first look-up resolves dct_coeff_first (ac_step)
	} else if (!intra && (br.peek32() >> 31)) {  // dct_coeff_first: a leading '1' is (0, +-1), never end_of_block
		br.consume(2);
		n = 1;
	}
	return true;
}
__device__ __forceinline__ void walk_block_tail(PictureState &ps, int n, bool &dc_only) {
	if (n > 64) ps.error = PARSE_ERR_COEF_INDEX;  // some run pushed the index past 63 (stores dropped, like JS)
	dc_only = (n == 1);  // mpeg1.js:838, 850
	ps.n_coded++;
}
template <class BR>
__device__ __forceinline__ bool walk_block(BR &br, uint32_t sbase, PictureState &ps, bool intra, int block,
                                           uint2 *__restrict__ park, bool store, bool &dc_only) {
	int n;
	bool unused;
	if (!walk_block_head<false>(br, sbase, ps, intra, block, park, store, n, unused)) return false;
	for (;;) {
		const uint32_t w = br.peek32();
		// (Resolving '10' / '11s' arithmetically before the look-up was SLOWER: it defeats the combining of
		// several codes per look-up.)
		// as many complete codes as fit in the next 13 bits, in one look-up
		const uint32_t m = lds_u16(sbase + OFF_MS + (w >> (32 - MS_BITS)) * 2u);
		if (m & 15u) {
			n += (int)((m >> 4) & 63u);
			br.consume((int)(m & 15u));
			if (m & 0x400u) break;  // the last code consumed was end_of_block
			continue;
		}
		// long code or escape: one symbol through the clz-indexed table
		const int z = __clz((int)w);
		if (z > VLC_DCT_MAX_Z) return false;
		const uint32_t e = lds_u16(sbase + OFF_DCT + (((uint32_t)z << 5) | ((w << (z + 1)) >> 27)) * 2u);
		if (e >> 11) {
			// escape (mpeg1.js:767-780): 6-bit code, 6-bit run, 8 (+8) bit level.  (end_of_block is
			// two bits and always resolved by the multi-symbol table.)
			n += (int)((w >> 20) & 63u) + 1;
			br.consume((w & 0x0007f000u) ? 20 : 28);  // level byte 0 or 128 -> a second byte follows
			continue;
		}
		if (e == 0) return false;  // hole in the code space
		n += (int)(e >> 5);
		br.consume((int)(e & 31u));
	}
	walk_block_tail(ps, n, dc_only);
	return true;
}
// The same loop, one look-up per call (the lane-parallel walk votes between look-ups so that the lanes
// stay in step): 0 = go on, 1 = end_of_block consumed, 2 = invalid code.  `combine` = several codes
// may be taken at once; `first` = the block's first coefficient of a non-intra block, where a leading
// '1' is (0, +-1) and never end_of_block (mpeg1.js:757-760): a second table covers that case so that
// a block start costs no extra trip.  The escape is resolved before the clz table: with 32 chains in
// lock-step every path some lane needs is issued for all, so the rare path must stay rare.
template <class BR>
__device__ __forceinline__ int ac_step(BR &br, uint32_t sbase, int &n, bool combine, bool first) {
	// every path only decides (bits, run sum, end_of_block); the window moves ONCE, after they rejoin
	const uint32_t w = br.peek32();
	const bool lead = first && (w >> 31);
	uint32_t m = lead ? (2u | (1u << 4)) : 0u;  // not combining: the leading '1s' alone, or the clz table
	if (combine)
		m = lds_u16(sbase + (lead ? OFF_MS_FIRST + ((w >> (32 - MS_BITS)) & ((1u << (MS_BITS - 1)) - 1u)) * 2u
		                          : OFF_MS + (w >> (32 - MS_BITS)) * 2u));
	int len = (int)(m & 15u), dn = (int)((m >> 4) & 63u), ret = (int)((m >> 10) & 1u);
	if (len == 0) {
		if ((w >> 26) == 1u) {  // escape (mpeg1.js:767-780): 6-bit run, 8 (+8) bit level
			dn = (int)((w >> 20) & 63u) + 1;
			len = (w & 0x0007f000u) ? 20 : 28;
		} else {  // a code longer than the window, or end_of_block when not combining
			const int z = __clz((int)w);
			if (z > VLC_DCT_MAX_Z) return 2;
			const uint32_t e = lds_u16(sbase + OFF_DCT + (((uint32_t)z << 5) | ((w << (z + 1)) >> 27)) * 2u);
			if (e == 0 || (e >> 11) == 2u) return 2;  // (the escape was taken above)
			ret = (int)(e >> 11);            // 1 = end_of_block (two bits)
			len = (int)(e & 31u);
			dn = ret ? 0 : (int)(e >> 5);
		}
	}
	n += dn;
	br.consume(len);
	return ret;
}


// mpeg1.js:395-457, one component
template <class BR>
__device__ __forceinline__ bool parse_motion(BR &br, uint32_t sbase, const PictureState &ps, int &prev, int &mv) {
	const uint32_t e = clz_lut(sbase + OFF_MOTION, br.peek32(), VLC_MOTION_MAX_Z);
	const int len = e & 31;
	if (len == 0) return false;
	br.consume(len);
	const int code = (int)(e >> 5) - 16;
	int d = code;
	if (code != 0 && ps.f != 1) {
		const int r = (int)br.read(ps.r_size);
		d = ((abs(code) - 1) << ps.r_size) + r + 1;
		if (code < 0) d = -d;
	}
	prev += d;
	if (prev > (ps.f << 4) - 1) prev -= ps.f << 5;
	else if (prev < -(ps.f << 4)) prev += ps.f << 5;
	mv = ps.full_pel ? prev * 2 : prev;
	return true;
}

template <class BR>
__device__ __forceinline__ int read_mba(BR &br, uint32_t sbase) {
	const uint32_t e = clz_lut(sbase + OFF_MBA, br.peek32(), VLC_MBA_MAX_Z);
	const int len = e & 31;
	if (len == 0) return -1;
	br.consume(len);
	return (int)(e >> 5);
}

__device__ __forceinline__ uint4 pack_record(int mv_h, int mv_v, int flags, int cbp, int dc_only, int qscale, uint32_t bit_pos) {
	uint4 r;
	r.x = ((uint32_t)mv_h & 0xffffu) | ((uint32_t)mv_v << 16);
	r.y = (uint32_t)flags | ((uint32_t)cbp << 8) | ((uint32_t)dc_only << 16) | ((uint32_t)qscale << 24);
	r.z = bit_pos;
	r.w = 0;
	return r;
}

// How a macroblock is walked:
//   WALK_SERIAL  the whole warp walks the same macroblock redundantly, lane 0 stores (one warp = one chain)
//   WALK_REL     one lane walks it, nothing is stored and no address is checked: the state is RELATIVE to the
//                unknown state at the lane's first macroblock (summary pass of the lane-parallel walk)
//   WALK_ABS     one lane walks it with the true state and stores; cases the lane-parallel walk leaves to
//                the serial walk set ps.anomaly
//   WALK_STAGE   WALK_REL that also leaves every macroblock as a RELATIVE record in the picture's staging
//                area; a fix-up (no bitstream access) then turns the staged records into the final ones and
//                the WALK_ABS pass is not needed
enum { WALK_SERIAL = 0, WALK_REL = 1, WALK_ABS = 2, WALK_STAGE = 3 };
#define WALK_IS_REL(MODE) ((MODE) == WALK_REL || (MODE) == WALK_STAGE)

struct MbHead {
	int mb, cbp, mv_h, mv_v, qscale;
	bool intra;
	uint32_t bit_pos;
	// WALK_STAGE only: the run of skipped macroblocks in front of this one
	int n_skip, skip_first, skip_qs;
	bool skip_qs_set;
	uint32_t skip_bit;
};

// mpeg1.js:294-384, decodeMacroblock up to the blocks.  0: the blocks of h.cbp follow; 1: nothing more
// to do for this macroblock, the slice goes on; 2: stop walking this slice.
template <int MODE, class BR>
__device__ __forceinline__ int walk_mb_header(BR &br, uint32_t sbase, PictureState &ps, const ParseTask &t, int mb_size, int lane, MbHead &h) {
	int increment = 0;
	int v = read_mba(br, sbase);
	while (v == 34) v = read_mba(br, sbase);                       // macroblock_stuffing
	while (v == 35) { increment += 33; v = read_mba(br, sbase); }  // macroblock_escape
	if (v < 0) return 2;
	increment += v;

	if (ps.slice_begin) {  // mpeg1.js:312-317
		ps.slice_begin = false;
		ps.mb_addr += increment;
	} else {
		if (MODE == WALK_SERIAL && ps.mb_addr + increment >= mb_size) return 1;  // mpeg1.js:319-322
		if (MODE == WALK_ABS && ps.mb_addr + increment >= mb_size) { ps.anomaly = true; return 2; }
		if (increment > 1) {  // mpeg1.js:323-334
			ps.dc_y = ps.dc_b4 = ps.dc_b5 = 128;
			if (WALK_IS_REL(MODE)) ps.dc_abs = true;
			if (ps.picture_type == 2) {
				ps.mv_h = ps.mv_v = ps.mv_h_prev = ps.mv_v_prev = 0;
				if (WALK_IS_REL(MODE)) ps.mv_abs = true;
			}
			// skipped macroblocks: predicted copy with the current vector (mpeg1.js:336-346)
			const int n_skip = increment - 1;
			const uint4 rec = pack_record(ps.mv_h, ps.mv_v, MBF_PRESENT | MBF_SKIPPED, 0, 0, ps.qscale, br.bitpos());
			if (MODE == WALK_SERIAL) {
				// In a broken stream these addresses may have been stored before, or be stored again later, by
				// lane 0 (a macroblock record): the order of the lanes' stores is part of the result, and
				// independent thread scheduling promises no program order between lanes without this.
				__syncwarp();
				for (int k = lane; k < n_skip; k += 32) reinterpret_cast<uint4 *>(t.hdr)[ps.mb_addr + 1 + k] = rec;
				__syncwarp();
			}
			if (MODE == WALK_ABS)
				for (int k = 0; k < n_skip; k++) reinterpret_cast<uint4 *>(t.hdr)[ps.mb_addr + 1 + k] = rec;
			if (MODE == WALK_STAGE) {
				h.n_skip = n_skip; h.skip_first = ps.mb_addr + 1; h.skip_qs = ps.qscale; h.skip_qs_set = ps.qs_set;
				h.skip_bit = br.bitpos();
			}
			ps.n_present += n_skip;
			ps.mb_addr += n_skip;
		}
		ps.mb_addr++;
	}
	const int mb = ps.mb_addr;
	h.mb = mb;
	if (!WALK_IS_REL(MODE) && (mb < 0 || mb >= mb_size)) {  // outside the picture: never write there
		if (MODE == WALK_ABS) ps.anomaly = true;
		return 2;
	}

	const uint32_t w = br.peek32();
	const uint32_t e = ps.picture_type == 1 ? lds_u16(sbase + OFF_TYPE_I + (w >> 30) * 2u)
	                                        : lds_u16(sbase + OFF_TYPE_P + (w >> 26) * 2u);
	if ((e & 31) == 0) return 2;
	br.consume(e & 31);
	const int type = e >> 5;
	const bool intra = type & 0x01;
	h.intra = intra;
	if (type & 0x10) {
		ps.qscale = (int)br.read(5);
		if (WALK_IS_REL(MODE)) ps.qs_set = true;
	}
	h.bit_pos = br.bitpos();

	if (intra) {
		ps.mv_h = ps.mv_v = ps.mv_h_prev = ps.mv_v_prev = 0;  // mpeg1.js:363-367
		if (WALK_IS_REL(MODE)) ps.mv_abs = true;
	} else {
		ps.dc_y = ps.dc_b4 = ps.dc_b5 = 128;                  // mpeg1.js:370-372
		if (WALK_IS_REL(MODE)) ps.dc_abs = true;
		if (type & 0x08) {
			if (!parse_motion(br, sbase, ps, ps.mv_h_prev, ps.mv_h)) return 2;
			if (!parse_motion(br, sbase, ps, ps.mv_v_prev, ps.mv_v)) return 2;
		} else if (ps.picture_type == 2) {
			ps.mv_h = ps.mv_v = ps.mv_h_prev = ps.mv_v_prev = 0;  // mpeg1.js:452-456
			if (WALK_IS_REL(MODE)) ps.mv_abs = true;
		}
	}

	int cbp = intra ? 0x3f : 0;
	if (type & 0x02) {
		const uint32_t ce = clz_lut(sbase + OFF_CBP, br.peek32(), VLC_CBP_MAX_Z);
		if ((ce & 31) == 0) return 2;
		br.consume(ce & 31);
		cbp = ce >> 5;
	}

	h.cbp = cbp;
	h.mv_h = ps.mv_h; h.mv_v = ps.mv_v; h.qscale = ps.qscale;
	return 0;
}

// mpeg1.js:294-392 decodeMacroblock, serial.  false = stop walking this slice.
template <class BR>
__device__ bool walk_macroblock(BR &br, uint32_t sbase, PictureState &ps, const ParseTask &t, int mb_size, int lane) {
	MbHead h;
	const int r = walk_mb_header<WALK_SERIAL>(br, sbase, ps, t, mb_size, lane, h);
	if (r) return r == 1;
	const int mb = h.mb, cbp = h.cbp;
	const bool intra = h.intra;
	uint2 *park_mb = t.park + (size_t)mb * 6;
	int done = 0, dc_mask = 0;
	bool ok = true;
#pragma unroll 1
	for (int block = 0; block < 6; block++) {
		if (cbp & (0x20 >> block)) {
			bool dc_only;
			ok = walk_block(br, sbase, ps, intra, block, park_mb + block, lane == 0, dc_only);
			if (!ok) break;
			done |= 0x20 >> block;
			if (dc_only) dc_mask |= 0x20 >> block;
		}
	}
	if (lane == 0)
		reinterpret_cast<uint4 *>(t.hdr)[mb] =
		    pack_record(h.mv_h, h.mv_v, MBF_PRESENT | (intra ? MBF_INTRA : 0), done, dc_mask, h.qscale, h.bit_pos);
	ps.n_present++;
	return ok;
}

// ==================================================================================================
// 1a, lane-parallel: 32 lanes walk 32 sub-sequences of ONE slice
//
// The serial walk spends 31 of 32 lanes re-executing lane 0's chain.  Here the bits of a slice are cut
// into up to 32 equal sub-sequences, one per lane, and the chain is recovered by self-synchronisation
// (the property of variable-length codes that a decoder started at a wrong position or in a wrong
// syntax state falls into step with the true one after a while; Klein & Wiseman 2003, and
// Weissenberger & Schmidt 2018/2021 for Huffman/JPEG on GPUs):
//
//   W  warm-up: every lane > 0 starts WARMUP_BITS before its sub-sequence in a GUESSED syntax state and
//      runs a syntax-only automaton (code lengths and the state machine of mpeg1.js:294-392/698-790,
//      no values) to the first macroblock start at or beyond the start of its sub-sequence.  By then
//      it has, almost always, merged with the true chain (chains merge within a few macroblocks).
//      Lane 0, and lanes whose warm-up would begin before the slice, start in the true state.
//   C  every lane walks the macroblocks that START in its sub-sequence with full semantics but
//      RELATIVE predictors (WALK_REL) -- a summary: address advance, last quantiser scale, DC and
//      motion predictors as "absolute after a reset" or "delta".  Where lane i stops must be exactly
//      where lane i+1 started: if that holds for every lane, every lane walked the true chain (lane 0
//      did, and each lane hands the true position to the next).  A warp scan of the summaries (an
//      associative composition) gives every lane the absolute state at its first macroblock.
//   D  every lane walks its macroblocks again with the absolute state and stores (WALK_ABS).
//
// Anything outside the clean domain -- a warm-up that did not merge, an invalid code on the true chain,
// an address outside the picture, a slice that does not end exactly at the next start code -- makes
// the warp discard the attempt and walk the whole picture with the serial code, which defines the
// behaviour there.
// (The first version followed Weissenberger & Schmidt more literally: full-length speculative pass,
// then rounds of "run on through the next sub-sequence and compare exit states" -- 4.3 passes over the
// bits instead of 2.2; see DESIGN.md.)

enum { PH_MBA = 0, PH_MBA_STUFF, PH_MBA_ESC, PH_TYPE, PH_MV_H, PH_MV_V, PH_CBP, PH_DC, PH_AC_FIRST, PH_AC, PH_END };

constexpr unsigned FULL_MASK = 0xffffffffu;
// the votes that close the lock-step loops; the host emulation counts trips and participating lanes per site
#ifdef JSMPEG_WALK_EMU
#define WK_VOTE(site, pred) emu_vote(site, pred)
#else

#define WK_VOTE(site, pred) __any_sync(FULL_MASK, pred)
#endif
enum { VOTE_SYN_MB = 0, VOTE_SYN_AC, VOTE_OWN_MB, VOTE_OWN_AC, VOTE_SITES };
constexpr uint32_t MIN_SUBSEQ_BITS = 2048;  // shorter sub-sequences are not worth a lane
#ifndef JSMPEG_WARMUP_BITS
#define JSMPEG_WARMUP_BITS 8192
#endif
constexpr uint32_t WARMUP_BITS = JSMPEG_WARMUP_BITS;  // how far before its sub-sequence a lane starts guessing
#ifndef JSMPEG_WARMUP_MBS
#define JSMPEG_WARMUP_MBS 48
#endif
constexpr uint32_t WARMUP_MBS = JSMPEG_WARMUP_MBS;    // ... or this many average macroblocks, whichever is longer

struct SliceConst {
	int picture_type, r_size, f;
	uint32_t end_byte;  // byte index of the start code prefix that ends the slice (or the end of the data)
};

// syntax state: phase | blocks still to come (mask, current block = highest bit) << 4 | macroblock type bits << 10
__device__ __forceinline__ uint32_t syn_make(int phase, uint32_t rem, uint32_t type) { return (uint32_t)phase | rem << 4 | type << 10; }
// The state a chain assumes where it knows nothing: inside the coefficients of the last block of a
// macroblock.  After the next end_of_block it tries a macroblock header; a true end_of_block is a
// true macroblock start often enough.
__device__ __forceinline__ uint32_t syn_guess(const SliceConst &sc) { return syn_make(PH_AC, 1u, sc.picture_type == 1 ? 1u : 0u); }

// Runs the syntax-only automaton from the reader's position in state `st` until the first MACROBLOCK
// START at or beyond bit `limit` (state PH_MBA) or the end of the slice (PH_END).
// An invalid code does not stop a chain: it drops one bit and guesses again (a chain that dies can
// never merge).  If it is the TRUE chain that meets an invalid code, pass C/D meet it too, with full
// semantics, and the picture goes to the serial walk.
//
// WARP-SYNCHRONOUS: all 32 lanes call it together (`live` = this lane has something to run).  The
// automaton is written in the order of the syntax, one macroblock per trip of the outer loop and one
// look-up per trip of the coefficient loop, and both loops are closed by a warp vote: the lanes run
// the same stage at the same time.  (Left to themselves, lanes that leave a loop early never wait for
// the others: the first version ran with 4 of 32 lanes active on average and its per-lane macroblock
// loops with ONE.)
template <class BR>
__device__ void syntax_run(BR &br, uint32_t sbase, const SliceConst &sc, bool live, uint32_t limit, uint32_t &st) {
	int ph = (int)(st & 15u);
	uint32_t rem = (st >> 4) & 63u, ty = st >> 10;
	const uint32_t guess_ty = sc.picture_type == 1 ? 1u : 0u;
	const uint32_t end_bit = sc.end_byte * 8u;
	bool run = live && ph < PH_END;
#define SYN_RESYNC() do { br.consume(1); ph = PH_AC; rem = 1u; ty = guess_ty; } while (0)
	while (WK_VOTE(VOTE_SYN_MB, run)) {
		if (run) do {  // the stages before the blocks; `break` leaves them
			// ---- macroblock_address_increment (mpeg1.js:295-310), after the slice-end test of mpeg1.js:276
			while (run && ph <= PH_MBA_ESC) {
				const uint32_t pos = br.bitpos();
				if (ph == PH_MBA && pos >= limit) { run = false; break; }
				if (ph == PH_MBA && ((pos + 7u) >> 3) >= sc.end_byte) { ph = PH_END; run = false; break; }
				const uint32_t e = clz_lut(sbase + OFF_MBA, br.peek32(), VLC_MBA_MAX_Z);
				if ((e & 31u) == 0) { SYN_RESYNC(); break; }
				br.consume((int)(e & 31u));
				const uint32_t v = e >> 5;
				if (v == 35u) ph = PH_MBA_ESC;
				else if (v == 34u && ph != PH_MBA_ESC) ph = PH_MBA_STUFF;  // after an escape, 34 is an increment (mpeg1.js:297-306)
				else ph = PH_TYPE;
			}
			if (!run) break;
			// ---- macroblock_type (+ quantiser scale), mpeg1.js:348-361
			if (ph == PH_TYPE) {
				const uint32_t w = br.peek32();
				const uint32_t e = sc.picture_type == 1 ? lds_u16(sbase + OFF_TYPE_I + (w >> 30) * 2u)
				                                        : lds_u16(sbase + OFF_TYPE_P + (w >> 26) * 2u);
				if ((e & 31u) == 0) {
					SYN_RESYNC();
				} else {
					const uint32_t type = e >> 5;
					br.consume((int)(e & 31u) + ((type & 0x10u) ? 5 : 0));
					ty = type & 3u;
					rem = 0;
					if (!(type & 1u) && (type & 8u)) ph = PH_MV_H;
					else if (type & 2u) ph = PH_CBP;
					else if (type & 1u) { ph = PH_DC; rem = 0x3fu; }
					else ph = PH_MBA;
				}
			}
			// ---- motion vectors (mpeg1.js:395-457): code + residual, values not needed
			while (ph == PH_MV_H || ph == PH_MV_V) {
				const uint32_t e = clz_lut(sbase + OFF_MOTION, br.peek32(), VLC_MOTION_MAX_Z);
				if ((e & 31u) == 0) { SYN_RESYNC(); break; }
				const int code = (int)(e >> 5) - 16;
				br.consume((int)(e & 31u) + ((code != 0 && sc.f != 1) ? sc.r_size : 0));
				if (ph == PH_MV_H) ph = PH_MV_V;
				else if (ty & 2u) ph = PH_CBP;
				else ph = PH_MBA;  // motion only: no blocks (intra macroblocks carry no vectors)
			}
			// ---- coded_block_pattern (mpeg1.js:376-384)
			if (ph == PH_CBP) {
				const uint32_t e = clz_lut(sbase + OFF_CBP, br.peek32(), VLC_CBP_MAX_Z);
				if ((e & 31u) == 0) {
					SYN_RESYNC();
				} else {
					br.consume((int)(e & 31u));
					rem = e >> 5;
					ty &= 1u;
					ph = rem == 0 ? PH_MBA : ((ty & 1u) ? PH_DC : PH_AC_FIRST);
				}
			}
		} while (0);
		// ---- blocks (mpeg1.js:698-790), current block = highest bit of rem.  One look-up per trip for
		// whatever block the lane is in: lanes wait for the longest MACROBLOCK of the 32, not the longest block
		bool in = run && ph >= PH_DC && ph <= PH_AC;
		while (WK_VOTE(VOTE_SYN_AC, in)) {
			if (in) {
				if (br.bitpos() >= end_bit) {  // a chain of garbage must end with the slice
					ph = PH_END; run = false; in = false;
				} else {
					if (ph == PH_DC) {
						const uint32_t w = br.peek32();  // blocks 0..3 are the mask bits 0x20..0x04
						const uint32_t e = rem >= 4u ? lds_u16(sbase + OFF_DC_LUMA + (w >> 25) * 2u)
						                             : lds_u16(sbase + OFF_DC_CHROMA + (w >> 24) * 2u);
						if ((e & 31u) == 0) SYN_RESYNC();
						else br.consume((int)(e & 31u) + (int)(e >> 5));
						ph = PH_AC;
					}
					int n_unused = 0;
					const int r = ac_step(br, sbase, n_unused, true, ph == PH_AC_FIRST);
					ph = PH_AC;
					if (r == 2) SYN_RESYNC();
					else if (r == 1) {
						rem &= ~(0x80000000u >> __clz((int)rem));
						ph = rem == 0 ? PH_MBA : ((ty & 1u) ? PH_DC : PH_AC_FIRST);
						if (rem == 0) in = false;
					}
				}
			}
		}
	}
#undef SYN_RESYNC
	if (ph <= PH_TYPE || ph >= PH_END) { rem = 0; ty = 0; }
	st = syn_make(ph, rem, ty);
}

// What the macroblocks a lane owns do to the slice state, relative to the state they start from.
struct LaneSum {
	int d_addr, qs, dcy, dc4, dc5, mvh, mvv;
	uint32_t flags;  // 1 quantiser scale set, 2 DC predictors absolute, 4 motion predictors absolute
};
__device__ __forceinline__ int wrap_mv(int v, int f) {  // mpeg1.js:413-419: arithmetic modulo 32 f in [-16 f, 16 f)
	if (v > (f << 4) - 1) v -= f << 5;
	else if (v < -(f << 4)) v += f << 5;
	return v;
}
__device__ __forceinline__ LaneSum compose(const LaneSum &a, const LaneSum &b, int f) {  // a, then b (associative)
	LaneSum r;
	r.d_addr = a.d_addr + b.d_addr;
	r.qs = (b.flags & 1u) ? b.qs : a.qs;
	const bool dabs = b.flags & 2u, mabs = b.flags & 4u;
	r.dcy = dabs ? b.dcy : a.dcy + b.dcy;
	r.dc4 = dabs ? b.dc4 : a.dc4 + b.dc4;
	r.dc5 = dabs ? b.dc5 : a.dc5 + b.dc5;
	r.mvh = mabs ? b.mvh : wrap_mv(a.mvh + b.mvh, f);
	r.mvv = mabs ? b.mvv : wrap_mv(a.mvv + b.mvv, f);
	r.flags = a.flags | b.flags;
	return r;
}
__device__ __forceinline__ LaneSum shfl_up_sum(const LaneSum &s, int d) {
	LaneSum r;
	r.d_addr = __shfl_up_sync(FULL_MASK, s.d_addr, d);
	r.qs = __shfl_up_sync(FULL_MASK, s.qs, d);
	r.dcy = __shfl_up_sync(FULL_MASK, s.dcy, d);
	r.dc4 = __shfl_up_sync(FULL_MASK, s.dc4, d);
	r.dc5 = __shfl_up_sync(FULL_MASK, s.dc5, d);
	r.mvh = __shfl_up_sync(FULL_MASK, s.mvh, d);
	r.mvv = __shfl_up_sync(FULL_MASK, s.mvv, d);
	r.flags = __shfl_up_sync(FULL_MASK, s.flags, d);
	return r;
}

// The byte index of the first start code prefix (00 00 01) at or after `from`, or len: where
// nextBytesAreStartCode (buffer.js:141-150) first becomes true.  The warp scans 128 bytes per step.
template <class BR>
__device__ uint32_t find_slice_end(const BR &br, uint32_t from, int lane, const ParseTask &t) {
	const uint32_t len = br.len;
	if (t.codes) {  // the host's sorted list of every prefix in the stream: a few steps from this picture's own start code
		uint32_t i = t.code_hint;
		while (i < t.n_codes && __ldg(t.codes + i) < from) i++;
		return i < t.n_codes ? __ldg(t.codes + i) : len;
	}
	for (uint32_t base = from >> 2; base * 4u < len; base += 32u) {
		const uint32_t wi = base + (uint32_t)lane;
		const uint64_t x = ((uint64_t)br.load_word_direct(wi) << 32) | br.load_word_direct(wi + 1u);  // bytes 4 wi .. 4 wi + 7
		uint32_t hit = 0xffffffffu;
#pragma unroll
		for (int k = 3; k >= 0; k--) {
			const uint32_t p = wi * 4u + (uint32_t)k;
			if (((uint32_t)(x >> (40 - 8 * k)) & 0xffffffu) == 1u && p >= from && p + 2u < len) hit = p;
		}
		const unsigned any = __ballot_sync(FULL_MASK, hit != 0xffffffffu);
		if (any) return __shfl_sync(FULL_MASK, hit, __ffs((int)any) - 1);
	}
	return len;
}

// The macroblocks that START in [reader position, limit), walked in MODE (WALK_REL / WALK_ABS).
// Returns 0 when the lane reached `limit` (or owns nothing), 1 when the slice ended cleanly at the
// start code, 2 on anything else; stop_pos = the bit position after the lane's last macroblock.
// WARP-SYNCHRONOUS like syntax_run: one vote closes the macroblock loop, one every look-up of the
// coefficient loop.
// WALK_STAGE: where a lane leaves its macroblocks as relative records: 64-byte entries of the picture's
// staging area (ParseTask::stage), the lane's own stretch [first, first + cap), in walking order.
//   word 0      motion predictors after the macroblock's header (int16 h | int16 v << 16); skip entry: the run length
//   word 1      flags (1 intra, 2 skip entry, 4 motion absolute, 8 DC absolute, 16 quantiser scale set)
//               | cbp << 8 | dc_only mask << 16 | quantiser scale << 24
//   word 2      bit_pos      word 3   macroblock address relative to the lane's start (skip entry: the first skipped one)
//   words 4..15 per block {bit offset of the first coefficient code, DC predictor value (relative unless flag 8)}
struct StageArea {
	int first, cap, count;
	bool ok;  // false: more macroblocks than room -- the summary is still right, the storing pass has to run
};
__device__ __forceinline__ uint4 *stage_entry(const ParseTask &t, const StageArea &sa, int k) { return t.stage + (size_t)(sa.first + k) * 4; }

template <int MODE, class BR>
__device__ int walk_owned(BR &br, uint32_t sbase, PictureState &ls, const ParseTask &t, int mb_size, bool owns,
                          uint32_t limit, uint32_t end_byte, int lane, uint32_t &stop_pos, StageArea *sa = nullptr) {
	int how = 0;
	bool work = owns;
	if (owns) stop_pos = br.bitpos();
	while (WK_VOTE(VOTE_OWN_MB, work)) {
		MbHead h;
		h.mb = 0; h.cbp = 0; h.mv_h = h.mv_v = h.qscale = 0; h.intra = false; h.bit_pos = 0;
		h.n_skip = 0; h.skip_first = 0; h.skip_qs = 0; h.skip_qs_set = false; h.skip_bit = 0;
		bool in_mb = false;
		if (work) {
			if (walk_mb_header<MODE>(br, sbase, ls, t, mb_size, lane, h) != 0) { how = 2; work = false; }
			else in_mb = true;
		}
		uint2 *park_mb = t.park + (size_t)(MODE == WALK_ABS ? h.mb : 0) * 6;
		bool staging = false;
		if (MODE == WALK_STAGE && in_mb && sa->ok) {
			if (sa->count + (h.n_skip > 0 ? 2 : 1) > sa->cap) {
				sa->ok = false;
			} else {
				if (h.n_skip > 0)
					*stage_entry(t, *sa, sa->count++) = make_uint4((uint32_t)h.n_skip, 2u | (h.skip_qs_set ? 16u : 0u) | ((uint32_t)h.skip_qs << 24),
					                                             h.skip_bit, (uint32_t)h.skip_first);
				park_mb = reinterpret_cast<uint2 *>(stage_entry(t, *sa, sa->count) + 1);  // the blocks' pairs go straight into the entry
				staging = true;
			}
		}
		int done = 0, dc_mask = 0;
		// the coded blocks of the macroblock, one look-up per trip; a block's head (intra DC, the parked
		// pair) rides on the trip of its first look-up
		uint32_t rem = in_mb ? (uint32_t)h.cbp : 0u;  // blocks still to walk, current = highest bit
		bool at_head = true, first = false;
		int n = 0;
		bool in = rem != 0;
		while (WK_VOTE(VOTE_OWN_AC, in)) {
			if (in) {
				const int block = __clz((int)rem) - 26;  // mask bit 0x20 >> block
				bool ok = true;
				if (at_head) {
					ok = MODE == WALK_STAGE ? walk_block_head<true, true>(br, sbase, ls, h.intra, block, park_mb + block, staging, n, first)
					                        : walk_block_head<true>(br, sbase, ls, h.intra, block, park_mb + block, MODE == WALK_ABS, n, first);
					at_head = false;
				}
				const int r = ok ? ac_step(br, sbase, n, true, first) : 2;
				first = false;
				if (r == 2) { how = 2; work = false; in_mb = false; in = false; }
				else if (r == 1) {
					bool dc_only;
					walk_block_tail(ls, n, dc_only);
					done |= 0x20 >> block;
					if (dc_only) dc_mask |= 0x20 >> block;
					rem &= ~(0x20u >> block);
					at_head = true;
					if (rem == 0) in = false;
				}
			}
		}
		if (in_mb) {
			if (MODE == WALK_ABS)
				reinterpret_cast<uint4 *>(t.hdr)[h.mb] =
				    pack_record(h.mv_h, h.mv_v, MBF_PRESENT | (h.intra ? MBF_INTRA : 0), done, dc_mask, h.qscale, h.bit_pos);
			if (MODE == WALK_STAGE && staging) {
				const uint32_t flags = (h.intra ? 1u : 0u) | (ls.mv_abs ? 4u : 0u) | (ls.dc_abs ? 8u : 0u) | (ls.qs_set ? 16u : 0u);
				*stage_entry(t, *sa, sa->count++) =
				    make_uint4(((uint32_t)ls.mv_h_prev & 0xffffu) | ((uint32_t)ls.mv_v_prev << 16),
				               flags | ((uint32_t)done << 8) | ((uint32_t)dc_mask << 16) | ((uint32_t)h.qscale << 24), h.bit_pos, (uint32_t)h.mb);
			}
			ls.n_present++;
			const uint32_t pos = br.bitpos();
			const uint32_t i = (pos + 7u) >> 3;
			stop_pos = pos;
			if (i >= end_byte) { how = i == end_byte ? 1 : 2; work = false; }
			else if (pos >= limit) work = false;
		}
	}
	return how;
}

// One slice: the reader is at its first macroblock (bit p_start), `ps` holds the picture constants and
// the slice's initial state (mb_addr, qscale).  true: records stored, ps totals updated, reader at the
// start code prefix that ended the slice.  false: outside the clean domain, nothing is to be trusted.
template <class BR>
__device__ bool walk_slice_lanes(BR &br, uint32_t sbase, PictureState &ps, const ParseTask &t, int mb_size, int lane) {
	const uint32_t p_start = br.bitpos();
	const uint32_t end_byte = find_slice_end(br, (p_start + 7u) >> 3, lane, t);
	if (((p_start + 7u) >> 3) >= end_byte) return false;
	const uint32_t end_bit = end_byte * 8u;
	const uint32_t total = end_bit - p_start;
	uint32_t L = (total + 31u) >> 5;
	if (L < MIN_SUBSEQ_BITS) L = MIN_SUBSEQ_BITS;
	const int K = (int)((total + L - 1u) / L);  // 1..32 sub-sequences
	const bool active = lane < K;
	const uint32_t s_lo = active ? p_start + (uint32_t)lane * L : end_bit;
	const uint32_t s_hi = (active && lane < K - 1) ? s_lo + L : end_bit;
	SliceConst sc;
	sc.picture_type = ps.picture_type; sc.r_size = ps.r_size; sc.f = ps.f; sc.end_byte = end_byte;

	// ---- W: warm-up to the first macroblock that starts in the sub-sequence.  Chains merge within a few
	// macroblocks, so the warm-up is WARMUP_BITS or 48 average macroblocks, whichever is longer
	const uint32_t warm = max(WARMUP_BITS, total / (uint32_t)mb_size * WARMUP_MBS);
	uint32_t st = PH_MBA;
	if (active) {
		if (lane == 0 || s_lo - p_start <= warm) {
			br.seek_bit(p_start);  // the true chain from the slice's first macroblock
		} else {
			br.seek_bit(s_lo - warm);
			st = syn_guess(sc);
		}
	}
	syntax_run(br, sbase, sc, active && lane > 0, s_lo, st);
	const uint32_t q = active ? br.bitpos() : end_bit;
	const bool owns = active && (st & 15u) == PH_MBA && q < s_hi && ((q + 7u) >> 3) < end_byte;
	bool bad = false;

	// ---- C: the relative summary of the owned macroblocks; every lane must stop where the next one started
	PictureState ls = ps;  // picture constants; the rest is set per pass
	LaneSum sum;
	sum.d_addr = 0; sum.qs = 0; sum.dcy = sum.dc4 = sum.dc5 = 0; sum.mvh = sum.mvv = 0; sum.flags = 0;
	int how = 0;
	if (owns) {
		ls.mb_addr = 0; ls.qscale = 0; ls.slice_begin = lane == 0;
		ls.mv_h = ls.mv_v = ls.mv_h_prev = ls.mv_v_prev = 0;
		ls.dc_y = ls.dc_b4 = ls.dc_b5 = 0;
		ls.qs_set = ls.dc_abs = ls.mv_abs = ls.anomaly = false;
		ls.n_present = ls.n_coded = ls.error = 0;
	}
	uint32_t stop_pos = q;
	if (!owns) ls.n_present = ls.n_coded = ls.error = 0;  // (with the fix-up, this pass's counts are the final ones)
	StageArea sa;
	sa.cap = t.stage ? t.stage_entries / K : 0;  // the picture's staging entries, shared out among the lanes in use
	sa.first = active ? lane * sa.cap : 0;
	sa.count = 0;
	sa.ok = sa.cap > 0;
	how = walk_owned<WALK_STAGE>(br, sbase, ls, t, mb_size, owns, s_hi, end_byte, lane, stop_pos, &sa);
	const uint32_t next_q = __shfl_down_sync(FULL_MASK, q, 1);
	if (active && lane < K - 1 && stop_pos != next_q) bad = true;  // the warm-up of lane + 1 had not merged
	if (owns) {
		if (how == 2) bad = true;
		sum.d_addr = ls.mb_addr; sum.qs = ls.qscale;
		sum.dcy = ls.dc_y; sum.dc4 = ls.dc_b4; sum.dc5 = ls.dc_b5;
		sum.mvh = ls.mv_h_prev; sum.mvv = ls.mv_v_prev;
		sum.flags = (ls.qs_set ? 1u : 0u) | (ls.dc_abs ? 2u : 0u) | (ls.mv_abs ? 4u : 0u);
	}
	if (__any_sync(FULL_MASK, bad)) return false;
	const unsigned enders = __ballot_sync(FULL_MASK, how == 1);
	if (__popc(enders) != 1) return false;  // exactly one lane sees the slice end at its start code

	// inclusive scan of the summaries, then the absolute state at each lane's first macroblock
	for (int d = 1; d < 32; d <<= 1) {
		const LaneSum o = shfl_up_sum(sum, d);
		if (lane >= d) sum = compose(o, sum, ps.f);
	}
	LaneSum x0;
	x0.d_addr = ps.mb_addr; x0.qs = ps.qscale; x0.dcy = x0.dc4 = x0.dc5 = 128; x0.mvh = x0.mvv = 0; x0.flags = 7u;
	const LaneSum before = shfl_up_sum(sum, 1);
	const LaneSum x = lane == 0 ? x0 : compose(x0, before, ps.f);

	if (!__any_sync(FULL_MASK, owns && !sa.ok)) {
		// ---- F: no second walk -- the staged relative records become the final ones.  Every staged value is
		// cumulative since the lane's start, so each entry only needs the lane's absolute start state `x`.
		// No bitstream access, no look-ups, all lanes busy: some 40 instructions per macroblock.
		int k = 0;
		while (WK_VOTE(VOTE_OWN_MB, k < sa.count)) {
			if (k < sa.count) {
				const uint4 *e = stage_entry(t, sa, k);
#ifndef JSMPEG_WALK_EMU
				if (k + 2 < sa.count) asm volatile("prefetch.global.L1 [%0];" ::"l"(e + 8));  // the entry after next (written by this lane, sits in L2)
#endif
				const uint4 w = e[0];
				const uint32_t flags = w.y & 0xffu;
				const int qs = (flags & 16u) ? (int)(w.y >> 24) : x.qs;
				const int mb = x.d_addr + (int)w.w;
				if (flags & 2u) {  // a run of skipped macroblocks (mpeg1.js:323-346): zero vector, the scale in force
					const int n_skip = (int)w.x;
					if (mb < 0 || mb + n_skip > mb_size) bad = true;
					else {
						const uint4 rec = pack_record(0, 0, MBF_PRESENT | MBF_SKIPPED, 0, 0, qs, w.z);
						for (int i = 0; i < n_skip; i++) reinterpret_cast<uint4 *>(t.hdr)[mb + i] = rec;
					}
				} else if (mb < 0 || mb >= mb_size) {
					bad = true;
				} else {
					int ph = (int)(int16_t)(w.x & 0xffffu), pv = (int)(int16_t)(w.x >> 16);
					if (!(flags & 4u)) { ph = wrap_mv(x.mvh + ph, ps.f); pv = wrap_mv(x.mvv + pv, ps.f); }
					const int cbp = (int)((w.y >> 8) & 0xffu);
					uint4 pr[3] = {e[1], e[2], e[3]};  // six {bit offset, DC predictor} pairs; uncoded blocks' are stale, never read
					if (flags & 1u) {  // intra: predictor value -> the record's clamped dc (x 256 = dc << 8 in stage 2, mpeg1.js:747)
						uint32_t *v = reinterpret_cast<uint32_t *>(pr);
#pragma unroll
						for (int block = 0; block < 6; block++) {
							int dc = (int)v[block * 2 + 1];
							if (!(flags & 8u)) dc += block < 4 ? x.dcy : (block == 4 ? x.dc4 : x.dc5);
							v[block * 2 + 1] = (uint32_t)max(-INTRA_DC_BOUND, min(255 + INTRA_DC_BOUND, dc)) & 0xffffu;
						}
					} else {
						pr[0].y = pr[0].w = pr[1].y = pr[1].w = pr[2].y = pr[2].w = 0u;
					}
					uint4 *park_mb = reinterpret_cast<uint4 *>(t.park + (size_t)mb * 6);
					park_mb[0] = pr[0]; park_mb[1] = pr[1]; park_mb[2] = pr[2];
					reinterpret_cast<uint4 *>(t.hdr)[mb] =
					    pack_record(ps.full_pel ? ph * 2 : ph, ps.full_pel ? pv * 2 : pv, MBF_PRESENT | ((flags & 1u) ? MBF_INTRA : 0),
					                cbp, (int)((w.y >> 16) & 0xffu), qs, w.z);
				}
				k++;
			}
		}
		if (__any_sync(FULL_MASK, bad)) return false;
		ps.n_fixup++;
	} else {
	// ---- D (a lane ran out of staging room): the owned macroblocks again, absolute, storing
	ls.n_present = ls.n_coded = ls.error = 0;
	ls.anomaly = false;
	if (owns) {
		br.seek_bit(q);
		ls.mb_addr = x.d_addr; ls.qscale = x.qs; ls.slice_begin = lane == 0;
		ls.dc_y = x.dcy; ls.dc_b4 = x.dc4; ls.dc_b5 = x.dc5;
		ls.mv_h_prev = x.mvh; ls.mv_v_prev = x.mvv;
		ls.mv_h = ps.full_pel ? x.mvh * 2 : x.mvh;
		ls.mv_v = ps.full_pel ? x.mvv * 2 : x.mvv;
	}
	const int how_abs = walk_owned<WALK_ABS>(br, sbase, ls, t, mb_size, owns, s_hi, end_byte, lane, stop_pos);
	if (how_abs != how || ls.anomaly) bad = true;
	if (__any_sync(FULL_MASK, bad)) return false;
	}
	int n_present = ls.n_present, n_coded = ls.n_coded, error = ls.error;
	for (int d = 16; d > 0; d >>= 1) {
		n_present += __shfl_xor_sync(FULL_MASK, n_present, d);
		n_coded += __shfl_xor_sync(FULL_MASK, n_coded, d);
		error = max(error, __shfl_xor_sync(FULL_MASK, error, d));
	}
	ps.n_present += n_present;
	ps.n_coded += n_coded;
	if (error) ps.error = error;
	br.seek_byte(end_byte);
	return true;
}

// ==================================================================================================
// one picture = one warp

// the shared-memory tables of the walk; `ms_table` is the device's multi-symbol table (build_ms_table)
__device__ __forceinline__ void walk_tables_init(uint8_t *smem, int tid, int nthreads, const uint4 *__restrict__ ms_table, bool with_first) {
	uint16_t *s16 = reinterpret_cast<uint16_t *>(smem);
	for (int i = tid; i < (VLC_DCT_MAX_Z + 1) * 32; i += nthreads) s16[OFF_DCT / 2 + i] = walk_entry(VLC_DCT_COEFF[i]);
	for (int i = tid; i < (VLC_MBA_MAX_Z + 1) * 32; i += nthreads) s16[OFF_MBA / 2 + i] = VLC_MBA[i];
	for (int i = tid; i < (VLC_CBP_MAX_Z + 1) * 32; i += nthreads) s16[OFF_CBP / 2 + i] = VLC_CBP[i];
	for (int i = tid; i < (VLC_MOTION_MAX_Z + 1) * 32; i += nthreads) s16[OFF_MOTION / 2 + i] = VLC_MOTION[i];
	for (int i = tid; i < 128; i += nthreads) s16[OFF_DC_LUMA / 2 + i] = VLC_DC_SIZE_LUMA[i];
	for (int i = tid; i < 256; i += nthreads) s16[OFF_DC_CHROMA / 2 + i] = VLC_DC_SIZE_CHROMA[i];
	for (int i = tid; i < 4; i += nthreads) s16[OFF_TYPE_I / 2 + i] = VLC_MBTYPE_I[i];
	for (int i = tid; i < 64; i += nthreads) s16[OFF_TYPE_P / 2 + i] = VLC_MBTYPE_P[i];
	uint4 *ms = reinterpret_cast<uint4 *>(smem + OFF_MS);
	const int n16 = (int)(with_first ? 2u * MS_TABLE_ENTRIES : (2u << MS_BITS)) / 16;
	for (int i = tid; i < n16; i += nthreads) ms[i] = __ldg(ms_table + i);
}

// decodePicture (mpeg1.js:174-247), bitstream side.  LANES: every slice is first tried with the
// lane-parallel walk; the first slice outside its domain makes the warp start the picture over with
// the serial walk (info.reserved[0] tells which one produced the records).
template <bool LANES>
__device__ void walk_picture(const ParseTask &t, uint32_t sbase, int lane, uint32_t ring) {
	const int mb_width = t.mb_width, mb_size = t.mb_size;
	bool lanes = LANES;
	for (;;) {
		// no macroblock is present until the walk reaches it (an address no slice covers keeps the
		// two-pictures-old samples, SURVEY Q12)
		for (int i = lane; i < mb_size; i += 32) reinterpret_cast<uint4 *>(t.hdr)[i] = make_uint4(0, 0, 0, 0);
		__syncwarp();

		BitReaderT<LANES> br;
		br.words = reinterpret_cast<const uint32_t *>(t.es);
		br.bytes = t.es;
		br.len = t.es_len;
		br.ring = ring;
		br.seek_byte(t.start_byte);

		PictureState ps;
		ps.n_present = ps.n_coded = ps.error = 0;
		ps.n_fixup = 0;
		ps.full_pel = 0; ps.r_size = 0; ps.f = 1;
		ps.qs_set = ps.dc_abs = ps.mv_abs = ps.anomaly = false;
		int f_code = 0;
		int status = PIC_IGNORED;

		// picture header (mpeg1.js:174-196)
		br.consume(10);
		ps.picture_type = (int)br.read(3);
		br.consume(16);
		bool go = ps.picture_type == 1 || ps.picture_type == 2;
		if (ps.picture_type == 2) {
			ps.full_pel = (int)br.read(1);
			f_code = (int)br.read(3);
			if (f_code == 0) go = false;
			else { ps.r_size = f_code - 1; ps.f = 1 << ps.r_size; }
		}
		uint32_t end_bit;
		bool again = false;
		if (!go) {
			end_bit = br.bitpos();
		} else {
			status = PIC_DECODED;
			int code;
			do { code = br.find_next_start_code(); } while (code == 0xB5 || code == 0xB2);  // mpeg1.js:198-201
			while (code >= 0x01 && code <= 0xAF) {
				// slice (mpeg1.js:255-276)
				ps.slice_begin = true;
				ps.mb_addr = (code - 1) * mb_width - 1;
				ps.mv_h = ps.mv_v = ps.mv_h_prev = ps.mv_v_prev = 0;
				ps.dc_y = ps.dc_b4 = ps.dc_b5 = 128;
				ps.qscale = (int)br.read(5);
				while (br.read(1)) br.consume(8);
				if (LANES && lanes) {
					if (!walk_slice_lanes(br, sbase, ps, t, mb_size, lane)) {
						again = true;
						break;
					}
				} else {
					do {
						if (!walk_macroblock(br, sbase, ps, t, mb_size, lane)) {
							if (!ps.error) ps.error = PARSE_ERR_INVALID_VLC;
							break;
						}
					} while (!br.next_bytes_are_start_code());
				}
				code = br.find_next_start_code();
			}
			end_bit = br.bitpos();
			if (code != -1) end_bit -= 32;  // mpeg1.js:209-213
		}
		if (LANES && again) {
			lanes = false;
			__syncwarp();
			continue;
		}
		if (lane == 0) {
			picture_info_t info;
			info.start_byte = t.start_byte;
			info.end_bit = end_bit;
			info.status = status;
			info.picture_type = ps.picture_type;
			info.full_pel = ps.full_pel;
			info.f_code = f_code;
			info.n_present = ps.n_present;
			info.n_coded_blocks = ps.n_coded;
			info.error = ps.error;
			info.reserved[0] = (LANES && lanes && go) ? 1 : 0;
			info.reserved[1] = 0;
			info.reserved[2] = (LANES && lanes && go) ? ps.n_fixup : 0;
			*t.info = info;
		}
		return;
	}
}

// ==================================================================================================
// 1b: coded blocks, from the offset the walk parked to the finished record.
// rec = the macroblock record's second word (flags | cbp << 8 | dc_only << 16 | quantiser scale << 24),
// parked = {bit offset of the block's first coefficient code, intra dc (clamped, records.h)} from the walk's dense side array.
//
// Run/level codes arrive in zig-zag order, and the compact record (coef_records.h) IS the position mask plus the
// values in zig-zag order: the k-th value a block's codes give is level[k].  So a block is built as its compact
// record directly, in a 32-byte row of its warp's staging area in shared memory (expand_compact_row), and the warp
// stores the rows of its 32 consecutive slots itself, as whole 512-byte stretches (store_compact_rows).  Only a
// block of more than COEF_RECORD_LEVELS positions is decoded a second time, into a zeroed 64 x int16 tile through
// the raster offsets, and leaves as the dense record (expand_dense_record).
//
// The code loop (expand_codes) is built to need few instructions per code:
//  * no bit window to maintain: the 32 bits at the current bit POSITION are two word loads (L1 hits: the
//    blocks of a warp lie side by side in the stream) and one funnel shift -- the loads go to the LSU, the
//    address to the FMA pipe; the window's shifts, counters and predicated refill were a quarter of the loop.
//    (Keeping the three words around the position in registers and loading one word per crossing -- the
//    load off the chain from code to code -- was slower: the predicated register moves cost more than the
//    L1 hits.)
//  * the frequent codes (at most 8 bits) come from a table indexed by the next 8 bits (VLC_DCT_EXPAND_TOP8),
//    no clz and no second shift; entries hold what a trip needs: bits to consume, run + 1, 2 * level
//  * dequantisation in sign-magnitude form.  The reference (mpeg1.js:794-807): level <<= 1;
//    if (!intra) level += level < 0 ? -1 : 1;  level = (level * qs * Q) >> 4;  if even: level -= level > 0 ? 1 : -1;
//    clamp to [-2048, 2047].  With m = 2 |level| + (intra ? 0 : 1) and p = m * qs * Q >= 0: the arithmetic
//    shift is floor, so the product's magnitude is t = p >> 4 for a positive level and t = (p + 15) >> 4 for a
//    negative one; "make odd, toward zero" is (t - 1) | 1 for t >= 1, and t = 0 becomes +1 WHATEVER the sign
//    (0 is even and not > 0); the clamp is min(., 2047 + negative).  The multiplies run on the FMA pipe.
//    (tests/test_expand_arith.py: all of it against the reference's statements, exhaustively.)
__device__ __forceinline__ int dequant_sm(int mag2_plus, int neg, int qs, uint32_t q) {
	// mag2_plus = 2 |level| + (intra ? 0 : 1), neg = 0 / 1, q = raster index * 2 | Q << 8
	const int p = mag2_plus * (qs * (int)(q >> 8)) + neg * 15;
	const int t = p >> 4;
	const int r = min(max((t - 1) | 1, 1), 2047 + neg);
	return (neg && t != 0) ? -r : r;
}
// The codes of one block: put(q, value) for every value in zig-zag order, q = the position's quantiser entry (its
// low byte: the raster offset in bytes; 0 for the intra DC).  Returns the zig-zag positions written (the compact
// record's mask).
template <class Put>
__device__ __forceinline__ uint64_t expand_codes(const ParseTask &t, uint32_t rec, uint2 parked, uint32_t sbase, Put put) {
	const bool intra = rec & MBF_INTRA;
	const int ni = intra ? 0 : 1;
	const int qs = (int)(rec >> 24);
	// quantiser table in coefficient (zig-zag) order: entry n = raster index * 2 | Q[raster index] << 8
	const uint32_t xq = sbase + EXP_OFF_XQ + (intra ? 0u : 128u);
	BitReaderT<false, ES_IS_PADDED> br;  // for its word loads only; every code of the block was validated by the walk:
	br.words = reinterpret_cast<const uint32_t *>(t.es);  // the reads stay inside data + pad
	br.bytes = t.es;
	br.len = t.es_len;
	br.ring = 0;
	auto window = [&](uint32_t pos) {  // the 32 bits at bit position pos, MSB first
		const uint32_t i = pos >> 5;
		return __funnelshift_l(br.load_word(i + 1u), br.load_word(i), pos);  // (shifts by pos & 31)
	};
	uint32_t pos = parked.x;
	uint32_t w = window(pos);

	int n = 0;
	uint64_t written = 0;
	if (intra) {
		put(0u, (int)(int16_t)(parked.y & 0xffffu));  // coefficient 0
		n = 1;
		written = 1;
	} else if (w >> 31) {
		// dct_coeff_first of a non-intra block: a leading '1' is (run 0, level +-1) with its sign bit, never
		// end_of_block (mpeg1.js:757-760, 781-787) -- handled here, once, instead of in every trip of the loop
		const uint32_t q = lds_u16(xq);
		put(q, dequant_sm(3, (int)((w >> 30) & 1u), qs, q));
		pos += 2u;
		w = window(pos);
		n = 1;
		written = 1;
	}
	for (;;) {  // mpeg1.js:757-811; the walk has already validated every code of this block
		uint32_t x = lds_u32(sbase + EXP_OFF_TOP8 + ((w >> 24) << 2));
		if (x == 0u) {  // a code of more than 8 bits (or none)
			const int z = min(__clz((int)w), VLC_DCT_MAX_Z);
			x = lds_u32(sbase + EXP_OFF_DCT + ((((uint32_t)z << 5) | ((w << (z + 1)) >> 27)) << 2));
		}
		int mag2 = (int)((x >> 16) & 0xffu);
		uint32_t nb = x & 63u;
		int run1 = (int)((x >> 8) & 63u);
		int neg;
		if (mag2 == 0) {
			if (!(x >> 30)) break;  // end_of_block (or, defensively, not a code)
			// escape (mpeg1.js:767-780): 6-bit run, 8 (+8) bit level
			run1 = (int)((w >> 20) & 63u) + 1;
			const int l8 = (int)((w >> 12) & 255u);
			int level;
			if ((l8 & 127) == 0) {
				level = (int)((w >> 4) & 255u) - (l8 << 1);  // l8 == 128: second byte - 256
				nb = 28u;
			} else {
				level = l8 > 128 ? l8 - 256 : l8;
				nb = 20u;
			}
			neg = level < 0;
			mag2 = 2 * abs(level);
		} else {
			neg = (int)((w >> (32u - nb)) & 1u);  // the sign is the last bit consumed
		}
		pos += nb;
		w = window(pos);  // (requested before the arithmetic of this code)
		n += run1;        // one past this coefficient's index
		if (n > 64) {     // JS: ZIG_ZAG[n] undefined -> the store is a no-op (the walk flagged the picture)
			if (n > 4097) break;
			continue;
		}
		const uint32_t q = lds_u16(xq + (uint32_t)(n - 1) * 2u);
		put(q, dequant_sm(mag2 + ni, neg, qs, q));
		written |= (uint64_t)1 << (n - 1);
	}
	return written;
}

// A warp's staging area: the lanes' 32-byte compact rows EXP_ROW_PITCH bytes apart.  40 keeps a row 8-byte aligned
// and starts the rows 10 banks apart: lanes storing their k-th value meet two to a bank (at 32 bytes: eight).
// A lane's 64 x int16 tile for a dense block lies over the same memory, EXP_TILE_PITCH apart (128 + 16: bank spread).
constexpr uint32_t EXP_ROW_PITCH = 40;
constexpr uint32_t EXP_TILE_PITCH = 144;
static_assert(32 * EXP_ROW_PITCH <= 32 * EXP_TILE_PITCH, "a warp's rows lie inside its tiles");

// One block as its compact record in the row at srow: mask at +0, the values from +8 in the order the codes give
// them, the unused levels 0.  Values past the record's twelve are dropped: the mask tells (coef_record_fits).
__device__ __forceinline__ uint64_t expand_compact_row(const ParseTask &t, uint32_t rec, uint2 parked, uint32_t sbase, uint32_t srow) {
	sts_u64(srow + 8u, 0);
	sts_u64(srow + 16u, 0);
	sts_u64(srow + 24u, 0);
	uint32_t at = srow + 8u;
	const uint64_t written = expand_codes(t, rec, parked, sbase, [&](uint32_t, int v) {
		if (at < srow + (uint32_t)sizeof(coef_record_t)) sts_s16(at, v);
		at += 2u;
	});
	sts_u64(srow, written);
	return written;
}

// The rows of the lanes in `fits` to the warp's stretch of the compact plane (first = the record of lane 0's slot):
// the kilobyte goes as 64 chunks of 16 bytes, lane l takes chunks l and l + 32, so one store instruction covers 512
// contiguous bytes, whole sectors.  A chunk whose record is not in `fits` (uncoded, or dense) stays unwritten.
__device__ __forceinline__ void store_compact_rows(coef_record_t *first, uint32_t wstage, int lane, uint32_t fits) {
#pragma unroll
	for (int c = lane; c < 64; c += 32) {
		if (!((fits >> (c >> 1)) & 1u)) continue;
		const uint32_t src = wstage + (uint32_t)(c >> 1) * EXP_ROW_PITCH + (uint32_t)(c & 1) * 16u;
#ifndef JSMPEG_WALK_EMU
		uint4 v;
		asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(src) : "memory");
		asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.z), "=r"(v.w) : "r"(src + 8u) : "memory");
		reinterpret_cast<uint4 *>(first)[c] = v;
#else
		memcpy(reinterpret_cast<uint8_t *>(first) + c * 16, emu_smem + src, 16);
#endif
	}
}

// One block as the dense 64 x int16 record at `slot`, through the thread's tile at stile.
// The finished block leaves as ONE 128-byte TMA bulk store (shared -> global, SASS UBLKCP): whole
// lines reach L2, whereas eight 16-byte stores per thread half-fill 32-byte sectors and made L2
// read every sector back before merging (about as many bytes read as written).
__device__ __forceinline__ void expand_dense_record(const ParseTask &t, uint32_t rec, uint2 parked, uint4 *__restrict__ slot,
                                                    uint32_t sbase, uint32_t stile) {
#pragma unroll
	for (uint32_t i = 0; i < 128u; i += 8u) sts_u64(stile + i, 0);
	expand_codes(t, rec, parked, sbase, [&](uint32_t q, int v) { sts_s16(stile + (q & 0xffu), v); });
#ifndef JSMPEG_WALK_EMU
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the copy engine
	asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], 128;" ::"l"(slot), "r"(stile) : "memory");
	asm volatile("cp.async.bulk.commit_group;" ::: "memory");
	asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // the tile must outlive the read
#else
	memcpy(slot, emu_smem + stile, 128);
#endif
}

// One run of a warp: its 32 consecutive block slots, lane `lane` on slot_id (coded: the slot holds a coded block).
// wstage = the warp's staging area in shared memory.  With a compact plane (t.stage) every coded block is built as
// its compact record and the warp stores the rows; the few blocks that do not fit mark their record dense and leave
// as dense records.  Without one (the host emulation's dense-only mode) every coded block leaves as a dense record.
// All 32 lanes call it.
__device__ __forceinline__ void expand_warp_run(const ParseTask &t, bool coded, uint32_t rec, uint2 parked, int slot_id, int lane,
                                                uint32_t sbase, uint32_t wstage) {
	bool dense = coded;
	if (t.stage) {
		uint64_t written = 0;
		if (coded) written = expand_compact_row(t, rec, parked, sbase, wstage + (uint32_t)lane * EXP_ROW_PITCH);
		const bool fits = coded && coef_record_fits(written);
		dense = coded && !fits;
		__syncwarp();  // the rows are written
		coef_record_t *first = compact_plane(t.stage) + (slot_id - lane);
		store_compact_rows(first, wstage, lane, __ballot_sync(0xffffffffu, fits));
		if (dense) first[lane].mask = COEF_RECORD_DENSE;
	}
	if (__any_sync(0xffffffffu, dense)) {  // (rare: more positions than the compact record holds)
		__syncwarp();  // the rows are read: the tiles lie over them
		if (dense)
			expand_dense_record(t, rec, parked, reinterpret_cast<uint4 *>(t.coef) + (size_t)slot_id * 8, sbase,
			                    wstage + (uint32_t)lane * EXP_TILE_PITCH);
	}
	__syncwarp();  // the next run writes the rows again
}

#ifdef JSMPEG_WALK_EMU
// One block on its own, for the host emulation's one-thread entry points: the row and the tile at stile, the record
// to crec (nullptr: dense records only) or, dense, to `slot` -- expand_warp_run without the warp.
static inline void expand_block(const ParseTask &t, uint32_t rec, uint2 parked, uint4 *slot, uint32_t sbase, uint32_t stile,
                                coef_record_t *crec = nullptr) {
	if (crec) {
		if (coef_record_fits(expand_compact_row(t, rec, parked, sbase, stile))) {
			memcpy(crec, emu_smem + stile, sizeof(coef_record_t));
			return;
		}
		crec->mask = COEF_RECORD_DENSE;
	}
	expand_dense_record(t, rec, parked, slot, sbase, stile);
}
#endif

// Multi-symbol walk table: for every MS_BITS-bit prefix, the complete dct_coeff_next codes (with their
// sign bits) that fit, greedily.  Entry: bits 0..3 = bits to consume (0 = first code does not fit
// or is an escape: take the single-symbol path), bits 4..9 = sum of (run + 1), bit 10 = the last
// code consumed was end_of_block.  `dct` is the generated clz-indexed DCT table (VLC_DCT_COEFF).
// It is followed by the dct_coeff_first variant for the prefixes with a leading 1: that '1s' is the
// code (0, +-1), then the same greedy continuation.  `ms` holds MS_TABLE_ENTRIES entries.
static inline void build_ms_table(const uint16_t *dct, uint16_t *ms) {
	auto greedy = [&](uint32_t w, int pos, int n) {
		int eob = 0;
		for (;;) {
			const uint32_t v = w << pos;  // bits beyond the prefix read as 0 and are never trusted: lengths are checked
			int z = 0;
			while (z < 32 && !((v << z) & 0x80000000u)) z++;
			if (z > VLC_DCT_MAX_Z) break;
			const uint16_t e = dct[(z << 5) | ((z + 1 < 32 ? (v << (z + 1)) : 0u) >> 27)];
			const int len = e & 31, run = (e >> 5) & 31, level = e >> 10;
			if (len == 0) break;
			if (level == 0) {
				if (run == 1 && pos + 2 <= MS_BITS) { pos += 2; eob = 1; }
				break;  // escape: single-symbol path
			}
			if (pos + len + 1 > MS_BITS) break;
			pos += len + 1;
			n += run + 1;
		}
		return (uint16_t)(pos | (n << 4) | (eob << 10));
	};
	for (uint32_t prefix = 0; prefix < (1u << MS_BITS); prefix++) ms[prefix] = greedy(prefix << (32 - MS_BITS), 0, 0);
	for (uint32_t low = 0; low < (1u << (MS_BITS - 1)); low++)
		ms[(1u << MS_BITS) + low] = greedy((1u << 31) | (low << (32 - MS_BITS)), 2, 1);
}

}  // namespace
