// walk_slices.cuh -- stage 1a for pictures cut into many slices (sm_90a): one LANE per slice.
//
// The lane-parallel walk (walk.cuh) was built for what FFmpeg's mpeg1video encoder writes: ONE slice per picture,
// whose bits it cuts into 32 sub-sequences that find each other by VLC self-synchronisation.  Streams from
// encoders that start a slice in every macroblock row (the classic MPEG-1 layout: 45 slices of a few hundred
// bytes in a 720p picture) defeat that: each slice is too short to cut, so the walk takes the slices one after
// the other with one or two lanes busy: such pictures took several times longer per picture than one-slice
// pictures of the same size.
//
// But slices are the unit the syntax makes independent: every predictor is reset in the slice header
// (src/mpeg1.js:255-266) and the address comes from the slice's start code.  So here lane i of the picture's warp
// walks slice i (then i + 32, ...) ALONE, from the true state, with the storing pass of the lane-parallel walk
// (walk_owned<WALK_ABS>: warp-synchronous lock-step loops, records and parked pairs written by the lane) -- no
// warm-up, no relative records, no composition.  The host's sorted list of start-code prefixes (ParseTask::codes)
// says where the slices are.
//
// Serial semantics (mpeg1.js:198-213: slices are decoded in stream order, a later one may overwrite an earlier
// one) are kept by construction inside the CLEAN DOMAIN and by falling back outside it: every slice must end
// exactly at the next prefix, and the address ranges of consecutive slices must be strictly increasing; anything
// else -- an invalid code, an address outside the picture, overlapping or backward slices, a picture without
// the host's list -- makes the warp walk the whole picture again with the serial walk (walk_picture<false>),
// which alone defines the behaviour there.  info.reserved[0] = 2 marks a picture walked this way.
//
// Opt-in (batch option "slice_walk"): the host routes I/P pictures with at least SLICE_WALK_MIN_SLICES (common.cuh) slices to
// walk_pictures_slices_kernel (parse.cu).  Compiles for the host emulation like walk.cuh.
#pragma once
#include "walk.cuh"

namespace {

// the start code (fourth byte) behind prefix k of the host's list, or -1 when its four bytes are not inside the data:
// findNextStartCode (buffer.js:115-128) needs them there
__device__ __forceinline__ int code_at(const ParseTask &t, uint32_t k) {
	if (k >= t.n_codes) return -1;
	const uint32_t p = __ldg(t.codes + k);
	return p + 3u < t.es_len ? (int)t.es[p + 3u] : -1;
}

__device__ void walk_picture_slices(const ParseTask &t, uint32_t sbase, int lane, uint32_t ring) {
	const int mb_width = t.mb_width, mb_size = t.mb_size;
	for (int i = lane; i < mb_size; i += 32) reinterpret_cast<uint4 *>(t.hdr)[i] = make_uint4(0, 0, 0, 0);
	__syncwarp();

	BitReaderT<true> br;
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
	uint32_t end_bit = br.bitpos();
	bool clean = t.codes != nullptr;
	if (go && clean) {
		status = PIC_DECODED;
		// the first start code findNextStartCode sees from here, past extension / user data (mpeg1.js:198-201)
		const uint32_t from = (br.bitpos() + 7u) >> 3;
		uint32_t k = t.code_hint;
		while (k < t.n_codes && __ldg(t.codes + k) < from) k++;
		int code = code_at(t, k);
		while (code == 0xB5 || code == 0xB2) code = code_at(t, ++k);
		uint32_t n_slices = 0;
		while (true) {
			const int c = code_at(t, k + n_slices);
			if (c < 0x01 || c > 0xAF) break;
			n_slices++;
		}
		int prev_last = -1;  // last address of the slice before this round's first one
		for (uint32_t base = 0; base < n_slices && clean; base += 32u) {
			const bool owns = base + (uint32_t)lane < n_slices;
			const uint32_t ks = k + base + (uint32_t)lane;
			PictureState ls = ps;  // picture constants; the slice's own state below
			ls.n_present = ls.n_coded = ls.error = 0;
			ls.anomaly = false;
			uint32_t end_byte = t.es_len;
			if (owns) {
				const uint32_t p = __ldg(t.codes + ks);
				if (ks + 1u < t.n_codes) end_byte = __ldg(t.codes + ks + 1u);
				// slice header (mpeg1.js:255-266)
				br.seek_byte(p + 4u);
				ls.slice_begin = true;
				ls.mb_addr = ((int)t.es[p + 3u] - 1) * mb_width - 1;
				ls.mv_h = ls.mv_v = ls.mv_h_prev = ls.mv_v_prev = 0;
				ls.dc_y = ls.dc_b4 = ls.dc_b5 = 128;
				ls.qscale = (int)br.read(5);
				while (br.read(1)) br.consume(8);
			}
			uint32_t stop_pos = 0;
			const int how = walk_owned<WALK_ABS>(br, sbase, ls, t, mb_size, owns, 0xffffffffu, end_byte, lane, stop_pos);
			// every slice ended exactly at the next prefix, nothing odd on the way, and the address ranges go up
			bool bad = owns && (how != 1 || ls.anomaly || ls.error != 0 || ls.n_present <= 0);
			const int last = owns ? ls.mb_addr : 0x7fffffff;
			const int first = owns ? ls.mb_addr - ls.n_present + 1 : 0x7fffffff;
			int before = __shfl_up_sync(FULL_MASK, last, 1);
			if (lane == 0) before = prev_last;
			if (owns && first <= before) bad = true;
			if (__any_sync(FULL_MASK, bad)) { clean = false; break; }
			const unsigned owners = __ballot_sync(FULL_MASK, owns);
			prev_last = __shfl_sync(FULL_MASK, last, 31 - __clz((int)owners));
			int n_present = ls.n_present, n_coded = ls.n_coded;
			for (int d = 16; d > 0; d >>= 1) {
				n_present += __shfl_xor_sync(FULL_MASK, n_present, d);
				n_coded += __shfl_xor_sync(FULL_MASK, n_coded, d);
			}
			ps.n_present += n_present;
			ps.n_coded += n_coded;
		}
		// where decodePicture leaves the bit index (mpeg1.js:203-213): at the first start code that is no slice
		// (rewound to its prefix), or at the end of the data when there is none
		const int after = code_at(t, k + n_slices);
		end_bit = after >= 0 ? __ldg(t.codes + k + n_slices) * 8u : t.es_len * 8u;
	}
	if (go && !clean) {  // outside the clean domain: the serial walk defines the result (it starts the picture over)
		__syncwarp();
		walk_picture<false>(t, sbase, lane, 0u);
		return;
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
		info.error = 0;
		info.reserved[0] = go ? 2 : 0;
		info.reserved[1] = 0;
		info.reserved[2] = 0;
		*t.info = info;
	}
}

}  // namespace
