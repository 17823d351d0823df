// walk_b.cuh -- stage 1a for B pictures (sm_90a): the opt-in extension, SURVEY 8(f) rank 4.
//
// The reference skips B pictures (src/mpeg1.js:181-184) although it carries their macroblock-type table
// (MACROBLOCK_TYPE_B, mpeg1.js:1152-1175 -> VLC_MBTYPE_B, pinned by tests/test_vlc_tables.py).  With the batch
// option "decode_b" the host routes every picture whose header says type 3 to walk_pictures_b_kernel
// (parse.cu) instead of the I/P walk.  The macroblock layer follows ISO/IEC 11172-2 2.4.3.6 with the
// reference's own building blocks -- the same bit reader, address-increment rules (mpeg1.js:294-346), vector
// arithmetic (mpeg1.js:395-457, once per direction with that direction's f_code), block walk and slice loop
// (mpeg1.js:255-276) -- and differs from a P picture in exactly these points:
//   * macroblock_type comes from table B.2d; 0x08 = forward vector follows, 0x04 = backward vector follows
//   * a direction that a macroblock does not use KEEPS its predictor (a P macroblock without vector resets it,
//     mpeg1.js:452-456); an intra macroblock resets both, a slice start too
//   * skipped macroblocks repeat the prediction (directions and vectors) of the macroblock before them and reset
//     only the DC predictors (ISO 11172-2 2.4.4.2; a P picture resets the vector, mpeg1.js:330-333)
// The record carries the directions in MBF_MOTION_FWD / MBF_MOTION_BWD and the backward vector in mv_bwd
// (records.h); stage 1b is unchanged, stage 2 is reconstruct_b_kernel.
//
// One warp per picture, all lanes on one chain, lane 0 stores: the serial walk.  (The lane-parallel walk's
// relative records would need the pair of vectors and the inherited directions composed as well; B pictures
// are the small pictures of a stream.)  Included by parse.cu after walk.cuh; compiles for the host emulation
// like walk.cuh (tests/emu/walk_emu.cpp).
#pragma once
#include "walk.cuh"

namespace {

struct BState {
	int full_pel, r_size, f;  // backward_f_code (ISO 11172-2 2.4.2.5)
	int mv_h, mv_v, mv_h_prev, mv_v_prev;
	int last_motion;  // MBF_MOTION_* of the macroblock before (what a skipped one repeats)
};

// mpeg1.js:395-457, one component, with the direction's own f / r_size / full_pel
template <class BR>
__device__ __forceinline__ bool parse_motion_dir(BR &br, uint32_t sbase, int f, int r_size, int full_pel, int &prev, int &mv) {
	const uint32_t e = clz_lut(sbase + OFF_MOTION, br.peek32(), VLC_MOTION_MAX_Z);
	const int len = e & 31;
	if (len == 0) return false;
	br.consume(len);
	const int code = (int)(e >> 5) - 16;
	int d = code;
	if (code != 0 && f != 1) {
		const int r = (int)br.read(r_size);
		d = ((abs(code) - 1) << r_size) + r + 1;
		if (code < 0) d = -d;
	}
	prev += d;
	if (prev > (f << 4) - 1) prev -= f << 5;
	else if (prev < -(f << 4)) prev += f << 5;
	mv = full_pel ? prev * 2 : prev;
	return true;
}

// the record of a predicted macroblock of a B picture; a vector that is not used is stored as zero
__device__ __forceinline__ uint4 pack_record_b(const PictureState &ps, const BState &bs, int motion, int flags, int cbp, int dc_only, uint32_t bit_pos) {
	const bool fwd = motion & MBF_MOTION_FWD, bwd = motion & MBF_MOTION_BWD;
	uint4 r = pack_record(fwd ? ps.mv_h : 0, fwd ? ps.mv_v : 0, flags | motion, cbp, dc_only, ps.qscale, bit_pos);
	r.w = bwd ? (((uint32_t)bs.mv_h & 0xffffu) | ((uint32_t)bs.mv_v << 16)) : 0u;
	return r;
}

// One macroblock of a B picture.  false = stop walking this slice.
template <class BR>
__device__ bool walk_macroblock_b(BR &br, uint32_t sbase, PictureState &ps, BState &bs, const ParseTask &t, int mb_size, int lane) {
	int increment = 0;
	int v = read_mba(br, sbase);
	while (v == 34) v = read_mba(br, sbase);                       // macroblock_stuffing
	while (v == 35) { increment += 33; v = read_mba(br, sbase); }  // macroblock_escape
	if (v < 0) return false;
	increment += v;

	if (ps.slice_begin) {  // mpeg1.js:312-317
		ps.slice_begin = false;
		ps.mb_addr += increment;
	} else {
		if (ps.mb_addr + increment >= mb_size) return true;  // mpeg1.js:319-322
		if (increment > 1) {
			ps.dc_y = ps.dc_b4 = ps.dc_b5 = 128;  // the vectors stay (ISO 11172-2 2.4.4.2)
			const int n_skip = increment - 1;
			const uint4 rec = pack_record_b(ps, bs, bs.last_motion, MBF_PRESENT | MBF_SKIPPED, 0, 0, br.bitpos());
			__syncwarp();  // (the order of the lanes' stores against lane 0's records: see walk_mb_header)
			for (int k = lane; k < n_skip; k += 32) reinterpret_cast<uint4 *>(t.hdr)[ps.mb_addr + 1 + k] = rec;
			__syncwarp();
			ps.n_present += n_skip;
			ps.mb_addr += n_skip;
		}
		ps.mb_addr++;
	}
	const int mb = ps.mb_addr;
	if (mb < 0 || mb >= mb_size) return false;  // outside the picture: never write there

	const uint32_t e = __ldg(&VLC_MBTYPE_B[br.peek32() >> 26]);
	if ((e & 31) == 0) return false;
	br.consume(e & 31);
	const int type = e >> 5;
	const bool intra = type & 0x01;
	if (type & 0x10) ps.qscale = (int)br.read(5);
	const uint32_t bit_pos = br.bitpos();

	if (intra) {
		ps.mv_h = ps.mv_v = ps.mv_h_prev = ps.mv_v_prev = 0;
		bs.mv_h = bs.mv_v = bs.mv_h_prev = bs.mv_v_prev = 0;
		// (a skipped macroblock must not follow an intra one; a stream that does it anyway gets a forward
		// prediction with the reset, i.e. zero, vector -- the same rule as the oracle's)
		bs.last_motion = MBF_MOTION_FWD;
	} else {
		ps.dc_y = ps.dc_b4 = ps.dc_b5 = 128;
		if (type & 0x08) {
			if (!parse_motion_dir(br, sbase, ps.f, ps.r_size, ps.full_pel, ps.mv_h_prev, ps.mv_h)) return false;
			if (!parse_motion_dir(br, sbase, ps.f, ps.r_size, ps.full_pel, ps.mv_v_prev, ps.mv_v)) return false;
		}
		if (type & 0x04) {
			if (!parse_motion_dir(br, sbase, bs.f, bs.r_size, bs.full_pel, bs.mv_h_prev, bs.mv_h)) return false;
			if (!parse_motion_dir(br, sbase, bs.f, bs.r_size, bs.full_pel, bs.mv_v_prev, bs.mv_v)) return false;
		}
		bs.last_motion = ((type & 0x08) ? MBF_MOTION_FWD : 0) | ((type & 0x04) ? MBF_MOTION_BWD : 0);
	}

	int cbp = intra ? 0x3f : 0;
	if (type & 0x02) {
		const uint32_t ce = clz_lut(sbase + OFF_CBP, br.peek32(), VLC_CBP_MAX_Z);
		if ((ce & 31) == 0) return false;
		br.consume(ce & 31);
		cbp = ce >> 5;
	}

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
		reinterpret_cast<uint4 *>(t.hdr)[mb] = intra ? pack_record(0, 0, MBF_PRESENT | MBF_INTRA, done, dc_mask, ps.qscale, bit_pos)
		                                             : pack_record_b(ps, bs, bs.last_motion, MBF_PRESENT, done, dc_mask, bit_pos);
	ps.n_present++;
	return ok;
}

// decodePicture (mpeg1.js:174-247), bitstream side, for a picture the host found to be of type 3.  Any other
// type is walked like walk_picture<false> does (so a mis-routed picture is still right).
__device__ void walk_picture_b(const ParseTask &t, uint32_t sbase, int lane) {
	const int mb_width = t.mb_width, mb_size = t.mb_size;
	for (int i = lane; i < mb_size; i += 32) reinterpret_cast<uint4 *>(t.hdr)[i] = make_uint4(0, 0, 0, 0);
	__syncwarp();

	BitReader br;
	br.words = reinterpret_cast<const uint32_t *>(t.es);
	br.bytes = t.es;
	br.len = t.es_len;
	br.ring = 0;
	br.seek_byte(t.start_byte);

	PictureState ps;
	ps.n_present = ps.n_coded = ps.error = 0;
	ps.n_fixup = 0;
	ps.full_pel = 0; ps.r_size = 0; ps.f = 1;
	ps.qs_set = ps.dc_abs = ps.mv_abs = ps.anomaly = false;
	BState bs;
	bs.full_pel = 0; bs.r_size = 0; bs.f = 1;
	bs.mv_h = bs.mv_v = bs.mv_h_prev = bs.mv_v_prev = 0;
	bs.last_motion = MBF_MOTION_FWD;
	int f_code = 0, f_code_b = 0;
	int status = PIC_IGNORED;

	br.consume(10);
	ps.picture_type = (int)br.read(3);
	br.consume(16);
	bool go = ps.picture_type >= 1 && ps.picture_type <= 3;
	if (ps.picture_type == 2 || ps.picture_type == 3) {
		ps.full_pel = (int)br.read(1);
		f_code = (int)br.read(3);
		if (f_code == 0) go = false;
		else { ps.r_size = f_code - 1; ps.f = 1 << ps.r_size; }
	}
	if (go && ps.picture_type == 3) {
		bs.full_pel = (int)br.read(1);
		f_code_b = (int)br.read(3);
		if (f_code_b == 0) go = false;
		else { bs.r_size = f_code_b - 1; bs.f = 1 << bs.r_size; }
	}
	uint32_t end_bit;
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
			bs.mv_h = bs.mv_v = bs.mv_h_prev = bs.mv_v_prev = 0;
			bs.last_motion = MBF_MOTION_FWD;
			ps.dc_y = ps.dc_b4 = ps.dc_b5 = 128;
			ps.qscale = (int)br.read(5);
			while (br.read(1)) br.consume(8);
			do {
				const bool ok = ps.picture_type == 3 ? walk_macroblock_b(br, sbase, ps, bs, t, mb_size, lane)
				                                     : walk_macroblock(br, sbase, ps, t, mb_size, lane);
				if (!ok) {
					if (!ps.error) ps.error = PARSE_ERR_INVALID_VLC;
					break;
				}
			} while (!br.next_bytes_are_start_code());
			code = br.find_next_start_code();
		}
		end_bit = br.bitpos();
		if (code != -1) end_bit -= 32;  // mpeg1.js:209-213
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
		info.reserved[0] = 0;
		info.reserved[1] = ps.picture_type == 3 ? (bs.full_pel << 4 | f_code_b) : 0;
		info.reserved[2] = 0;
		*t.info = info;
	}
}

}  // namespace
