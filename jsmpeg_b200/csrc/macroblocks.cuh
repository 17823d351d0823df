// macroblocks.cuh -- the one place that knows both the walks' macroblock record (records.h: mb_record_t) and the
// public per-macroblock layout of jsmpeg_b200_batch_decode_macroblocks (include/jsmpeg_b200.h:
// jsmpeg_b200_macroblock_t).  Kept apart so that the host compiler can build it too
// (tests/emu/macroblocks_check.cpp checks it against the Python model, tools/macroblock_model.py).
#pragma once
#include <stdint.h>

#include "../../include/jsmpeg_b200.h"
#include "records.h"

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

static_assert(sizeof(mb_record_t) == 16 && sizeof(jsmpeg_b200_macroblock_t) == 16, "one 16-byte load, one 16-byte store");

// The public entry of record `r` of a picture of picture_coding_type `picture_type` (1 I, 2 P, 3 B).  In I and P
// records both motion bits are 0 and a non-intra macroblock predicts from the forward picture (with mv_h / mv_v, 0
// when the macroblock has no motion): its entry says FORWARD.  A vector whose direction flag is clear is 0.
__host__ __device__ inline jsmpeg_b200_macroblock_t export_macroblock(const mb_record_t &r, int picture_type) {
	jsmpeg_b200_macroblock_t m = {};
	if (!(r.flags & MBF_PRESENT)) return m;
	uint8_t flags = JSMPEG_B200_MB_PRESENT;
	if (r.flags & MBF_SKIPPED) flags |= JSMPEG_B200_MB_SKIPPED;
	if (r.flags & MBF_INTRA) {
		flags |= JSMPEG_B200_MB_INTRA;
	} else if (picture_type == 3) {
		if (r.flags & MBF_MOTION_FWD) flags |= JSMPEG_B200_MB_FORWARD;
		if (r.flags & MBF_MOTION_BWD) flags |= JSMPEG_B200_MB_BACKWARD;
	} else {
		flags |= JSMPEG_B200_MB_FORWARD;
	}
	if (flags & JSMPEG_B200_MB_FORWARD) {
		m.fwd_x = r.mv_h;
		m.fwd_y = r.mv_v;
	}
	if (flags & JSMPEG_B200_MB_BACKWARD) {
		m.bwd_x = (int16_t)(uint16_t)(r.mv_bwd & 0xffffu);
		m.bwd_y = (int16_t)(uint16_t)(r.mv_bwd >> 16);
	}
	m.flags = flags;
	m.cbp = r.cbp;
	m.qscale = r.qscale;
	return m;
}
