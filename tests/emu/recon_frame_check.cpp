// recon_frame_check.cpp -- TEST INFRASTRUCTURE, not part of the product library.
//
// compact_emu.cpp (the host emulation of walk, expand and reconstruct) plus stage 2's decode_frames variant
// (reconstruct_at<..., FRAME = true>, jsmpeg_b200/csrc/recon.cuh, DESIGN 3.16): the same reconstruction, each block also
// storing its output rows to a planar frame.  tests/test_recon_frame_emu.py drives it against the plain and RES paths.
// Build: g++ -O2 -std=c++17 -shared -fPIC -pthread -I/usr/local/cuda/include.
#include "compact_emu.cpp"

static ReconFrameParamsT<CompactTaskB, 1> frame_params;
static bool frame_bidir, frame_on;
static uint8_t frame_wstage[WARP_STAGE];
static int frame_first_slot, frame_mb_row, frame_first_col, frame_warp;
static uint2 *frame_rows_out;

template <bool FRAME>
static void rgba_lane(int lane) {
	// reconstruct_rgba_block's numbering (the RGBA kernel's three warps of 16 macroblocks), up to the rows it hands its
	// epilogue: those go to frame_rows_out, 8 per block, [mb][b]
	const auto &t = frame_params.t[0];
	int b, local;
	if (frame_warp < 2) { b = frame_warp * 2 + (lane & 1); local = lane >> 1; }
	else { b = 4 + (lane >> 4); local = lane & 15; }
	const int mb_col = frame_first_col + local;
	const bool in_picture = mb_col < t.mb_width && frame_mb_row < t.mb_height;
	uint2 rows[8];
	for (int r = 0; r < 8; r++) rows[r] = make_uint2(0u, 0u);
	if (frame_bidir) reconstruct_at<true, true, true, FRAME>(frame_params, 0, frame_mb_row, in_picture ? mb_col : 0, b, in_picture, lane, frame_wstage, rows);
	else reconstruct_at<true, false, true, FRAME>(frame_params, 0, frame_mb_row, in_picture ? mb_col : 0, b, in_picture, lane, frame_wstage, rows);
	if (in_picture) memcpy(frame_rows_out + ((size_t)(frame_mb_row * t.mb_width + mb_col) * 6 + b) * 8, rows, sizeof(rows));
}

// Stage 2 as emu_reconstruct_picture_compact, through the FRAME variant (frame_on) or the RES variant (!frame_on) with
// the residual into `res` and the planar frame into `frame` (either may be nullptr).  rows_out == nullptr: the plain
// kernel's numbering (reconstruct_block); else the RGBA kernel's (KEEP), its rows into rows_out (mb_size * 6 * 8 uint2).
extern "C" int emu_reconstruct_picture_frame(const mb_record_t *hdr, const int16_t *coef, const coef_record_t *compact,
                                             uint8_t *cur, const uint8_t *fwd, const uint8_t *bwd, int mb_width, int mb_height,
                                             int16_t *res, uint8_t *frame, int use_frame_variant, uint2 *rows_out) {
	CompactTaskB &task = frame_params.t[0];
	task.hdr = hdr; task.coef = coef; task.compact = compact; task.cur = cur; task.fwd = fwd; task.bwd = bwd;
	task.mb_width = mb_width; task.mb_height = mb_height;
	task.row_magic = (uint32_t)(0x100000000ull / (uint64_t)(6 * mb_width)) + 1u;
	task.flags = 0;
	frame_params.n_tasks = 1;
	frame_params.res[0] = res;
	frame_params.frame[0] = frame;
	frame_bidir = bwd != nullptr;
	frame_on = use_frame_variant != 0;
	if (!rows_out) {
		const int slots = mb_width * mb_height * 6;
		for (frame_first_slot = 0; frame_first_slot < slots; frame_first_slot += 32)
			run_warp([](int l) {
				if (frame_on) {
					if (frame_bidir) reconstruct_block<true, true, true>(frame_params, 0, frame_first_slot, l, frame_wstage);
					else reconstruct_block<false, true, true>(frame_params, 0, frame_first_slot, l, frame_wstage);
				} else {
					if (frame_bidir) reconstruct_block<true, true>(frame_params, 0, frame_first_slot, l, frame_wstage);
					else reconstruct_block<false, true>(frame_params, 0, frame_first_slot, l, frame_wstage);
				}
			});
		return 0;
	}
	frame_rows_out = rows_out;
	for (frame_mb_row = 0; frame_mb_row < mb_height; frame_mb_row++)
		for (frame_first_col = 0; frame_first_col < mb_width; frame_first_col += 16)
			for (frame_warp = 0; frame_warp < 3; frame_warp++)
				run_warp(frame_on ? rgba_lane<true> : rgba_lane<false>);
	return 0;
}
