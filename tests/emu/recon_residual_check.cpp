// recon_residual_check.cpp -- TEST INFRASTRUCTURE, not part of the product library.
//
// compact_emu.cpp (the host emulation of walk, expand and reconstruct) plus stage 2's OUT_RESIDUALS variant
// (reconstruct_block<..., RES = true>, jsmpeg_b200/csrc/recon.cuh, DESIGN 3.15): the same reconstruction, each block
// also storing its residual.  tests/test_recon_residual_emu.py drives it against the plain path and the numpy transform.
// Build: g++ -O2 -std=c++17 -shared -fPIC -pthread -I/usr/local/cuda/include.
#include "compact_emu.cpp"

// Stage 2 as emu_reconstruct_picture_compact, through the RES variant with the residual into `res` (coded_size * 3 / 2
// int16 in the planes' layout); res == nullptr: the RES variant with no residual task (it must store nothing).
extern "C" int emu_reconstruct_picture_res(const mb_record_t *hdr, const int16_t *coef, const coef_record_t *compact,
                                           uint8_t *cur, const uint8_t *fwd, const uint8_t *bwd, int mb_width, int mb_height,
                                           int16_t *res) {
	static ReconResParamsT<CompactTaskB, 1> params;
	static int first_slot;
	static bool bidir;
	static uint8_t wstage[WARP_STAGE];
	CompactTaskB &task = params.t[0];
	task.hdr = hdr; task.coef = coef; task.compact = compact; task.cur = cur; task.fwd = fwd; task.bwd = bwd;
	task.mb_width = mb_width; task.mb_height = mb_height;
	task.row_magic = (uint32_t)(0x100000000ull / (uint64_t)(6 * mb_width)) + 1u;
	task.flags = 0;
	params.n_tasks = 1;
	params.res[0] = res;
	bidir = bwd != nullptr;
	const int slots = mb_width * mb_height * 6;
	for (first_slot = 0; first_slot < slots; first_slot += 32)
		run_warp([](int l) {
			if (bidir) reconstruct_block<true, true>(params, 0, first_slot, l, wstage);
			else reconstruct_block<false, true>(params, 0, first_slot, l, wstage);
		});
	return 0;
}
