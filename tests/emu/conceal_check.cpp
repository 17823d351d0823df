// conceal_check.cpp -- TEST INFRASTRUCTURE, not part of the product library.
//
// compact_emu.cpp (the host emulation of walk, expand and reconstruct) plus the conceal option's copy
// (conceal_macroblock, jsmpeg_b200/csrc/conceal.cuh, DESIGN 3.19), so that tests/test_conceal_oracle.py can run walk ->
// expand -> conceal -> reconstruct against the oracle with the rule (tools/conceal_model.py).
// Build: g++ -O2 -std=c++17 -shared -fPIC -pthread -I/usr/local/cuda/include.
#include "compact_emu.cpp"
#include "../../jsmpeg_b200/csrc/conceal.cuh"

// conceal_kernel's work for one picture: every lane of the warp of every macroblock, over the plane sets at `cur`
// and `fwd` (Y | Cr | Cb of mb_width x mb_height macroblocks).  Returns the macroblocks that lacked MBF_PRESENT.
extern "C" int emu_conceal_picture(const mb_record_t *hdr, uint8_t *cur, const uint8_t *fwd, int mb_width, int mb_height) {
	const int mb_size = mb_width * mb_height;
	const size_t ysize = (size_t)mb_size * 256;
	ConcealTask t;
	t.hdr = hdr;
	t.cur = PlaneSet{cur, cur + ysize, cur + ysize + ysize / 4};
	t.fwd = PlaneSet{const_cast<uint8_t *>(fwd), const_cast<uint8_t *>(fwd) + ysize, const_cast<uint8_t *>(fwd) + ysize + ysize / 4};
	t.mb_width = mb_width;
	t.mb_size = mb_size;
	t.first = 0;
	t.pad = 0;
	int absent = 0;
	for (int mb = 0; mb < mb_size; mb++) {
		for (int lane = 0; lane < 32; lane++) conceal_macroblock(t, mb, lane);
		absent += !(hdr[mb].flags & MBF_PRESENT);
	}
	return absent;
}
