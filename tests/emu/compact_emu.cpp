// compact_emu.cpp -- TEST INFRASTRUCTURE, not part of the product library.
//
// The host emulation of walk_emu.cpp (one warp = 32 coroutines) plus entry points for the compact coefficient
// records (jsmpeg_b200/csrc/coef_records.h): the format's pack / unpack / zig-zag map as g++ compiles them, stage 1b
// writing compact records into a caller-given plane, and stage 2 reading them.  tests/test_compact_records.py
// drives it.  Build: g++ -O2 -std=c++17 -shared -fPIC -pthread -I/usr/local/cuda/include.
#include "walk_emu.cpp"

extern "C" int emu_coef_zigzag_raster(int k) { return coef_zigzag_raster(k); }

// returns 1 and the record when `written` fits one, else 0
extern "C" int emu_coef_pack(uint64_t written, const int16_t *raster, coef_record_t *out) {
	if (!coef_record_fits(written)) return 0;
	*out = coef_record_pack(written, raster);
	return 1;
}

extern "C" void emu_coef_unpack(const coef_record_t *r, int16_t *raster) { coef_record_unpack(*r, raster); }

extern "C" uint64_t emu_coef_nonzero_positions(const int16_t *raster) { return coef_nonzero_positions(raster); }

// Stage 1b as the product runs it when the picture has a staging area: every coded block slot through expand_block
// with its compact record at compact[slot] (compact: mb_size * 6 records); blocks that do not fit go to `coef`.
extern "C" int emu_expand_picture_compact(const uint8_t *es, uint32_t es_len, int mb_width, int mb_height, const mb_record_t *hdr,
                                          const uint2 *park, int16_t *coef, coef_record_t *compact, const picture_info_t *info) {
	if (info->status != PIC_DECODED) return 0;
	memcpy(emu_smem + EMU_EXPAND_BASE + EXP_OFF_DCT, VLC_DCT_EXPAND, sizeof(VLC_DCT_EXPAND));
	memcpy(emu_smem + EMU_EXPAND_BASE + EXP_OFF_TOP8, VLC_DCT_EXPAND_TOP8, sizeof(VLC_DCT_EXPAND_TOP8));
	SeqParams seq;
	memset(&seq, 0, sizeof(seq));
	seq.mb_width = mb_width;
	seq.mb_height = mb_height;
	seq.mb_size = mb_width * mb_height;
	memcpy(seq.intra_q, emu_intra_q, 64);
	memcpy(seq.non_intra_q, emu_non_intra_q, 64);
	seq_fill_xq(seq);
	memcpy(emu_smem + EMU_EXPAND_BASE + EXP_OFF_XQ, seq.xq, sizeof(seq.xq));
	ParseTask t;
	memset(&t, 0, sizeof(t));
	t.es = es; t.es_len = es_len; t.seq = &seq; t.coef = coef; t.mb_width = mb_width; t.mb_size = seq.mb_size;
	for (int slot_id = 0; slot_id < seq.mb_size * 6; slot_id++) {
		const int mb = slot_id / 6, block = slot_id - mb * 6;
		const uint32_t rec = reinterpret_cast<const uint32_t *>(hdr + mb)[1];
		if (!(rec & MBF_PRESENT) || !((rec >> 8) & (0x20u >> block))) continue;
		memset(emu_smem + EMU_EXPAND_BASE + EXP_OFF_TILES, 0, 128);
		expand_block(t, rec, park[slot_id], reinterpret_cast<uint4 *>(coef) + (size_t)slot_id * 8, EMU_EXPAND_BASE,
		             EMU_EXPAND_BASE + EXP_OFF_TILES, compact + slot_id);
	}
	return 0;
}

// Stage 2 reading compact records (compact != nullptr) and, for the blocks they mark dense, `coef`.  bwd != nullptr:
// a B picture (reconstruct_block<true>).
extern "C" int emu_reconstruct_picture_compact(const mb_record_t *hdr, const int16_t *coef, const coef_record_t *compact,
                                               uint8_t *cur, const uint8_t *fwd, const uint8_t *bwd, int mb_width, int mb_height) {
	static ReconParamsB params;
	static int first_slot;
	static bool bidir;
	static uint8_t wstage[WARP_STAGE];
	CompactTaskB &task = params.t[0];
	task.hdr = hdr; task.coef = coef; task.compact = compact; task.cur = cur; task.fwd = fwd; task.bwd = bwd;
	task.mb_width = mb_width; task.mb_height = mb_height;
	task.row_magic = (uint32_t)(0x100000000ull / (uint64_t)(6 * mb_width)) + 1u;
	task.flags = 0;
	params.n_tasks = 1;
	bidir = bwd != nullptr;
	const int slots = mb_width * mb_height * 6;
	for (first_slot = 0; first_slot < slots; first_slot += 32)
		run_warp([](int l) {
			if (bidir) reconstruct_block<true>(params, 0, first_slot, l, wstage);
			else reconstruct_block<false>(params, 0, first_slot, l, wstage);
		});
	return 0;
}
