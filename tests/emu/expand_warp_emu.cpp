// expand_warp_emu.cpp -- TEST INFRASTRUCTURE, not part of the product library.
//
// The host emulation of compact_emu.cpp plus stage 1b as a WARP runs it (jsmpeg_b200/csrc/walk.cuh: expand_warp_run):
// 32 consecutive block slots as 32 coroutines, the lanes' compact rows in the warp's staging area, the warp's store of
// the rows to the compact plane, and the dense records of the blocks that do not fit.
// tests/test_expand_code_order.py drives it.  Build: g++ -O2 -std=c++17 -shared -fPIC -pthread -I/usr/local/cuda/include.
#include "compact_emu.cpp"

// Every block slot of the picture, a warp of 32 consecutive slots at a time, as the kernel shell of parse.cu runs
// them.  compact: mb_size * 6 records, or nullptr (a task without a compact plane: dense records only).
extern "C" int emu_expand_picture_warps(const uint8_t *es, uint32_t es_len, int mb_width, int mb_height, const mb_record_t *hdr,
                                        const uint2 *park, int16_t *coef, coef_record_t *compact, const picture_info_t *info) {
	if (info->status != PIC_DECODED) return 0;
	memcpy(emu_smem + EMU_EXPAND_BASE + EXP_OFF_DCT, VLC_DCT_EXPAND, sizeof(VLC_DCT_EXPAND));
	memcpy(emu_smem + EMU_EXPAND_BASE + EXP_OFF_TOP8, VLC_DCT_EXPAND_TOP8, sizeof(VLC_DCT_EXPAND_TOP8));
	static SeqParams seq;
	memset(&seq, 0, sizeof(seq));
	seq.mb_width = mb_width;
	seq.mb_height = mb_height;
	seq.mb_size = mb_width * mb_height;
	memcpy(seq.intra_q, emu_intra_q, 64);
	memcpy(seq.non_intra_q, emu_non_intra_q, 64);
	seq_fill_xq(seq);
	memcpy(emu_smem + EMU_EXPAND_BASE + EXP_OFF_XQ, seq.xq, sizeof(seq.xq));
	static ParseTask task;
	static int first_slot;
	memset(&task, 0, sizeof(task));
	task.es = es; task.es_len = es_len; task.seq = &seq; task.hdr = const_cast<mb_record_t *>(hdr); task.coef = coef;
	task.park = const_cast<uint2 *>(park); task.mb_width = mb_width; task.mb_size = seq.mb_size;
	task.stage = reinterpret_cast<uint4 *>(compact);
	static_assert(EMU_EXPAND_BASE + EXP_OFF_TILES + 32 * EXP_TILE_PITCH <= sizeof(emu_smem), "one warp's staging area fits");
	for (first_slot = 0; first_slot < seq.mb_size * 6; first_slot += 32)
		run_warp([](int l) {
			const int slot_id = first_slot + l, n_slots = task.mb_size * 6;
			uint32_t rec = 0;
			uint2 parked = make_uint2(0u, 0u);
			if (slot_id < n_slots) {
				rec = reinterpret_cast<const uint32_t *>(task.hdr + slot_id / 6)[1];
				parked = task.park[slot_id];
			}
			const bool coded = slot_id < n_slots && (rec & MBF_PRESENT) && ((rec >> 8) & (0x20u >> (slot_id % 6)));
			expand_warp_run(task, coded, rec, parked, slot_id, l, EMU_EXPAND_BASE, EMU_EXPAND_BASE + EXP_OFF_TILES);
		});
	return 0;
}
