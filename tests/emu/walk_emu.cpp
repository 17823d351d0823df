// walk_emu.cpp -- TEST INFRASTRUCTURE, not part of the product library.
//
// Compiles jsmpeg_b200/csrc/walk.cuh (the stage-1a walk, device code) for the HOST and runs one "warp"
// as 32 coroutines of one thread: the warp collectives become barrier + exchange, shared memory becomes a static
// array.  tests/test_walk_emu.py uses it to check, on machines without a GPU, that the lane-parallel
// walk produces exactly the records of the serial walk (the GPU parity tests then check both against
// the oracle).  Build: g++ -O2 -std=c++17 -shared -fPIC -pthread -I/usr/local/cuda/include.
#define JSMPEG_WALK_EMU 1
#include <string.h>

#include <ucontext.h>

#include <algorithm>
#include <mutex>
#include <vector>

#include <cuda_runtime.h>  // vector types only

using std::max;
using std::min;

// ---- the 32 "lanes" are coroutines of one thread: a collective yields round-robin until all arrived
namespace emu {
static ucontext_t main_ctx, ctx[32];
static bool finished[32];
static int lane;  // the lane that is running
static int arrived = 0, generation = 0;
static uint64_t slots[32];

static void yield_to_next() {
	const int from = lane;
	int to = from;
	do { to = (to + 1) & 31; } while (finished[to] && to != from);
	if (to == from) return;
	lane = to;
	swapcontext(&ctx[from], &ctx[to]);
	lane = from;
}
struct Barrier {
	void wait() {
		const int gen = generation;
		if (++arrived == 32) {  // the last lane to arrive releases the others
			arrived = 0;
			generation++;
			return;
		}
		while (generation == gen) yield_to_next();
	}
};
static Barrier bar;

template <class T>
static T exchange(T v, int src) {
	uint64_t raw = 0;
	memcpy(&raw, &v, sizeof(T));
	slots[lane] = raw;
	bar.wait();
	T r;
	memcpy(&r, &slots[src & 31], sizeof(T));
	bar.wait();
	return r;
}
}  // namespace emu

// ---- the CUDA intrinsics walk.cuh uses
static inline void __syncwarp(unsigned = 0xffffffffu) { emu::bar.wait(); }
template <class T> static inline T __shfl_sync(unsigned, T v, int src) { return emu::exchange(v, src); }
template <class T> static inline T __shfl_up_sync(unsigned, T v, int d) { return emu::exchange(v, emu::lane - d >= 0 ? emu::lane - d : emu::lane); }
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int m) { return emu::exchange(v, emu::lane ^ m); }
template <class T> static inline T __shfl_down_sync(unsigned, T v, int d) { return emu::exchange(v, emu::lane + d < 32 ? emu::lane + d : emu::lane); }
static inline unsigned __ballot_sync(unsigned, int pred) {
	emu::slots[emu::lane] = pred ? 1 : 0;
	emu::bar.wait();
	unsigned r = 0;
	for (int l = 0; l < 32; l++) r |= (unsigned)emu::slots[l] << l;
	emu::bar.wait();
	return r;
}
static inline int __any_sync(unsigned m, int pred) { return __ballot_sync(m, pred) != 0; }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline uint32_t __byte_perm(uint32_t a, uint32_t b, uint32_t sel) {  // PRMT, default mode (selectors 0..7)
	const uint64_t ab = ((uint64_t)b << 32) | a;
	uint32_t r = 0;
	for (int i = 0; i < 4; i++) {
		const uint32_t k = (sel >> (4 * i)) & 15u;
		if (k > 7) abort();  // sign-replicating selectors are not used
		r |= (uint32_t)((ab >> (8 * k)) & 255u) << (8 * i);
	}
	return r;
}
static inline uint32_t __funnelshift_l(uint32_t lo, uint32_t hi, uint32_t sh) { return (uint32_t)((((((uint64_t)hi << 32) | lo) << (sh & 31u))) >> 32); }
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t sh) { return (uint32_t)((((uint64_t)hi << 32) | lo) >> (sh & 31u)); }
static inline int __dp2a_lo(int a, int b, int c) {  // c + a.lo16 * b.byte0 + a.hi16 * b.byte1 (all signed)
	return c + (int)(int16_t)(a & 0xffff) * (int)(int8_t)(b & 0xff) + (int)(int16_t)((uint32_t)a >> 16) * (int)(int8_t)((b >> 8) & 0xff);
}
template <class T> static inline T __ldg(const T *p) { return *p; }

// trips and participating lanes of the lock-step loops, per vote site (walk.cuh: WK_VOTE)
static uint64_t vote_trips[8], vote_lanes[8];
static inline int emu_vote(int site, int pred) {
	const unsigned m = __ballot_sync(0xffffffffu, pred);
	if (emu::lane == 0 && m) {
		vote_trips[site]++;
		vote_lanes[site] += __builtin_popcount(m);
	}
	return m != 0;
}
extern "C" void emu_vote_counters(uint64_t *trips, uint64_t *lanes, int reset) {
	for (int i = 0; i < 8; i++) {
		trips[i] = vote_trips[i];
		lanes[i] = vote_lanes[i];
		if (reset) vote_trips[i] = vote_lanes[i] = 0;
	}
}

#define VLC_TABLE_QUALIFIER static const
#include "../../jsmpeg_b200/csrc/walk.cuh"
#include "../../jsmpeg_b200/csrc/walk_b.cuh"
#include "../../jsmpeg_b200/csrc/walk_slices.cuh"
#include "../../jsmpeg_b200/csrc/recon.cuh"

// Runs `body(lane)` as the 32 lanes of one warp.  Every collective is executed by all 32 lanes (the
// device code's rule), so no lane finishes while another still waits in one: a finished lane is simply
// skipped by the round-robin.
static void (*warp_body)(int);
static void warp_entry() {
	const int l = emu::lane;
	warp_body(l);
	emu::finished[l] = true;
	for (int k = 0; k < 32; k++)
		if (!emu::finished[k]) {
			emu::lane = k;
			setcontext(&emu::ctx[k]);
		}
	setcontext(&emu::main_ctx);
}
static void run_warp(void (*body)(int)) {
	static std::vector<std::vector<char>> stacks(32, std::vector<char>(1 << 20));
	warp_body = body;
	emu::arrived = 0;
	for (int l = 0; l < 32; l++) {
		emu::finished[l] = false;
		getcontext(&emu::ctx[l]);
		emu::ctx[l].uc_stack.ss_sp = stacks[l].data();
		emu::ctx[l].uc_stack.ss_size = stacks[l].size();
		emu::ctx[l].uc_link = nullptr;
		makecontext(&emu::ctx[l], warp_entry, 0);
	}
	emu::lane = 0;
	swapcontext(&emu::main_ctx, &emu::ctx[0]);
}

// the stream's quantiser matrices (de-zigzagged, as in SeqParams); stage 1b reads them
static uint8_t emu_intra_q[64], emu_non_intra_q[64];
extern "C" void emu_set_quant(const uint8_t *intra_q, const uint8_t *non_intra_q) {
	memcpy(emu_intra_q, intra_q, 64);
	memcpy(emu_non_intra_q, non_intra_q, 64);
}

// park: [mb_size][6] x {bit offset, intra dc (clamped, records.h)}, the walk's dense hand-over to stage 1b.
// lanes: 0 serial walk, 1 lane-parallel walk with its staging area (stage_entries_for(mb_size) entries, the
// product's size), 2 lane-parallel walk with a staging area of 40 entries (lanes run out: second-pass
// fall-back), 3 lane-parallel walk without staging area (always the second pass), 4 the slice walk (walk_slices.cuh:
// a lane per slice, serial fall-back).
extern "C" int emu_walk_picture(const uint8_t *es, uint32_t es_len, uint32_t start_byte, int mb_width, int mb_height,
                                mb_record_t *hdr, uint2 *park, picture_info_t *info, int lanes) {
	static std::once_flag once;
	static std::vector<uint16_t> ms(MS_TABLE_ENTRIES);
	std::call_once(once, [] {
		build_ms_table(VLC_DCT_COEFF, ms.data());
		walk_tables_init(emu_smem, 0, 1, reinterpret_cast<const uint4 *>(ms.data()), true);
	});
	SeqParams seq;
	memset(&seq, 0, sizeof(seq));
	seq.mb_width = mb_width;
	seq.mb_height = mb_height;
	seq.mb_size = mb_width * mb_height;
	memcpy(seq.intra_q, emu_intra_q, 64);
	memcpy(seq.non_intra_q, emu_non_intra_q, 64);
	ParseTask t;
	t.es = es; t.es_len = es_len; t.start_byte = start_byte; t.seq = &seq; t.hdr = hdr; t.coef = nullptr; t.info = info;
	t.park = park; t.mb_width = mb_width; t.mb_size = seq.mb_size;
	// exact-size staging area on the heap (AddressSanitizer sees any entry outside it)
	const int entries = lanes == 1 ? stage_entries_for(seq.mb_size) : (lanes == 2 ? 40 : 0);
	std::vector<uint4> stage((size_t)entries * 4);
	t.stage = entries ? stage.data() : nullptr;
	t.stage_entries = entries;
	// the start-code prefix list the host hands the product's walk (engine.cu): every 00 00 01 with its three bytes inside
	// the data.  lanes == 3 walks without it (the in-kernel search).
	std::vector<uint32_t> codes;
	uint32_t hint = 0;
	for (uint32_t p = 0; p + 2 < es_len; p++)
		if (es[p] == 0 && es[p + 1] == 0 && es[p + 2] == 1) {
			if (p + 4 == start_byte) hint = (uint32_t)codes.size();
			codes.push_back(p);
		}
	t.codes = lanes == 3 ? nullptr : codes.data();
	t.n_codes = (uint32_t)codes.size();
	t.code_hint = hint;
	static ParseTask task;
	static int use_lanes;
	task = t;
	use_lanes = lanes;
	run_warp([](int l) {
		if (use_lanes == 4) walk_picture_slices(task, 0, l, 0);
		else if (use_lanes) walk_picture<true>(task, 0, l, 0);
		else walk_picture<false>(task, 0, l, 0);
	});
	return 0;
}

// The B-picture walk (jsmpeg_b200/csrc/walk_b.cuh, the opt-in extension): one warp, all lanes on one chain.
extern "C" int emu_walk_picture_b(const uint8_t *es, uint32_t es_len, uint32_t start_byte, int mb_width, int mb_height,
                                  mb_record_t *hdr, uint2 *park, picture_info_t *info) {
	static std::once_flag once;
	static std::vector<uint16_t> ms(MS_TABLE_ENTRIES);
	std::call_once(once, [] {
		build_ms_table(VLC_DCT_COEFF, ms.data());
		walk_tables_init(emu_smem, 0, 1, reinterpret_cast<const uint4 *>(ms.data()), true);
	});
	static ParseTask task;
	memset(&task, 0, sizeof(task));
	task.es = es; task.es_len = es_len; task.start_byte = start_byte; task.hdr = hdr; task.info = info;
	task.park = park; task.mb_width = mb_width; task.mb_size = mb_width * mb_height;
	run_warp([](int l) { walk_picture_b(task, 0, l); });
	return 0;
}

// Stage 1b on the records the walk left: every block slot of the picture through expand_block
// (jsmpeg_b200/csrc/walk.cuh), one "thread" after the other with its own zeroed tile.
extern "C" int emu_expand_picture(const uint8_t *es, uint32_t es_len, int mb_width, int mb_height,
                                  mb_record_t *hdr, const uint2 *park, int16_t *coef, picture_info_t *info) {
	if (info->status != PIC_DECODED) return 0;
	memcpy(emu_smem + EMU_EXPAND_BASE + EXP_OFF_DCT, VLC_DCT_EXPAND, sizeof(VLC_DCT_EXPAND));  // as the kernel shell stages them
	memcpy(emu_smem + EMU_EXPAND_BASE + EXP_OFF_TOP8, VLC_DCT_EXPAND_TOP8, sizeof(VLC_DCT_EXPAND_TOP8));
	SeqParams seq;
	memset(&seq, 0, sizeof(seq));
	seq.mb_width = mb_width;
	seq.mb_height = mb_height;
	seq.mb_size = mb_width * mb_height;
	memcpy(seq.intra_q, emu_intra_q, 64);
	memcpy(seq.non_intra_q, emu_non_intra_q, 64);
	seq_fill_xq(seq);  // the host helper the product uses (common.cuh)
	memcpy(emu_smem + EMU_EXPAND_BASE + EXP_OFF_XQ, seq.xq, sizeof(seq.xq));
	ParseTask t;
	t.es = es; t.es_len = es_len; t.start_byte = 0; t.seq = &seq; t.hdr = hdr; t.coef = coef; t.info = info;
	t.park = const_cast<uint2 *>(park); t.mb_width = mb_width; t.mb_size = seq.mb_size;
	t.stage = nullptr; t.stage_entries = 0;
	t.codes = nullptr; t.n_codes = 0; t.code_hint = 0;
	for (int slot_id = 0; slot_id < seq.mb_size * 6; slot_id++) {  // the kernel shell of parse.cu, one thread after the other
		const int mb = slot_id / 6, block = slot_id - mb * 6;
		const uint32_t rec = reinterpret_cast<const uint32_t *>(hdr + mb)[1];
		if (!(rec & MBF_PRESENT) || !((rec >> 8) & (0x20u >> block))) continue;
		memset(emu_smem + EMU_EXPAND_BASE + EXP_OFF_TILES, 0, 128);
		expand_block(t, rec, park[slot_id], reinterpret_cast<uint4 *>(coef) + (size_t)slot_id * 8, EMU_EXPAND_BASE,
		             EMU_EXPAND_BASE + EXP_OFF_TILES);
	}
	return 0;
}


// Stage 2: every block slot of the picture through reconstruct_block (jsmpeg_b200/csrc/recon.cuh), a
// warp of 32 consecutive slots at a time.  cur / fwd: Y | Cr | Cb contiguous, like the product's plane sets.
// Planes need mb_width * 16 + 64 readable bytes past their end, like the product's.
extern "C" int emu_reconstruct_picture(const mb_record_t *hdr, const int16_t *coef, uint8_t *cur, const uint8_t *fwd,
                                       int mb_width, int mb_height) {
	static ReconParams params;
	static int first_slot;
	static uint8_t wstage[WARP_STAGE];
	CompactTask &task = params.t[0];
	task.hdr = hdr; task.coef = coef; task.cur = cur; task.fwd = fwd; task.mb_width = mb_width; task.mb_height = mb_height;
	task.row_magic = (uint32_t)(0x100000000ull / (uint64_t)(6 * mb_width)) + 1u;  // as launch_reconstruct (recon.cu)
	task.flags = 0;
	params.n_tasks = 1;
	const int slots = mb_width * mb_height * 6;
	for (first_slot = 0; first_slot < slots; first_slot += 32)
		run_warp([](int l) { reconstruct_block(params, 0, first_slot, l, wstage); });
	return 0;
}

// Stage 2 of a B picture (reconstruct_block<true>): fwd = the older, bwd = the newer reference.
extern "C" int emu_reconstruct_picture_b(const mb_record_t *hdr, const int16_t *coef, uint8_t *cur, const uint8_t *fwd,
                                         const uint8_t *bwd, int mb_width, int mb_height) {
	static ReconParamsB params;
	static int first_slot;
	static uint8_t wstage[WARP_STAGE];
	CompactTaskB &task = params.t[0];
	task.hdr = hdr; task.coef = coef; task.cur = cur; task.fwd = fwd; task.bwd = bwd; task.mb_width = mb_width; task.mb_height = mb_height;
	task.row_magic = (uint32_t)(0x100000000ull / (uint64_t)(6 * mb_width)) + 1u;
	task.flags = 0;
	params.n_tasks = 1;
	const int slots = mb_width * mb_height * 6;
	for (first_slot = 0; first_slot < slots; first_slot += 32)
		run_warp([](int l) { reconstruct_block<true>(params, 0, first_slot, l, wstage); });
	return 0;
}

// Stage 1b's sign-magnitude dequantisation (dequant_sm, walk.cuh) against the reference's statements
// (src/mpeg1.js:794-807, src/wasm/mpeg1.c decode_block), every level an escape or a table code can carry
// (-256 included: the escape (128, 0)),
// every quantiser scale (0 included: a corrupt stream can carry it), every matrix entry, intra and not.
// Returns the number of mismatches; first_bad = {level, qs, Q, intra, got, want} of the first one.
extern "C" long emu_check_dequant(int *first_bad) {
	long bad = 0;
	for (int intra = 0; intra < 2; intra++)
		for (int qs = 0; qs < 32; qs++)
			for (int Q = 0; Q < 256; Q++)
				for (int lv = -256; lv <= 255; lv++) {
					int level = lv;  // the reference, statement for statement
					level <<= 1;
					if (!intra) level += (level < 0 ? -1 : 1);
					level = (level * qs * Q) >> 4;
					if ((level & 1) == 0) level -= level > 0 ? 1 : -1;
					if (level > 2047) level = 2047;
					else if (level < -2048) level = -2048;
					const int got = dequant_sm(2 * abs(lv) + (intra ? 0 : 1), lv < 0, qs, (uint32_t)Q << 8);
					if (got != level && bad++ == 0 && first_bad) {
						first_bad[0] = lv; first_bad[1] = qs; first_bad[2] = Q; first_bad[3] = intra; first_bad[4] = got; first_bad[5] = level;
					}
				}
	return bad;
}
