// engine.cu -- host side of libjsmpeg_b200.so: stream state, HBM residency, wave planning, and
// the two C ABIs declared in include/jsmpeg_b200.h.
//
// What stays on the host is exactly what is bookkeeping in the reference too: the bit-buffer write
// protocol (src/wasm/buffer.c:48-71, 157-190; bitbuffer.h), the sequence header (src/mpeg1.js:78-153,
// parsed once per stream) and the decode() state machine (src/wasm/mpeg1.c:853-864, 947-995: which
// picture is next, where the bit index ends up, when planes swap).  All per-byte, per-bit and
// per-pixel work runs in the kernels (scan.cu, parse.cu, recon.cu).  There is no CPU fallback:
// without a usable CUDA device a decoder is created DEAD -- every entry point returns its failure
// value (decode() == false, like "no sequence header yet"), the reason is printed once and kept for
// jsmpeg_b200_batch_last_error.  Nothing here calls abort(): a plugin must not take its host process
// (a Node player) down.
//
// Wave model.  decode() on a stream needs (a) the next picture start code, (b) that picture's
// records, (c) its reconstruction from the previous picture.  (a) comes from the start-code index
// built when bytes become resident; (b) for MANY pictures (all streams x pictures ahead) is one
// parse wave, one warp per picture; (c) is one launch per picture STEP covering every stream
// that has a picture at that step.  The reference's serial semantics are re-established on the
// host after the parse: picture j+1 of a stream is accepted only if its start code is the first
// one at/after the bit index where picture j's parse ended (otherwise the look-ahead is discarded
// and re-planned from there).
//
// Pipeline.  decode() and decode_pictures / decode_intra share it.  A round plans its pictures, parses
// them in one stage-1 wave (parse_wave: walk + expand per walk kernel, the kernels beside each other on
// side streams) and waits for the picture infos; the host then consumes them in decode() order and
// queues one reconstruct step per picture depth (ReconStep, launch_reconstruct) on the reconstruct stream.
// Cutting the wave into chunks to overlap stage 1 with stage 2 was measured not to pay (DESIGN 8).
// decode_macroblocks runs the same waves walk-only (no expand, no reconstruct) and exports the records (DESIGN 3.8);
// decode_coefficients runs them with expand and exports the coefficients too (DESIGN 3.9), decode_residuals their
// inverse transform (DESIGN 3.10).  Each wave's exports are a stage-2 step without reconstruct tasks, queued by the
// same step runner (run_steps) on the reconstruct stream.
#include <sched.h>

#include <algorithm>
#include <chrono>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "bitbuffer.h"
#include "buffers.h"
#include "common.cuh"
#include "conceal.cuh"
#include "demux.h"
#include "psdemux.cuh"
#include "tsdemux.cuh"
#include "../../include/jsmpeg_b200.h"

namespace {

constexpr int HOST_RING = 4;
constexpr uint32_t ES_PAD = 512;  // readable, zeroed slack after the ES mirror (the walk's ring prefetches 64 bytes ahead)

// the bit buffer lives in pinned host memory (H2D copies of new bytes run at PCIe speed); bitbuffer.h owns it
// through these hooks
void *bb_pinned_alloc(size_t n, void *) { return PinnedAlloc::alloc(std::max<size_t>(n, 1)); }
void bb_pinned_release(void *p, void *) { PinnedAlloc::release(p); }
const bitbuffer::Allocator kPinned = {bb_pinned_alloc, bb_pinned_release, nullptr};

struct Parsed {
	uint32_t pos;           // byte position of the 00 00 01 00 start code
	uint32_t len_at_parse;  // buffer length the parse saw
	int slot;
	picture_info_t info;
};

// One plane set of a stream in HBM and what stage 2 writes beside it: the macroblock entries of its picture
// (OUT_MACROBLOCKS, DESIGN 3.13) and, on the I/P sets, its accumulated map (OUT_ACCUMULATED, DESIGN 3.14).  A picture's
// entries and map go where its planes go, so every ordering rule of the planes covers them.
struct StreamSet {
	DeviceBuffer<uint8_t> planes;
	DeviceBuffer<uint8_t> entries;  // made zeroed on first use (reserve_entries)
	DeviceBuffer<uint2> map;        // made on first use (reserve_maps)
	// a call with the flag wrote `map` for the picture `planes` holds now; an unwritten map is never read as a trace's
	// previous map
	bool map_written = false;
	// decode_frames_into (DESIGN 3.17): the map frame that holds that picture's map instead of `map`, while the call runs;
	// nullptr: `map`
	const uint2 *map_at = nullptr;
};

// One slot of a stream's host ring (OUT_HOST): a picture's planes and, under OUT_MACROBLOCKS, its entries (made zeroed on
// first use, reserve_entries)
struct HostSlot {
	PinnedBuffer<uint8_t> planes, entries;
};

// decode_frames_display (DESIGN 3.18): one frame of each kind of one stream -- where one picture's planes, RGBA,
// residual, entries, coefficients and map go (nullptr: that kind not at all)
struct FrameAt {
	uint8_t *planes = nullptr, *rgba = nullptr, *mb = nullptr;
	int16_t *res = nullptr, *coef = nullptr;
	uint2 *acc = nullptr;
};

// The kinds of frame, as bits of FrameStore::kinds and FrameCursor::kinds
enum : unsigned { KIND_PLANES = 1, KIND_RGBA = 2, KIND_RES = 4, KIND_MB = 8, KIND_COEF = 16, KIND_ACC = 32 };

// decode_frames_display: the I/P picture a stream holds back until its successor reference (or flush_frames) presents
// it, in a store of one frame per kind made on first use.  `kinds`: the kinds the holding call wrote into the store;
// `info`: the picture's frame info.
struct FrameStore {
	DeviceBuffer<uint8_t> planes, rgba, mb;
	DeviceBuffer<int16_t> res, coef;
	DeviceBuffer<uint2> acc;
	bool held = false;
	unsigned kinds = 0;
	jsmpeg_b200_frame_t info{};
};

struct Stream {
	bitbuffer::Buffer bb;  // host bit buffer (pinned) -- src/wasm/buffer.c
	// sequence header
	bool has_seq = false;
	float frame_rate = 0.f;
	int width = 0, height = 0, coded_size = 0;
	uint32_t seq_end_index = 0;  // bit index right after the sequence header
	uint32_t seq_floor = 0;      // byte position in the CURRENT buffer from which pictures follow the sequence header
	SeqParams seq{};
	DeviceBuffer<SeqParams> d_seq;
	// ES mirror in HBM + start-code index
	DeviceBuffer<uint8_t> d_es;
	uint32_t d_valid = 0;
	std::vector<uint32_t> pics;  // sorted byte positions of picture start codes (00 00 01 00)
	std::vector<uint32_t> codes, pic_code;  // every start-code prefix (00 00 01), sorted; pics[k] == codes[pic_code[k]]
	uint32_t codes_classified = 0;          // codes[0 .. codes_classified) have had their fourth byte looked at
	uint32_t scanned = 0;        // every prefix with pos + 2 < scanned is in `codes`
	uint32_t scan_from = 0;      // the span a pending scan covers starts here
	bool scan_pending = false;
	// plane sets: 0 and 1 the I/P ping-pong (mpeg1.js:221-246); 2 and 3 the B-picture extension's ("decode_b"), made on
	// the first B picture and written in turn -- a B picture is no reference, the ping-pong is untouched by it
	StreamSet sets[4];
	int cur = 0;    // I/P set written by the next I/P picture; forward = 1 - cur
	int b_cur = 0;  // set 2 + b_cur is written by the next B picture
	int last = 1;   // the set holding the most recently decoded picture (none yet: forward)
	HostSlot ring[HOST_RING];
	int h_head = -1;
	int last_type = 0, last_temporal = 0;  // picture_coding_type / temporal_reference of the last picture decode() consumed
	// residual (OUT_RESIDUALS, DESIGN 3.15): that of the newest picture a call with the flag reconstructed, stored by
	// stage 2 (ReconTask::res); made zeroed on first use (reserve_residuals)
	DeviceBuffer<int16_t> d_res;
	DeviceBuffer<uint8_t> d_rgba;
	DeviceBuffer<int16_t> ts_bound;    // device TS demux: the stream id every PID is bound to, 0 = none (ts.js pidsToStreamIds)
	std::vector<uint8_t> ts_leftover;  // ... and the bytes the last write_ts left over (ts.js leftoverBytes)
	std::vector<uint8_t> ps_leftover;  // device PS demux: the bytes the last write_ps left over
	bool ps_in_sync = false;           // ... and whether they continue the item chain (else: look for a pack header)
	// parsed-ahead pictures, consecutive, front = next picture decode() consumes
	std::deque<Parsed> cache;
	// decode_frames_display's held picture: dropped by reset, rewind, set_index, a seek and every other call that
	// reconstructs into the stream's sets (DESIGN 3.18)
	FrameStore hold;
};

struct ScratchDeleter {
	void operator()(TsScratch *s) const { ts_scratch_destroy(s); }
	void operator()(PsScratch *s) const { ps_scratch_destroy(s); }
};

}  // namespace

struct jsmpeg_b200_batch_t {
	int device = 0;
	bool dead = false;  // a CUDA call failed: every entry point returns its failure value from now on
	std::string error;
	std::vector<uint8_t> dead_scratch;  // where get_write_ptr points a caller's memcpy once dead
	std::vector<Stream> streams;
	// start-code scan of all streams in one launch (scan.cu): span list, per-span hit counts and positions;
	// and the device's copy of every stream's sorted prefix list (ParseTask::codes), one row per stream
	// (scan_seg(), codes_stride(): the row lengths)
	DeviceBuffer<ScanSpan> d_spans;
	PinnedBuffer<ScanSpan> h_spans;
	DeviceBuffer<uint32_t> d_scan_counts, d_scan_pos;
	PinnedBuffer<uint32_t> h_scan_counts, h_scan_pos;
	DeviceBuffer<uint32_t> d_codes;  // empty until the first list is staged: the walks then search slice ends themselves
	PinnedBuffer<uint32_t> h_codes;
	// uploads + scan + parse | reconstruct | copy-out | decode(): the infos' way to the host, behind the walks alone
	cudaStream_t st_main = nullptr, st_recon = nullptr, st_copy = nullptr, st_info = nullptr;
	cudaEvent_t ev_a = nullptr, ev_b = nullptr, ev_mid = nullptr, ev_step = nullptr, ev_round = nullptr, ev_copied[2] = {nullptr, nullptr};
	cudaEvent_t ev_recon[2] = {nullptr, nullptr};  // around a round's reconstruct launches (timing)
	cudaEvent_t ev_info = nullptr;  // decode(): the infos of a wave are on the host
	// record slots
	unsigned max_slots_req = 0;
	int slot_mb = 0, n_slots = 0;
	DeviceBuffer<mb_record_t> d_hdr;
	DeviceBuffer<int16_t> d_coef;
	DeviceBuffer<uint2> d_park;
	DeviceBuffer<uint4> d_stage;  // per slot: stage_entries_for(slot_mb) x 64 B (lane-parallel walk, relative records)
	DeviceBuffer<picture_info_t> d_info;
	PinnedBuffer<picture_info_t> h_info;
	std::vector<int> free_slots;
	int lookahead = 1;
	bool decode_b = false;       // the B-picture extension: off = B pictures are skipped like the reference does (mpeg1.js:181-184)
	bool slice_walk = false;     // I/P pictures of >= SLICE_WALK_MIN_SLICES slices go to the one-lane-per-slice walk (walk_slices.cuh)
	bool conceal = false;        // the macroblocks a decoded picture lacks are copied from its forward set (DESIGN 3.19)
	// pictures with a walk kernel of their own (B pictures; with "slice_walk", I/P pictures of many slices) are
	// walked beside the others, on these streams
	cudaStream_t st_side[2] = {nullptr, nullptr};
	cudaEvent_t ev_sfork = nullptr, ev_sjoin[2] = {nullptr, nullptr};
	bool recon_pending = false;  // reconstruct launches of an earlier round may still read record slots
	// parse task staging
	PinnedBuffer<ParseTask> h_ptasks;
	DeviceBuffer<ParseTask> d_ptasks;
	uint64_t copy_steps = 0;  // reconstruct launches with a copy-out so far (event parity)
	ParseFork fork{};
	bool batch_copy_ok = true;
	// write_ts_many / write_ps_many: each format's scratch and the per-call I/O (demux_many)
	std::unique_ptr<TsScratch, ScratchDeleter> ts;
	std::unique_ptr<PsScratch, ScratchDeleter> ps;
	TsIo ts_io;
	PsIo ps_io;
	// decode_pictures / decode_intra: the forward plane set a chain of one picture names, zeroed and never written
	// (DESIGN 3.6); and the pool of the other chains' plane sets, zeroed per chain group (DESIGN 3.7)
	DeviceBuffer<uint8_t> d_intra_fwd;
	DeviceBuffer<uint8_t> d_chain_sets;
	// the export and accumulate tasks of a call's steps (run_steps: a decode() round, a wave of the others), one table
	// per task type, read on st_recon: macroblock entries (decode_macroblocks, OUT_MACROBLOCKS and macroblock frames,
	// DESIGN 3.8, 3.13), coefficients (decode_coefficients and coefficient frames, DESIGN 3.9, 3.17), residuals
	// (decode_residuals, DESIGN 3.10) and accumulated maps (decode_accumulated and OUT_ACCUMULATED, DESIGN 3.11, 3.14)
	PinnedBuffer<MbExportTask> h_etasks;
	DeviceBuffer<MbExportTask> d_etasks;
	PinnedBuffer<CoefExportTask> h_ctasks;
	DeviceBuffer<CoefExportTask> d_ctasks;
	PinnedBuffer<ResExportTask> h_rtasks;
	DeviceBuffer<ResExportTask> d_rtasks;
	PinnedBuffer<AccTask> h_atasks;
	DeviceBuffer<AccTask> d_atasks;
	// the conceal option's copies (DESIGN 3.19), read on st_recon like the tables above
	PinnedBuffer<ConcealTask> h_ktasks;
	DeviceBuffer<ConcealTask> d_ktasks;
	// decode_accumulated: the pool of the chains' two scratch map sets (DESIGN 3.11)
	DeviceBuffer<uint8_t> d_map_sets;
	jsmpeg_b200_stats_t stats{};
	// JSMPEG_B200_HOST_TRACE=1: decode() prints where the host's time of the call went (tools/time_stages.py), in ms:
	// upload_all | planning the waves | building and queueing stage 1 | waiting for the infos | consuming them |
	// queueing stage 2 | the closing synchronises; and `device`, from the tasks' upload to the later of the last expand
	// and the last reconstruct launch
	struct HostTrace {
		bool on = false;
		double upload = 0, plan = 0, stage1 = 0, infos = 0, consume = 0, stage2 = 0, close = 0, device = 0;
	} trace;
};

namespace {

using Batch = jsmpeg_b200_batch_t;

void use_device(Batch *b) { CUDA_CHECK(cudaSetDevice(b->device)); }

// Adds the host time since `since` to `sum` (Batch::HostTrace) and restarts the clock
using HostClock = std::chrono::steady_clock;
void lap(double &sum, HostClock::time_point &since) {
	const HostClock::time_point now = HostClock::now();
	sum += std::chrono::duration<double, std::milli>(now - since).count();
	since = now;
}

void mark_dead(Batch *b, const char *what) {
	if (!b->dead) fprintf(stderr, "%s\njsmpeg_b200: decoder disabled (decode() returns false from now on)\n", what);
	b->dead = true;
	if (b->error.empty()) b->error = what;
}

// Every C-ABI entry point that touches CUDA runs through here.
template <typename R, typename F>
R guarded(Batch *b, R fail, F &&f) {
	if (!b || b->dead) return fail;
	try {
		return f();
	} catch (const std::exception &e) {
		mark_dead(b, e.what());
	} catch (...) {
		mark_dead(b, "jsmpeg_b200: unknown failure");
	}
	return fail;
}
template <typename F>
void guarded_void(Batch *b, F &&f) {
	guarded<int>(b, 0, [&] { f(); return 0; });
}

void release_slot(Batch *b, int slot) { b->free_slots.push_back(slot); }

void flush_cache(Batch *b, Stream &s) {
	for (auto &p : s.cache) release_slot(b, p.slot);
	s.cache.clear();
}

void forget_index(Batch *b, Stream &s) {
	flush_cache(b, s);
	s.pics.clear();
	s.codes.clear();
	s.pic_code.clear();
	s.codes_classified = 0;
	s.scanned = 0;
	s.d_valid = 0;
}

// ---- bit buffer (host) ------------------------------------------------------------------------

// src/wasm/buffer.c:48-65 get_write_ptr, :167-190 evict (bitbuffer.h)
void *stream_get_write_ptr(Batch *b, Stream &s, uint32_t n) {
	bool moved = false;
	const uint32_t old_length = s.bb.length;
	uint8_t *p = bitbuffer::get_write_ptr(s.bb, n, kPinned, moved);
	if (moved) {
		forget_index(b, s);  // byte positions changed: the HBM mirror, the index and the look-ahead are void
		const uint32_t dropped = old_length - s.bb.length;  // EVICT drops bytes from the front only
		s.seq_floor = s.seq_floor > dropped ? s.seq_floor - dropped : 0;
	}
	if (!p) throw std::runtime_error("jsmpeg_b200: bit buffer cannot hold the write (more than 4 GiB - 1 bytes)");
	return p;
}

// MSB-first reader for the headers the host reads itself (sequence header, picture headers); bytes beyond `len` read
// as 0, as they do to the walks
struct HostBits {
	const uint8_t *p;
	uint32_t len;
	uint64_t idx;
	uint32_t read(int n) {  // n <= 32
		uint32_t v = 0;
		while (n > 0) {  // the bits of one byte at a time
			const uint64_t byte = idx >> 3;
			const int left = 8 - (int)(idx & 7), take = n < left ? n : left;
			const uint32_t bits = byte < len ? p[byte] : 0u;
			v = v << take | ((bits >> (left - take)) & ((1u << take) - 1u));
			idx += take;
			n -= take;
		}
		return v;
	}
};

const float kPictureRate[16] = {0.f, 23.976f, 24.f, 25.f, 29.97f, 30.f, 50.f, 59.94f, 60.f, 0, 0, 0, 0, 0, 0, 0};
const uint8_t kZigZag[64] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22,
                             15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
const uint8_t kDefaultIntraQ[64] = {8, 16, 19, 22, 26, 27, 29, 34, 16, 16, 22, 24, 27, 29, 34, 37,
                                    19, 22, 26, 27, 29, 34, 34, 38, 22, 22, 26, 27, 29, 34, 37, 40,
                                    22, 26, 27, 29, 32, 35, 40, 48, 26, 27, 29, 32, 35, 40, 48, 58,
                                    26, 27, 29, 34, 38, 46, 56, 69, 27, 29, 35, 38, 46, 56, 69, 83};

// The planes of `set`, made zeroed on `st` (JS typed arrays start zeroed).  + coded_width + 64: stage 2's row loads may
// touch (never use) up to one row past a plane set's end.
void make_planes(const Stream &s, StreamSet &set, cudaStream_t st) {
	const size_t bytes = (size_t)s.coded_size * 3 / 2 + s.seq.coded_width + 64;
	set.planes.reserve(bytes);
	CUDA_CHECK(cudaMemsetAsync(set.planes.data(), 0, bytes, st));
}

// src/mpeg1.js:78-153 decodeSequenceHeader + initBuffers (first header only, mpeg1.c:812-819)
void parse_sequence_header(Batch *b, Stream &s, uint32_t bit_index) {
	HostBits hb{s.bb.bytes, s.bb.length, bit_index};
	s.width = (int)hb.read(12);
	s.height = (int)hb.read(12);
	hb.read(4);
	s.frame_rate = kPictureRate[hb.read(4)];
	hb.read(18 + 1 + 10 + 1);
	if (hb.read(1)) { for (int i = 0; i < 64; i++) s.seq.intra_q[kZigZag[i]] = (uint8_t)hb.read(8); }
	else memcpy(s.seq.intra_q, kDefaultIntraQ, 64);
	if (hb.read(1)) { for (int i = 0; i < 64; i++) s.seq.non_intra_q[kZigZag[i]] = (uint8_t)hb.read(8); }
	else memset(s.seq.non_intra_q, 16, 64);
	seq_fill_xq(s.seq);
	s.bb.index = (uint32_t)hb.idx;
	s.seq_end_index = (uint32_t)hb.idx;
	s.seq_floor = (uint32_t)((hb.idx + 7) >> 3);  // where decode() starts looking for the first picture
	s.seq.mb_width = (s.width + 15) >> 4;
	s.seq.mb_height = (s.height + 15) >> 4;
	s.seq.mb_size = s.seq.mb_width * s.seq.mb_height;
	s.seq.coded_width = s.seq.mb_width << 4;
	s.seq.coded_height = s.seq.mb_height << 4;
	s.coded_size = s.seq.coded_width * s.seq.coded_height;
	s.has_seq = true;

	const size_t plane_bytes = (size_t)s.coded_size * 3 / 2;
	s.d_seq.reserve(1);
	CUDA_CHECK(cudaMemcpyAsync(s.d_seq.data(), &s.seq, sizeof(SeqParams), cudaMemcpyHostToDevice, b->st_main));
	for (int i = 0; i < 2; i++) make_planes(s, s.sets[i], b->st_main);  // the I/P sets
	for (HostSlot &h : s.ring) {
		h.planes.reserve(plane_bytes);
		memset(h.planes.data(), 0, plane_bytes);
	}
	CUDA_CHECK(cudaStreamSynchronize(b->st_main));  // s.seq is read by the async copy
}

// src/wasm/mpeg1.c:812-819 did_write
void stream_did_write(Batch *b, Stream &s, uint32_t n) {
	if ((uint64_t)s.bb.length + n > s.bb.capacity) n = s.bb.capacity - s.bb.length;  // never beyond what get_write_ptr handed out
	s.bb.length += n;
	if (!s.has_seq) {
		// findStartCode(SEQUENCE): serial host scan of the not-yet-consumed head of the stream
		uint32_t i = (s.bb.index + 7) >> 3;
		bool found = false;
		for (; i + 3 < s.bb.length; i++) {
			if (s.bb.bytes[i] == 0 && s.bb.bytes[i + 1] == 0 && s.bb.bytes[i + 2] == 1) {
				if (s.bb.bytes[i + 3] == 0xB3) { found = true; break; }
				i += 3;  // index jumps past the code (buffer.js:121-123)
			}
		}
		if (found) parse_sequence_header(b, s, (i + 4) << 3);
		else s.bb.index = s.bb.length << 3;
	}
}

// ---- residency: H2D of new bytes + start-code scan -----------------------------------------------

// Room for `need` ES bytes (+ pad) in the HBM mirror; what is already resident stays resident.
void reserve_device_es(Batch *b, Stream &s, uint32_t need) {
	if ((uint64_t)need + ES_PAD <= s.d_es.size()) return;
	uint64_t cap = std::max<uint64_t>((uint64_t)need + ES_PAD, (uint64_t)s.d_es.size() * 2);
	cap = std::min<uint64_t>((cap + 255u) & ~255ull, 0xffffff00ull);
	DeviceBuffer<uint8_t> n(cap);
	if (s.d_es.data()) {
		if (s.d_valid) CUDA_CHECK(cudaMemcpyAsync(n.data(), s.d_es.data(), s.d_valid, cudaMemcpyDeviceToDevice, b->st_main));
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));
	}
	s.d_es = std::move(n);
}

// Positions per span of the scan buffers, entries per stream of the device's prefix lists
uint32_t scan_seg(const Batch *b) { return b->d_spans.size() ? (uint32_t)(b->d_scan_pos.size() / b->d_spans.size()) : 0; }
uint32_t codes_stride(const Batch *b) { return (uint32_t)(b->d_codes.size() / b->streams.size()); }

// Room for `rows` spans with `seg` positions each (contents are per scan: nothing to keep).
void reserve_scan(Batch *b, uint32_t rows, uint32_t seg) {
	const uint32_t have_rows = (uint32_t)b->d_spans.size(), have_seg = scan_seg(b);
	if (rows <= have_rows && seg <= have_seg) return;
	rows = std::max(rows, have_rows);
	seg = std::max(seg, have_seg);
	b->d_spans.reserve(rows);
	b->h_spans.reserve(rows);
	b->d_scan_counts.reserve(rows);
	b->h_scan_counts.reserve(rows);
	b->d_scan_pos.reserve((size_t)rows * seg);
	b->h_scan_pos.reserve((size_t)rows * seg);
}

// One launch over the pending spans (h_spans[0 .. n)); the counts come back to h_scan_counts.
void launch_scan(Batch *b, int n, uint32_t longest) {
	CUDA_CHECK(cudaMemcpyAsync(b->d_spans.data(), b->h_spans.data(), n * sizeof(ScanSpan), cudaMemcpyHostToDevice, b->st_main));
	CUDA_CHECK(cudaMemsetAsync(b->d_scan_counts.data(), 0, n * sizeof(uint32_t), b->st_main));
	launch_scan_start_codes(b->d_spans.data(), n, longest, b->d_scan_pos.data(), scan_seg(b), b->d_scan_counts.data(), b->st_main);
	b->stats.kernel_launches++;
	CUDA_CHECK(cudaMemcpyAsync(b->h_scan_counts.data(), b->d_scan_counts.data(), n * sizeof(uint32_t), cudaMemcpyDeviceToHost, b->st_main));
}

// The device's copy of every stream's prefix list: row si = streams[si].codes.  The host has them all, so a
// change of geometry (more streams, a longer list) just stages everything again.  Returns true if rebuilt.
bool reserve_codes(Batch *b, uint32_t entries) {
	if (b->d_codes.data() && entries <= codes_stride(b)) return false;
	const uint32_t stride = std::max<uint32_t>(std::max<uint32_t>(2 * codes_stride(b), entries + 256u), 1024u);
	if (b->d_codes.data()) {
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));  // (tasks of an earlier round may still name the old rows)
		CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
	}
	b->d_codes.reserve(b->streams.size() * stride);
	b->h_codes.reserve(b->streams.size() * stride);
	return true;
}

void begin_upload(Batch *b, Stream &s) {
	s.scan_pending = false;
	if (s.d_valid >= s.bb.length && s.scanned >= s.bb.length) return;
	reserve_device_es(b, s, s.bb.length);
	if (s.d_valid < s.bb.length) {
		uint32_t from = s.d_valid & ~15u;
		CUDA_CHECK(cudaMemcpyAsync(s.d_es.data() + from, s.bb.bytes + from, s.bb.length - from, cudaMemcpyHostToDevice, b->st_main));
		b->stats.h2d_bytes += s.bb.length - from;
		s.d_valid = s.bb.length;
		// the kernels rely on zeros right after the data (bytes past the end read as 0, like JS)
		CUDA_CHECK(cudaMemsetAsync(s.d_es.data() + s.bb.length, 0, ES_PAD, b->st_main));
	}
	if (s.scanned < s.bb.length) {
		s.scan_from = s.scanned >= 2 ? s.scanned - 2 : 0;  // a prefix needs its three bytes: those from scanned - 2 on were not complete
		s.scan_pending = true;  // (upload_all scans all pending spans in one launch)
	}
}

long upload_all(Batch *b) {
	CUDA_CHECK(cudaEventRecord(b->ev_a, b->st_main));
	const int S = (int)b->streams.size();
	std::vector<int> pending;
	uint32_t longest = 0, seg = 4096u;
	for (int si = 0; si < S; si++) {
		Stream &s = b->streams[si];
		begin_upload(b, s);
		if (!s.scan_pending) continue;
		pending.push_back(si);
		const uint32_t span = s.bb.length - (s.scan_from & ~15u);
		longest = std::max(longest, span);
		// room for one start code per 512 bytes (FFmpeg streams: two per picture of tens of KiB; a slice per
		// macroblock row: ~70 per picture).  A stream that packs them denser overflows its list; the scan is
		// then repeated with the count it reported.
		seg = std::max(seg, span / 512u + 16u);
	}
	if (!pending.empty()) {
		const int n = (int)pending.size();
		reserve_scan(b, (uint32_t)n, seg);
		for (int k = 0; k < n; k++) {
			const Stream &s = b->streams[pending[k]];
			b->h_spans[k] = ScanSpan{s.d_es.data(), s.scan_from, s.bb.length};
		}
		launch_scan(b, n, longest);
		CUDA_CHECK(cudaEventRecord(b->ev_b, b->st_main));
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));
		float ms = 0;
		CUDA_CHECK(cudaEventElapsedTime(&ms, b->ev_a, b->ev_b));
		b->stats.scan_ms += ms;
		uint32_t most = *std::max_element(b->h_scan_counts.data(), b->h_scan_counts.data() + n);
		if (most > scan_seg(b)) {
			// a list overflowed (hostile input: start codes cannot overlap, so at most length / 3 of them): once
			// more, with room for the count the kernel reported
			reserve_scan(b, (uint32_t)n, most + 16u);
			for (int k = 0; k < n; k++) {  // (the pinned span list may have been reallocated)
				const Stream &s = b->streams[pending[k]];
				b->h_spans[k] = ScanSpan{s.d_es.data(), s.scan_from, s.bb.length};
			}
			launch_scan(b, n, longest);
			CUDA_CHECK(cudaStreamSynchronize(b->st_main));
			most = *std::max_element(b->h_scan_counts.data(), b->h_scan_counts.data() + n);
			if (most > scan_seg(b)) throw std::runtime_error("jsmpeg_b200: start-code index overflow after a rescan");
		}
		if (most) {  // the positions of all spans in one (strided) copy
			CUDA_CHECK(cudaMemcpy2DAsync(b->h_scan_pos.data(), (size_t)scan_seg(b) * sizeof(uint32_t), b->d_scan_pos.data(),
			                             (size_t)scan_seg(b) * sizeof(uint32_t), (size_t)most * sizeof(uint32_t), (size_t)n,
			                             cudaMemcpyDeviceToHost, b->st_main));
			b->stats.d2h_bytes += (uint64_t)most * n * sizeof(uint32_t);
			CUDA_CHECK(cudaStreamSynchronize(b->st_main));
		}
		bool grew = false;
		for (int k = 0; k < n; k++) {
			Stream &s = b->streams[pending[k]];
			uint32_t *hits = b->h_scan_pos.data() + (size_t)k * scan_seg(b);
			const uint32_t cnt = b->h_scan_counts[k];
			std::sort(hits, hits + cnt);
			// the rescanned window starts 2 bytes before the old frontier, so nothing is reported twice
			s.codes.insert(s.codes.end(), hits, hits + cnt);
			grew |= cnt != 0;
			s.scanned = s.bb.length;
			s.scan_pending = false;
		}
		if (grew) {  // the device's copy, for the lane-parallel walk's slice ends: every row that changed, in one copy
			size_t longest_list = 0;
			for (auto &s : b->streams) longest_list = std::max(longest_list, s.codes.size());
			const bool rebuilt = reserve_codes(b, (uint32_t)longest_list);
			const uint32_t stride = codes_stride(b);
			for (int si = 0; si < S; si++) {
				const Stream &s = b->streams[si];
				// (a rewound stream's list starts over: staging whole rows keeps this free of bookkeeping; they are short)
				if (!s.codes.empty() && (rebuilt || std::find(pending.begin(), pending.end(), si) != pending.end()))
					memcpy(b->h_codes.data() + (size_t)si * stride, s.codes.data(), s.codes.size() * sizeof(uint32_t));
			}
			CUDA_CHECK(cudaMemcpy2DAsync(b->d_codes.data(), (size_t)stride * sizeof(uint32_t), b->h_codes.data(),
			                             (size_t)stride * sizeof(uint32_t), longest_list * sizeof(uint32_t), (size_t)S,
			                             cudaMemcpyHostToDevice, b->st_main));
			b->stats.h2d_bytes += (uint64_t)longest_list * S * sizeof(uint32_t);
			CUDA_CHECK(cudaStreamSynchronize(b->st_main));  // the pinned staging is written again by the next scan
		}
	}
	// picture start codes = prefixes whose fourth byte is 00 and inside the buffer (findStartCode, buffer.js:130-139).
	// Only the very last prefix can still be waiting for its fourth byte.
	long total = 0;
	for (auto &s : b->streams) {
		while (s.codes_classified < s.codes.size()) {
			const uint32_t p = s.codes[s.codes_classified];
			if (p + 3u >= s.bb.length) break;
			if (s.bb.bytes[p + 3u] == 0) { s.pics.push_back(p); s.pic_code.push_back(s.codes_classified); }
			s.codes_classified++;
		}
		total += (long)s.pics.size();
	}
	return total;
}

// ---- record slots ----------------------------------------------------------------------------------

void ensure_pool(Batch *b) {
	int need_mb = 0;
	for (auto &s : b->streams) if (s.has_seq) need_mb = std::max(need_mb, s.seq.mb_size);
	if (need_mb <= b->slot_mb || need_mb == 0) return;
	for (auto &s : b->streams) flush_cache(b, s);
	CUDA_CHECK(cudaStreamSynchronize(b->st_main));
	CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
	b->recon_pending = false;
	// the old pool goes before the free memory is measured
	b->d_hdr.reset(); b->d_coef.reset(); b->d_park.reset(); b->d_stage.reset(); b->d_info.reset(); b->h_info.reset();
	b->slot_mb = 0;
	b->n_slots = 0;
	b->free_slots.clear();
	// per macroblock: 16 B record + 6 x 128 B coefficient blocks + 6 x 8 B {bit offset, dc} side array; per picture
	// the lane-parallel walk's staging entries
	const size_t slot_bytes = (size_t)need_mb * (sizeof(mb_record_t) + MB_COEF_INT16 * sizeof(int16_t) + 6 * sizeof(uint2)) +
	                          (size_t)stage_entries_for(need_mb) * 64;
	size_t n = b->max_slots_req;
	size_t free_b = 0, total_b = 0;
	CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
	const size_t fit = (size_t)(0.9 * (double)free_b) / slot_bytes;  // a request beyond the device is cut, not fatal
	if (n == 0) n = std::min<size_t>((size_t)(0.45 * (double)free_b) / slot_bytes, 4096);
	n = std::max<size_t>(std::min(n, fit), 2);
	b->d_hdr.reserve(n * need_mb);
	b->d_coef.reserve(n * need_mb * MB_COEF_INT16);
	b->d_park.reserve(n * need_mb * 6);
	b->d_stage.reserve(n * (size_t)stage_entries_for(need_mb) * 4);
	b->d_info.reserve(n);
	b->h_info.reserve(n);
	b->slot_mb = need_mb;
	b->n_slots = (int)n;
	for (int i = (int)n - 1; i >= 0; i--) b->free_slots.push_back(i);
}

void ensure_task_caps(Batch *b, int n_parse) {
	if ((size_t)n_parse <= b->d_ptasks.size()) return;
	const size_t cap = std::max<size_t>(n_parse, b->d_ptasks.size() * 2);
	b->h_ptasks.reserve(cap);
	b->d_ptasks.reserve(cap);
}

PlaneSet plane_set(const Stream &s, uint8_t *base) {
	PlaneSet p;
	p.y = base;
	p.cr = base + s.coded_size;
	p.cb = base + s.coded_size + (s.coded_size >> 2);
	return p;
}

bool entry_stale(const Stream &s, const Parsed &e) {
	// a parse that ran into the end of the data it saw must be redone once more data is there (SURVEY Q15)
	return e.len_at_parse != s.bb.length && (uint64_t)e.info.end_bit + 64 >= (uint64_t)e.len_at_parse * 8;
}

// dst[i] <- src[i], size[i] bytes, in ONE batched copy call on `st` (cudaMemcpyBatchAsync, CUDA 12.8+); plain copies
// where the driver has no batched copy.  `order`: cudaMemcpySrcAccessOrderDuringApiCall for sources the caller may
// change once the call returns (pageable memory)
void copy_batch(Batch *b, std::vector<void *> &dst, std::vector<void *> &src, std::vector<size_t> &size, cudaStream_t st,
                cudaMemcpySrcAccessOrder order = cudaMemcpySrcAccessOrderStream) {
	const size_t n_copy = dst.size();
	bool batched = false;
	if (b->batch_copy_ok && n_copy > 1) {
		cudaMemcpyAttributes attr{};
		attr.srcAccessOrder = order;
		size_t attr_idx = 0, fail_idx = 0;
		cudaError_t e = cudaMemcpyBatchAsync(dst.data(), src.data(), size.data(), n_copy, &attr, &attr_idx, 1, &fail_idx, st);
		if (e == cudaSuccess) batched = true;
		else { (void)cudaGetLastError(); b->batch_copy_ok = false; }  // older driver: plain copies from now on
	}
	if (!batched)
		for (size_t i = 0; i < n_copy; i++) CUDA_CHECK(cudaMemcpyAsync(dst[i], src[i], size[i], cudaMemcpyDefault, st));
}

// What stage 1 left in record `slot`, as its readers (stage 2, the coefficient export) take it: the macroblock records,
// the dense coefficient records and the compact coefficient plane
struct SlotRecords {
	const mb_record_t *hdr;
	const int16_t *coef;
	const coef_record_t *compact;
};
SlotRecords slot_records(const Batch *b, int slot) {
	return {b->d_hdr.data() + (size_t)slot * b->slot_mb, b->d_coef.data() + (size_t)slot * b->slot_mb * MB_COEF_INT16,
	        compact_plane(b->d_stage.data() + (size_t)slot * stage_entries_for(b->slot_mb) * 4)};  // (stage 1b wrote it: parse_task)
}

// Room for `n` tasks in the pinned task table `h` and its device copy `d`; the reads of the device copy queued on
// `reader` finish before it is reallocated
template <typename T>
void reserve_tasks(PinnedBuffer<T> &h, DeviceBuffer<T> &d, size_t n, cudaStream_t reader) {
	if (n <= d.size()) return;
	CUDA_CHECK(cudaStreamSynchronize(reader));
	h.reserve(n);
	d.reserve(n);
}

// Whether picture `e` of `s` may lack a macroblock, for the conceal option (DESIGN 3.19).  Every walk counts one per
// record it writes, so a picture whose walk met no invalid code and counted mb_size lacks one only if it wrote one
// twice.  A slice that goes back to an earlier row (a slice start code below the one before it) does that; a picture
// no longer in the stream's listing (its bytes were evicted since it was walked) is taken as one that may.
bool may_lack_macroblocks(const Stream &s, const picture_info_t &e) {
	if (e.error != 0 || e.n_present != s.seq.mb_size) return true;
	const auto at = std::lower_bound(s.pics.begin(), s.pics.end(), e.start_byte - 4);
	if (at == s.pics.end() || *at != e.start_byte - 4) return true;
	const size_t pic = at - s.pics.begin();
	const uint32_t hi = pic + 1 < s.pic_code.size() ? s.pic_code[pic + 1] : (uint32_t)s.codes.size();
	int last = 0;  // the slice start code before (0: none yet)
	for (uint32_t k = s.pic_code[pic] + 1; k < hi; k++) {
		const uint32_t q = s.codes[k];
		if (q + 3u >= s.bb.length) break;
		const int code = s.bb.bytes[q + 3u];
		if (!last && (code == 0xB2 || code == 0xB5)) continue;  // extension and user data before the first slice
		if (code < 0x01 || code > 0xAF) break;                   // (the picture ends at any other start code)
		if (code < last) return true;
		last = code;
	}
	return false;
}

// One step of stage 2 (run_steps): the reconstruct tasks of one step of decode() (or one depth of run_chains), queued
// by launch_reconstruct; the export of macroblock entries (OUT_MACROBLOCKS, decode_macroblocks: `entries`, one launch
// of export_macroblocks_kernel over `entry_mb` macroblocks); accumulated maps (OUT_ACCUMULATED, decode_accumulated:
// `maps`, one launch of accumulate_kernel over `map_warps` warps); coefficients (decode_frames_into,
// decode_coefficients: `coefs`, one launch of export_coefficients_kernel over `coef_mb` macroblocks); residuals
// (decode_residuals: `residuals`, one launch of export_residuals_kernel over `res_warps` warps); and the copies of its
// pictures that follow them.  A step of decode_macroblocks' wave has exports and no reconstruct task.  With the conceal
// option, `conceals` (one launch of conceal_kernel over `conceal_mb` macroblocks) runs before the step's reconstruct.
struct ReconStep {
	std::vector<ReconTask> tasks;
	std::vector<ConcealTask> conceals;
	uint32_t conceal_mb = 0;
	std::vector<MbExportTask> entries;
	uint32_t entry_mb = 0;
	std::vector<AccTask> maps;
	uint32_t map_warps = 0;
	std::vector<CoefExportTask> coefs;
	uint32_t coef_mb = 0;
	std::vector<ResExportTask> residuals;
	uint32_t res_warps = 0;
	std::vector<void *> dst, src;
	std::vector<size_t> size;
	void copy(void *to, void *from, size_t n) {
		dst.push_back(to);
		src.push_back(from);
		size.push_back(n);
	}
	// the entries of the picture whose records are `sr` (`mb_size` macroblocks, picture_coding_type `type`) into `to`
	void entry(const SlotRecords &sr, int mb_size, int type, void *to) {
		entries.push_back(MbExportTask{sr.hdr, to, entry_mb, mb_size, type, 0});
		entry_mb += (uint32_t)mb_size;
	}
	// the map of the I/P picture whose records are `sr` (of a stream with sequence parameters `seq`) into `to`, one depth
	// step from `prev` (nullptr: no previous map)
	void map(const SlotRecords &sr, const SeqParams &seq, const uint2 *prev, uint2 *to) {
		maps.push_back(AccTask{sr.hdr, sr.coef, sr.compact, prev, to, map_warps, seq.mb_width, seq.mb_height});
		map_warps += res_export_warps(seq.mb_size);
	}
	// the coefficients of the picture whose records are `sr` (`mb_size` macroblocks) into `to`
	void coef(const SlotRecords &sr, int mb_size, void *to) {
		coefs.push_back(CoefExportTask{sr.hdr, sr.coef, sr.compact, to, coef_mb, mb_size});
		coef_mb += (uint32_t)mb_size;
	}
	// the residual of the picture whose records are `sr` (of a stream with sequence parameters `seq`) into `to`
	void residual(const SlotRecords &sr, const SeqParams &seq, int16_t *to) {
		residuals.push_back(ResExportTask{sr.hdr, sr.coef, sr.compact, to, res_warps, seq.mb_width, seq.mb_height, 0});
		res_warps += res_export_warps(seq.mb_size);
	}
	// With the conceal option `on`, the copy of the macroblocks picture `e` of `s` lacks from the forward set of its
	// reconstruct task `t` into its destination set (DESIGN 3.19), queued only for a picture that may lack one
	// (may_lack_macroblocks): a clean picture costs nothing.
	void conceal(const ReconTask &t, const Stream &s, const picture_info_t &e, bool on) {
		if (!on || !may_lack_macroblocks(s, e)) return;
		conceals.push_back(ConcealTask{t.hdr, t.cur, t.fwd, t.mb_width, t.mb_size, conceal_mb, 0});
		conceal_mb += (uint32_t)t.mb_size;
	}
};

// The tasks `list` of all `steps` (ReconStep::entries, maps, coefs, residuals, conceals) go up in one copy on the reconstruct
// stream, through the pinned table `h` into `d`; returns where each step's tasks begin in `d`.  The previous upload's
// readers are done before the pinned table is written again: every call ends with its reconstruction complete, and the
// next wave of run_chains or decode_macroblocks waits for ev_round.
template <typename T>
std::vector<const T *> upload_step_tasks(Batch *b, const std::vector<ReconStep> &steps, std::vector<T> ReconStep::*list,
                                         PinnedBuffer<T> &h, DeviceBuffer<T> &d) {
	size_t n = 0;
	for (const ReconStep &r : steps) n += (r.*list).size();
	reserve_tasks(h, d, n, b->st_recon);
	std::vector<const T *> at;
	size_t m = 0;
	for (const ReconStep &r : steps) {
		at.push_back(d.data() + m);
		for (const T &t : r.*list) h[m++] = t;
	}
	if (m) CUDA_CHECK(cudaMemcpyAsync(d.data(), h.data(), m * sizeof(T), cudaMemcpyHostToDevice, b->st_recon));
	return at;
}

// The copy-out of one step's pictures (OUT_HOST) on the copy stream, behind the step's launches
void copy_out_step(Batch *b, ReconStep &r) {
	CUDA_CHECK(cudaEventRecord(b->ev_step, b->st_recon));
	CUDA_CHECK(cudaStreamWaitEvent(b->st_copy, b->ev_step, 0));
	copy_batch(b, r.dst, r.src, r.size, b->st_copy);  // all pictures of the step leave in one batched copy call
	CUDA_CHECK(cudaEventRecord(b->ev_copied[b->copy_steps & 1], b->st_copy));
	b->copy_steps++;
}

// Stage 2 of decode_round and of a run_chains or decode_macroblocks wave: `steps`, one after the other on the
// reconstruct stream.  Every step's export and accumulate tasks go up in one copy per table (upload_step_tasks, before
// ev_recon[0]); then, behind the latest stage-1 wave (ev_b: the records are final; where the host waited for the wave,
// an ordering already met) and between ev_recon[0] and ev_recon[1] (decode()'s recon_ms), each step's reconstruct,
// entry export, accumulate, coefficient export and residual export launch, those it has tasks for, and its copies:
// with `copy_out` on the copy stream (copy_out_step), else on the reconstruct stream.  The record slots stay until
// ev_round.  Returns the kernels launched.
int run_steps(Batch *b, std::vector<ReconStep> &steps, bool copy_out) {
	const std::vector<const MbExportTask *> entries = upload_step_tasks(b, steps, &ReconStep::entries, b->h_etasks, b->d_etasks);
	const std::vector<const AccTask *> maps = upload_step_tasks(b, steps, &ReconStep::maps, b->h_atasks, b->d_atasks);
	const std::vector<const CoefExportTask *> coefs = upload_step_tasks(b, steps, &ReconStep::coefs, b->h_ctasks, b->d_ctasks);
	const std::vector<const ResExportTask *> residuals =
	    upload_step_tasks(b, steps, &ReconStep::residuals, b->h_rtasks, b->d_rtasks);
	const std::vector<const ConcealTask *> conceals = upload_step_tasks(b, steps, &ReconStep::conceals, b->h_ktasks, b->d_ktasks);
	CUDA_CHECK(cudaStreamWaitEvent(b->st_recon, b->ev_b, 0));
	CUDA_CHECK(cudaEventRecord(b->ev_recon[0], b->st_recon));
	int launches = 0;
	for (size_t i = 0; i < steps.size(); i++) {
		ReconStep &r = steps[i];
		// A launch overwrites, per stream, the plane set written two of that stream's pictures ago, i.e. by a launch
		// at least two copy-out launches back: the copy-out recorded two launches ago must be done (the copy stream is
		// in order, so that covers every earlier one).  The same holds for the set's entries.
		if (copy_out && b->copy_steps >= 2) CUDA_CHECK(cudaStreamWaitEvent(b->st_recon, b->ev_copied[b->copy_steps & 1], 0));
		if (!r.conceals.empty()) {  // (it writes the destination sets the reconstruct launch then leaves alone there)
			launch_conceal(conceals[i], (int)r.conceals.size(), r.conceal_mb, b->st_recon);
			launches++;
		}
		if (!r.tasks.empty()) launches += launch_reconstruct(r.tasks.data(), (int)r.tasks.size(), b->st_recon);
		if (!r.entries.empty()) {
			launch_export_macroblocks(entries[i], (int)r.entries.size(), r.entry_mb, b->st_recon);
			launches++;
		}
		if (!r.maps.empty()) {  // (a map a step reads as `prev` was written by an earlier step)
			launch_accumulate(maps[i], (int)r.maps.size(), r.map_warps, b->st_recon);
			launches++;
		}
		if (!r.coefs.empty()) {
			launch_export_coefficients(coefs[i], (int)r.coefs.size(), r.coef_mb, b->st_recon);
			launches++;
		}
		if (!r.residuals.empty()) {
			launch_export_residuals(residuals[i], (int)r.residuals.size(), r.res_warps, b->st_recon);
			launches++;
		}
		if (r.dst.empty()) continue;
		if (copy_out) copy_out_step(b, r);  // while the next step reconstructs
		else copy_batch(b, r.dst, r.src, r.size, b->st_recon);
	}
	CUDA_CHECK(cudaEventRecord(b->ev_recon[1], b->st_recon));
	CUDA_CHECK(cudaEventRecord(b->ev_round, b->st_recon));
	b->recon_pending = true;
	return launches;
}

// The header of the picture whose start code is at byte `pos` (ISO 11172-2 2.4.2.5); fields whose bytes are not in the
// buffer yet read as 0
struct PictureHeader {
	int temporal_reference, type;  // type: picture_coding_type
	int full_pel_forward, forward_f_code, full_pel_backward, backward_f_code;
};
PictureHeader picture_header(const Stream &s, uint32_t pos) {
	// the 40 bits after the start code: temporal_reference 10, picture_coding_type 3, vbv_delay 16,
	// full_pel_forward_vector 1, forward_f_code 3, full_pel_backward_vector 1, backward_f_code 3 (and one more).
	// (Read as two words: decode() reads a header per picture.)
	HostBits hb{s.bb.bytes, s.bb.length, ((uint64_t)pos + 4) * 8};
	const uint64_t w = (uint64_t)hb.read(32) << 8 | hb.read(8);
	auto field = [w](int first, int n) { return (int)(w >> (40 - first - n)) & ((1 << n) - 1); };
	return {field(0, 10), field(10, 3), field(29, 1), field(30, 3), field(33, 1), field(34, 3)};
}

// Which walk kernel takes picture `pic` of a stream.  b_walk: a type 3 picture goes to the B-picture walk (decode() and
// decode_pictures: the decode_b option); everything else, and everything without it, to an I/P walk
WalkKind walk_kind(const Batch *b, const Stream &s, uint32_t pic, bool b_walk) {
	const int type = picture_header(s, s.pics[pic]).type;
	WalkKind kind = (b_walk && type == 3) ? WALK_B : WALK_LANES;
	if (b->slice_walk && (type == 1 || type == 2)) {  // enough slice start codes between this picture's and the next one's?
		const uint32_t hi = pic + 1 < s.pic_code.size() ? s.pic_code[pic + 1] : (uint32_t)s.codes.size();
		int n_slices = 0;
		for (uint32_t k = s.pic_code[pic] + 1; k < hi && n_slices < SLICE_WALK_MIN_SLICES; k++) {
			const uint32_t q = s.codes[k];
			if (q + 3u < s.bb.length && s.bb.bytes[q + 3u] >= 0x01 && s.bb.bytes[q + 3u] <= 0xAF) n_slices++;
		}
		if (n_slices >= SLICE_WALK_MIN_SLICES) kind = WALK_SLICES;
	}
	return kind;
}

// The stage-1 task of picture `pic` of stream `si`: records into `slot`, its info into d_info[info_idx]
ParseTask parse_task(const Batch *b, int si, uint32_t pic, int slot, int info_idx) {
	const Stream &s = b->streams[si];
	ParseTask t{};
	t.es = s.d_es.data();
	t.es_len = s.bb.length;
	t.start_byte = s.pics[pic] + 4;
	t.seq = s.d_seq.data();
	t.hdr = b->d_hdr.data() + (size_t)slot * b->slot_mb;
	t.coef = b->d_coef.data() + (size_t)slot * b->slot_mb * MB_COEF_INT16;
	t.park = b->d_park.data() + (size_t)slot * b->slot_mb * 6;
	t.info = b->d_info.data() + info_idx;
	t.mb_width = s.seq.mb_width;
	t.mb_size = s.seq.mb_size;
	t.stage = b->d_stage.data() + (size_t)slot * stage_entries_for(b->slot_mb) * 4;
	t.stage_entries = stage_entries_for(b->slot_mb);
	t.codes = b->d_codes.data() ? b->d_codes.data() + (size_t)si * codes_stride(b) : nullptr;
	t.n_codes = (uint32_t)s.codes.size();
	t.code_hint = s.pic_code[pic];
	return t;
}

// One picture of a stage-1 wave: picture `pic` of stream `stream`, records into `slot`; `kind` is its walk kernel
// (walk_kind), `bytes` its length up to the next picture start code
struct WaveItem {
	int stream;
	uint32_t pic;
	int slot;
	WalkKind kind;
	uint32_t bytes;
};

// Picture `pic` of stream `si` as an item of a stage-1 wave, in a record slot it takes from the free ones; b_walk as in
// walk_kind
WaveItem take_slot(Batch *b, int si, uint32_t pic, bool b_walk) {
	const Stream &s = b->streams[si];
	const int slot = b->free_slots.back();
	b->free_slots.pop_back();
	const uint32_t end = pic + 1 < s.pics.size() ? s.pics[pic + 1] : s.bb.length;
	return {si, pic, slot, walk_kind(b, s, pic, b_walk), end - s.pics[pic]};
}

// Frees the look-ahead's record slots too when the free ones do not cover `need` pictures (decode() parses the
// look-ahead again)
void free_slots_for(Batch *b, size_t need) {
	if (b->free_slots.size() < need)
		for (auto &s : b->streams) flush_cache(b, s);
}

// Stage 1 of `wave` as one wave, for decode(), decode_chains and decode_macroblocks alike; expand = false runs the walks
// alone (records without coefficients: decode_macroblocks).  The tasks are grouped by walk kernel and,
// within a kernel, longest first: a CTA's warps, and consecutive CTAs (which land on different SMs), then carry
// similar amounts of work and the walk ends without a long tail.  The first kernel present runs on the main stream;
// the others have walk kernels of their own (one warp per picture, latency-bound like every walk) and run beside it on
// side streams, forked after the upload and joined on the main stream, where ev_a / ev_b bracket the wave.  On return
// the infos are on the host, b->h_info[i] that of wave[i].
// early_infos = false: stage 1 is complete on return.  true (decode()): the infos, which the walks write, leave behind
// the walks alone (ev_mid: every walk done) and the host returns with them while the expand of the biggest pictures is
// still running; a reader of the coefficients waits for ev_b.
// Returns the number of kernels launched.
int parse_wave(Batch *b, const std::vector<WaveItem> &wave, bool expand, bool early_infos = false) {
	const int n = (int)wave.size();
	std::vector<int> order(n);
	for (int i = 0; i < n; i++) order[i] = i;
	std::stable_sort(order.begin(), order.end(), [&](int x, int y) {
		return wave[x].kind != wave[y].kind ? wave[x].kind < wave[y].kind : wave[x].bytes > wave[y].bytes;
	});
	ensure_task_caps(b, n);
	int cnt[N_WALK_KINDS] = {};
	for (int j = 0; j < n; j++) {
		const WaveItem &w = wave[order[j]];
		b->h_ptasks[j] = parse_task(b, w.stream, w.pic, w.slot, order[j]);
		cnt[w.kind]++;
	}
	if (b->recon_pending) {  // slots freed by an earlier round or wave may still be read by its reconstruct launches
		CUDA_CHECK(cudaStreamWaitEvent(b->st_main, b->ev_round, 0));
		b->recon_pending = false;
	}
	CUDA_CHECK(cudaMemcpyAsync(b->d_ptasks.data(), b->h_ptasks.data(), n * sizeof(ParseTask), cudaMemcpyHostToDevice, b->st_main));
	CUDA_CHECK(cudaEventRecord(b->ev_a, b->st_main));
	int primary = 0;
	while (cnt[primary] == 0) primary++;
	if (cnt[primary] < n) CUDA_CHECK(cudaEventRecord(b->ev_sfork, b->st_main));
	// the wave's pictures by walk kernel, in WalkKind order
	int launches = 0, n_side = 0;
	for (int kind = 0, off = 0; kind < N_WALK_KINDS; off += cnt[kind++]) {
		if (cnt[kind] == 0) continue;
		cudaStream_t st = b->st_main;
		if (kind != primary) {
			st = b->st_side[n_side];
			CUDA_CHECK(cudaStreamWaitEvent(st, b->ev_sfork, 0));
		}
		launches += launch_parse_pictures((WalkKind)kind, b->d_ptasks.data() + off, cnt[kind], b->slot_mb, expand, st, &b->fork,
		                                  early_infos ? b->st_info : nullptr);
		if (kind != primary) {
			CUDA_CHECK(cudaEventRecord(b->ev_sjoin[n_side], st));
			CUDA_CHECK(cudaStreamWaitEvent(b->st_main, b->ev_sjoin[n_side], 0));
			n_side++;
		}
	}
	cudaStream_t st_info = early_infos ? b->st_info : b->st_main;
	if (early_infos) CUDA_CHECK(cudaEventRecord(b->ev_mid, st_info));
	CUDA_CHECK(cudaMemcpyAsync(b->h_info.data(), b->d_info.data(), n * sizeof(picture_info_t), cudaMemcpyDeviceToHost, st_info));
	if (early_infos) CUDA_CHECK(cudaEventRecord(b->ev_info, st_info));
	CUDA_CHECK(cudaEventRecord(b->ev_b, b->st_main));
	HostClock::time_point t = HostClock::now();
	CUDA_CHECK(cudaEventSynchronize(early_infos ? b->ev_info : b->ev_b));
	lap(b->trace.infos, t);
	return launches;
}

// The reconstruct task of a picture of `s` whose records are in `slot`: written into the plane set at `cur`, predicted
// from `fwd` (and, for a B picture, `bwd`), with the fused RGBA conversion into `rgba` unless that is nullptr
ReconTask recon_task(const Batch *b, const Stream &s, int slot, uint8_t *cur, uint8_t *fwd, uint8_t *bwd, uint8_t *rgba) {
	ReconTask t{};
	const SlotRecords sr = slot_records(b, slot);
	t.hdr = sr.hdr;
	t.coef = sr.coef;
	t.compact = sr.compact;
	t.cur = plane_set(s, cur);
	t.fwd = plane_set(s, fwd);
	if (bwd) t.bwd = plane_set(s, bwd);
	t.mb_width = s.seq.mb_width;
	t.mb_size = s.seq.mb_size;
	t.coded_width = s.seq.coded_width;
	t.coded_height = s.seq.coded_height;
	t.width = s.width;
	t.height = s.height;
	t.rgba = rgba;
	return t;
}

// The stream's RGBA picture, made on first use: opaque white, like the canvas the reference creates
// (canvas2d.js:24-29); the odd edge keeps it
uint8_t *stream_rgba(Batch *b, Stream &s) {
	if (!s.d_rgba.data()) {
		s.d_rgba.reserve((size_t)s.width * s.height * 4);
		CUDA_CHECK(cudaMemsetAsync(s.d_rgba.data(), 0xff, (size_t)s.width * s.height * 4, b->st_recon));
	}
	return s.d_rgba.data();
}

// The stream's two B-picture sets, made zeroed on first use
void reserve_b_sets(Batch *b, Stream &s) {
	if (s.sets[2].planes.data()) return;
	for (int i = 2; i < 4; i++) make_planes(s, s.sets[i], b->st_recon);
}

// The stream's entry buffers (OUT_MACROBLOCKS), made on first use: every plane set's, zeroed on the reconstruct stream,
// and every host-ring slot's
void reserve_entries(Batch *b, Stream &s) {
	if (s.sets[0].entries.data()) return;
	const size_t bytes = (size_t)s.seq.mb_size * sizeof(jsmpeg_b200_macroblock_t);
	for (StreamSet &set : s.sets) {
		set.entries.reserve(bytes);
		CUDA_CHECK(cudaMemsetAsync(set.entries.data(), 0, bytes, b->st_recon));
	}
	for (HostSlot &h : s.ring) {
		h.entries.reserve(bytes);
		memset(h.entries.data(), 0, bytes);
	}
}

// The maps of the stream's two I/P sets (OUT_ACCUMULATED), made on first use, unwritten: nothing reads them before a
// call with the flag writes them, or get / read_accumulated fills them untraced (fill_untraced)
void reserve_maps(Stream &s) {
	if (s.sets[0].map.data()) return;
	for (int i = 0; i < 2; i++) {
		s.sets[i].map.reserve((size_t)s.coded_size * 3 / 2);
		s.sets[i].map_written = false;
	}
}

// The stream's residual (OUT_RESIDUALS), made zeroed on the reconstruct stream on first use
int16_t *reserve_residuals(Batch *b, Stream &s) {
	if (!s.d_res.data()) {
		s.d_res.reserve((size_t)s.coded_size * 3 / 2);
		CUDA_CHECK(cudaMemsetAsync(s.d_res.data(), 0, s.d_res.size() * sizeof(int16_t), b->st_recon));
	}
	return s.d_res.data();
}

// Every record of `n_rec` from `map` untraced {0, 0, 0, -1}, on `st`
void fill_untraced(uint2 *map, size_t n_rec, cudaStream_t st) {
	CUDA_CHECK(cudaMemsetAsync(map, 0, n_rec * 8, st));
	CUDA_CHECK(cudaMemset2DAsync(reinterpret_cast<uint8_t *>(map) + 6, 8, 0xff, 2, n_rec, st));
}

// Where a task is in a list of steps: steps[step].tasks[task]; step -1: nowhere
struct TaskAt {
	int step = -1, task = 0;
};

// decode_frames (DESIGN 3.16) and decode_frames_into (DESIGN 3.17): where one stream's frames go -- each destination
// nullptr or the stream's frame 0 in device memory, `info` its row of the caller's info_out on the host -- and how many
// the call has given it so far.  decode_frames_display (DESIGN 3.18, `display`) presents them: frame j is the j-th
// picture the call presents, and `n` counts those.
struct FrameCursor {
	uint8_t *planes = nullptr, *rgba = nullptr, *mb = nullptr;
	int16_t *res = nullptr, *coef = nullptr;
	uint2 *acc = nullptr;
	jsmpeg_b200_frame_t *info = nullptr;
	int n = 0;
	bool display = false;
	unsigned kinds = 0;  // (display) the KIND_* bits of the destinations given
	int made = 0;        // pictures reconstructed
	int reserved = -1;   // (display) the frame the stream's held I/P picture was written to, its successor in the round
	bool stored = false;  // (display) a picture of the call went to the stream's store
	uint8_t *last_rgba = nullptr;  // where the newest reconstructed picture's RGBA and residual went
	int16_t *last_res = nullptr;
	// frame j of the stream `s`
	FrameAt at(const Stream &s, size_t j) const {
		const size_t planes_n = (size_t)s.coded_size * 3 / 2, mb_n = (size_t)s.seq.mb_size;
		FrameAt f;
		if (planes) f.planes = planes + j * planes_n;
		if (rgba) f.rgba = rgba + j * s.width * s.height * 4;
		if (mb) f.mb = mb + j * mb_n * sizeof(jsmpeg_b200_macroblock_t);
		if (res) f.res = res + j * planes_n;
		if (coef) f.coef = coef + j * mb_n * 384;
		if (acc) f.acc = acc + j * planes_n;
		return f;
	}
};

// Picture `e` of stream `s`, records in `slot`, consumed by decode() or by a seek, reconstructed by step `step` of
// `steps` into the stream's own sets with decode()'s rotation; `visible`: the call leaves it in get_planes (decode():
// every picture it consumes, a seek: each chain's last).  Beside its planes go, under OUT_MACROBLOCKS, its entries and,
// for an I/P picture, under OUT_ACCUMULATED its map (else the set's map no longer matches it); the visible picture also
// goes to the stream's RGBA under OUT_RGBA and, under OUT_HOST, with its entries to the next slot of its host ring.
// `newest` gets where its task is (OUT_RESIDUALS: the caller's newest picture stores its residual).  With a frame `to`
// (decode_frames: the stream's next frame; decode_frames_display: its presentation frame or the stream's store) stage 2
// also stores its planes there, and its RGBA and residual go there instead of the stream's own, and its entries are also
// exported there.  decode_frames_into adds its coefficients, exported from its records, and its map: an I/P picture's map
// goes to the frame INSTEAD of the set's map (the set's map_at says so; finish_frames brings the newest one back), a B
// picture's frame is untraced.  Returns the bytes its copies bring to the host.
uint64_t consume_picture(Batch *b, Stream &s, std::vector<ReconStep> &steps, size_t step, int slot, const picture_info_t &e,
                         int flags, bool visible, TaskAt &newest, const FrameAt *to = nullptr) {
	const bool is_b = e.picture_type == 3;  // (only the extension's walk answers PIC_DECODED for one)
	const size_t planes = (size_t)s.coded_size * 3 / 2;
	uint8_t *rgba = to && to->rgba ? to->rgba : visible && (flags & JSMPEG_B200_OUT_RGBA) ? stream_rgba(b, s) : nullptr;
	ReconTask t;
	if (is_b) {
		// `cur` holds the older and `1 - cur` the newer of the two most recent I/P pictures: the B picture's forward
		// (past) and backward (future) reference.  It goes to a set of its own.
		reserve_b_sets(b, s);
		s.last = 2 + s.b_cur;
		t = recon_task(b, s, slot, s.sets[s.last].planes.data(), s.sets[s.cur].planes.data(), s.sets[1 - s.cur].planes.data(), rgba);
		s.b_cur ^= 1;  // no reference: the I/P ping-pong stays as it is
	} else {
		s.last = s.cur;
		t = recon_task(b, s, slot, s.sets[s.cur].planes.data(), s.sets[1 - s.cur].planes.data(), nullptr, rgba);
		s.cur ^= 1;  // mpeg1.js:221-246: the picture just decoded becomes `forward`
	}
	if (to && to->planes) t.frame = to->planes;
	if (to && to->res) t.res = to->res;
	StreamSet &set = s.sets[s.last];
	if (steps.size() <= step) steps.emplace_back();
	ReconStep &r = steps[step];
	r.conceal(t, s, e, b->conceal);
	r.tasks.push_back(t);
	newest = {(int)step, (int)r.tasks.size() - 1};
	const SlotRecords sr = slot_records(b, slot);
	if (flags & JSMPEG_B200_OUT_MACROBLOCKS) {
		reserve_entries(b, s);
		r.entry(sr, s.seq.mb_size, e.picture_type, set.entries.data());
	}
	if (to && to->mb) r.entry(sr, s.seq.mb_size, e.picture_type, to->mb);
	if (to && to->coef) r.coef(sr, s.seq.mb_size, to->coef);
	uint2 *acc = to ? to->acc : nullptr;  // (only under OUT_ACCUMULATED)
	if (!is_b) {  // the map beside the set (or in its map frame), one depth step from the forward set's picture's map
		if (flags & JSMPEG_B200_OUT_ACCUMULATED) {
			reserve_maps(s);
			const StreamSet &fwd = s.sets[s.cur];  // (swapped above)
			const uint2 *prev = !fwd.map_written ? nullptr : fwd.map_at ? fwd.map_at : fwd.map.data();
			r.map(sr, s.seq, prev, acc ? acc : set.map.data());
		}
		set.map_written = (flags & JSMPEG_B200_OUT_ACCUMULATED) != 0;
		set.map_at = acc;
	} else if (acc) {  // (queued before the step's launches, which do not touch it)
		fill_untraced(acc, planes, b->st_recon);
	}
	uint64_t host_bytes = 0;
	if (visible && (flags & JSMPEG_B200_OUT_HOST)) {
		s.h_head = (s.h_head + 1) % HOST_RING;
		HostSlot &h = s.ring[s.h_head];
		r.copy(h.planes.data(), t.cur.y, planes);
		host_bytes += planes;
		if (flags & JSMPEG_B200_OUT_MACROBLOCKS) {
			const size_t n = (size_t)s.seq.mb_size * sizeof(jsmpeg_b200_macroblock_t);
			r.copy(h.entries.data(), set.entries.data(), n);
			host_bytes += n;
		}
	}
	return host_bytes;
}

// How many of the stream's parsed-ahead pictures a round that wants `want` of them consumes: decode_round's consumption
// loop over the cache, run ahead without consuming (its stop rules, in its order)
size_t consumable(const Stream &s, int want) {
	uint64_t index = s.bb.index;
	size_t k = 0;
	for (; (int)k < want && k < s.cache.size(); k++) {
		auto it = std::lower_bound(s.pics.begin(), s.pics.end(), (uint32_t)((index + 7) >> 3));
		const Parsed &e = s.cache[k];
		if (it == s.pics.end() || e.pos != *it || entry_stale(s, e)) break;
		index = e.info.end_bit;
	}
	return k;
}

// The stream's store, with room for one frame of each kind `f` asks for
FrameAt store_frame(Stream &s, const FrameCursor &f) {
	const size_t planes = (size_t)s.coded_size * 3 / 2, mb = (size_t)s.seq.mb_size;
	FrameStore &h = s.hold;
	FrameAt to;
	if (f.planes) { h.planes.reserve(planes); to.planes = h.planes.data(); }
	if (f.rgba) { h.rgba.reserve((size_t)s.width * s.height * 4); to.rgba = h.rgba.data(); }
	if (f.mb) { h.mb.reserve(mb * sizeof(jsmpeg_b200_macroblock_t)); to.mb = h.mb.data(); }
	if (f.res) { h.res.reserve(planes); to.res = h.res.data(); }
	if (f.coef) { h.coef.reserve(mb * 384); to.coef = h.coef.data(); }
	if (f.acc) { h.acc.reserve(planes); to.acc = h.acc.data(); }
	return to;
}

// The held picture's frame of each kind in `kinds` into `to`, queued as copies (copy_batch)
void copy_held(const Stream &s, unsigned kinds, const FrameAt &to, std::vector<void *> &dst, std::vector<void *> &src,
               std::vector<size_t> &size) {
	const FrameStore &h = s.hold;
	const size_t planes = (size_t)s.coded_size * 3 / 2, mb = (size_t)s.seq.mb_size;
	auto add = [&](unsigned kind, void *d, const void *from, size_t n) {
		if (!(kinds & kind) || !d) return;
		dst.push_back(d);
		src.push_back(const_cast<void *>(from));
		size.push_back(n);
	};
	add(KIND_PLANES, to.planes, h.planes.data(), planes);
	add(KIND_RGBA, to.rgba, h.rgba.data(), (size_t)s.width * s.height * 4);
	add(KIND_MB, to.mb, h.mb.data(), mb * sizeof(jsmpeg_b200_macroblock_t));
	add(KIND_RES, to.res, h.res.data(), planes * sizeof(int16_t));
	add(KIND_COEF, to.coef, h.coef.data(), mb * 384 * sizeof(int16_t));
	add(KIND_ACC, to.acc, h.acc.data(), planes * sizeof(uint2));
}

// decode_frames_display (DESIGN 3.18): where the reconstructed picture `e` of stream `s`, frame info `info`, goes, by the
// presentation rule.  A B picture is presented at once: the next frame.  An I/P picture first presents the picture the
// stream holds, then is held itself (without decode_b: presented at once).  `left`: the cache entries after it that
// the round consumes.  If its successor reference is among them, its frame is known now -- after the B pictures
// between -- and it goes there directly (f.reserved); else it goes to the stream's store, and a later round, call or
// flush_frames copies it to its frame.  Such a copy (held from an earlier round or call) is queued into `dst`, `src`,
// `size`, for the reconstruct stream ahead of the round's launches: behind the store's writer, before its next one.
FrameAt present_picture(Stream &s, FrameCursor &f, const Parsed &e, const jsmpeg_b200_frame_t &info, size_t left,
                        bool decode_b, std::vector<void *> &dst, std::vector<void *> &src, std::vector<size_t> &size) {
	auto frame = [&](int j) {
		if (f.info) f.info[j] = info;
		return f.at(s, (size_t)j);
	};
	if (!f.display) return frame(f.n++);
	if (e.info.picture_type == 3) return frame(f.n++);
	if (f.reserved >= 0) {  // the held picture went to its frame directly, and the B pictures before it have theirs
		if (f.reserved != f.n) throw std::logic_error("jsmpeg_b200: display order: a held frame out of place");
		f.reserved = -1;
		f.n++;
	} else if (s.hold.held) {
		const FrameAt at = f.at(s, (size_t)f.n);
		copy_held(s, s.hold.kinds, at, dst, src, size);
		if (f.info) f.info[f.n] = s.hold.info;
		// the map_at invariant (finish_frames): the held picture's map is in its frame once the copy has run, and the
		// store may be rewritten by this round -- the next I/P picture reads its `prev` from the frame
		for (int i = 0; i < 2; i++)
			if (s.sets[i].map_at && s.sets[i].map_at == s.hold.acc.data()) s.sets[i].map_at = at.acc;
		s.hold.held = false;
		f.n++;
	}
	if (!decode_b) return frame(f.n++);
	int n_b = 0;
	for (size_t k = 0; k < left; k++) {
		const picture_info_t &q = s.cache[k].info;
		if (q.status != PIC_DECODED) continue;
		if (q.picture_type != 3) {
			f.reserved = f.n + n_b;
			return frame(f.reserved);
		}
		n_b++;
	}
	s.hold.held = true;
	s.hold.kinds = f.kinds;
	s.hold.info = info;
	f.stored = true;
	return store_frame(s, f);
}

// One round: parse ahead what is missing in one wave, then consume up to want[s] pictures per stream in decode()
// order and queue their reconstruction.  Returns pictures consumed; `progress[s]` gets the per-stream count, `more[s]`
// whether the stream may have further pictures.  `frames` (decode_frames): per stream, the cursor its reconstructed
// pictures go to as frames.
long decode_round(Batch *b, const std::vector<int> &want, std::vector<int> &progress, std::vector<char> &more, int flags,
                  std::vector<FrameCursor> *frames) {
	const int S = (int)b->streams.size();
	HostClock::time_point t = HostClock::now();
	// ---- 1. plan the parse wave
	std::vector<WaveItem> wave;
	std::vector<size_t> fresh(S, 0);  // per stream: the cache index of its first picture in the wave
	for (int si = 0; si < S; si++) {
		Stream &s = b->streams[si];
		progress[si] = 0;
		more[si] = s.has_seq && want[si] > 0;
		if (!more[si]) continue;
		const uint32_t from_byte = (s.bb.index + 7) >> 3;
		auto it = std::lower_bound(s.pics.begin(), s.pics.end(), from_byte);
		if (!s.cache.empty() && (it == s.pics.end() || s.cache.front().pos != *it)) flush_cache(b, s);
		for (size_t j = 0; j < s.cache.size(); j++) {
			if (entry_stale(s, s.cache[j])) {
				while (s.cache.size() > j) { release_slot(b, s.cache.back().slot); s.cache.pop_back(); }
				break;
			}
		}
		fresh[si] = s.cache.size();
		if ((int)s.cache.size() >= want[si]) continue;
		int target = std::max(want[si], b->lookahead);
		auto next = it + (ptrdiff_t)s.cache.size();
		// `it` may be end(); cache is then empty
		while ((int)s.cache.size() < target && next < s.pics.end() && !b->free_slots.empty()) {
			wave.push_back(take_slot(b, si, (uint32_t)(next - s.pics.begin()), b->decode_b));
			Parsed p{};
			p.pos = *next++;
			p.len_at_parse = s.bb.length;
			p.slot = wave.back().slot;
			s.cache.push_back(p);
		}
	}
	// ---- 2. stage 1: the wave, every picture's info on the host before consumption starts; the end of its expand goes
	// on beside steps 3 and 4
	lap(b->trace.plan, t);
	if (!wave.empty()) {
		const double infos = b->trace.infos;
		b->stats.kernel_launches += parse_wave(b, wave, true, true);
		lap(b->trace.stage1, t);
		b->trace.stage1 -= b->trace.infos - infos;
		for (size_t i = 0; i < wave.size(); i++) {  // a stream's pictures are in the wave in cache order
			const int si = wave[i].stream;
			Parsed &p = b->streams[si].cache[fresh[si]++];
			p.info = b->h_info[i];
			if (p.info.error == PARSE_ERR_INVALID_VLC) b->stats.parse_errors++;
			if (p.info.reserved[0]) b->stats.lane_walk_pictures++;
		}
		b->stats.h2d_bytes += wave.size() * sizeof(ParseTask);
		b->stats.d2h_bytes += wave.size() * sizeof(picture_info_t);
	}
	// ---- 3. consume in decode() order; the j-th reconstructed picture of a stream goes to step j
	long consumed = 0;
	std::vector<ReconStep> steps;
	std::vector<void *> held_dst, held_src;  // decode_frames_display: held pictures this round presents (present_picture)
	std::vector<size_t> held_size;
	for (int si = 0; si < S; si++) {
		if (!more[si]) continue;
		Stream &s = b->streams[si];
		FrameCursor *frame = frames ? &(*frames)[si] : nullptr;
		const size_t ahead = frame && frame->display ? consumable(s, want[si]) : 0;
		size_t step = 0;
		TaskAt newest;
		while (progress[si] < want[si]) {
			const uint32_t from_byte = (s.bb.index + 7) >> 3;
			auto it = std::lower_bound(s.pics.begin(), s.pics.end(), from_byte);
			if (it == s.pics.end()) {  // findStartCode(PICTURE) == -1: index parks at the end (buffer.js:126-127)
				s.bb.index = s.bb.length << 3;
				more[si] = 0;
				break;
			}
			if (s.cache.empty() || s.cache.front().pos != *it || entry_stale(s, s.cache.front())) {
				flush_cache(b, s);  // the look-ahead does not match the serial order: re-plan in the next round
				break;
			}
			const Parsed e = s.cache.front();
			s.cache.pop_front();
			s.bb.index = e.info.end_bit;
			progress[si]++;
			consumed++;
			b->stats.pictures++;
			b->stats.es_bytes += (e.info.end_bit >> 3) - e.pos;
			s.last_type = e.info.picture_type;
			// (0 unless both of its bytes are in the buffer)
			s.last_temporal = (uint64_t)e.pos + 5 < s.bb.length ? picture_header(s, e.pos).temporal_reference : 0;
			if (e.info.status == PIC_DECODED) {
				FrameAt to;
				if (frame) {
					const jsmpeg_b200_frame_t info{e.pos, (int16_t)e.info.picture_type, (int16_t)s.last_temporal, e.info.n_present,
					                               e.info.error};
					const size_t left = ahead > (size_t)progress[si] ? ahead - progress[si] : 0;
					to = present_picture(s, *frame, e, info, left, b->decode_b, held_dst, held_src, held_size);
					frame->made++;
					frame->last_rgba = to.rgba;
					frame->last_res = to.res;
				}
				if (!(frame && frame->display)) s.hold.held = false;
				b->stats.d2h_bytes += consume_picture(b, s, steps, step++, e.slot, e.info, flags, true, newest, frame ? &to : nullptr);
				const bool is_b = e.info.picture_type == 3;
				const uint64_t planes = (uint64_t)s.coded_size * 3 / 2;
				b->stats.pictures_decoded++;
				b->stats.coded_blocks += e.info.n_coded_blocks;
				b->stats.macroblocks += e.info.n_present;
				b->stats.algorithmic_bytes += planes + (e.info.picture_type == 2 ? planes : (is_b ? 2 * planes : 0)) +
				                              (uint64_t)s.seq.mb_size * sizeof(mb_record_t) + (uint64_t)e.info.n_coded_blocks * sizeof(coef_record_t);
			}
			// reused by the NEXT round's parse, which waits for this round's reconstruction (ev_round) and is queued behind
			// this round's expand on the main stream
			release_slot(b, e.slot);
		}
		// OUT_RESIDUALS: the stream's last reconstructed picture of the round stores its residual; the earlier ones of the
		// round could not be observed.  (With residual frames the last one is copied at the end of the call: finish_frames.)
		if ((flags & JSMPEG_B200_OUT_RESIDUALS) && newest.step >= 0 && !(frame && frame->res))
			steps[newest.step].tasks[newest.task].res = reserve_residuals(b, s);
		// (consumable() foresaw this loop: a picture whose successor it saw has been presented)
		if (frame && frame->reserved >= 0) throw std::logic_error("jsmpeg_b200: display order: a successor not consumed");
	}
	if (!held_dst.empty()) copy_batch(b, held_dst, held_src, held_size, b->st_recon);
	lap(b->trace.consume, t);
	// ---- 4. reconstruction, behind the wave's expand: the host has consumed the infos and queues the launches while the
	// expand of the biggest pictures is still running.  Every step reconstructs.
	if (!steps.empty()) {
		b->stats.kernel_launches += run_steps(b, steps, (flags & JSMPEG_B200_OUT_HOST) != 0);
		b->stats.recon_launches += steps.size();
	}
	lap(b->trace.stage2, t);
	// ---- 5. the round ends with its wave complete (a round that reconstructs nothing has not waited for its expand yet)
	float ms = 0;
	if (!steps.empty()) {
		CUDA_CHECK(cudaEventSynchronize(b->ev_recon[1]));
		CUDA_CHECK(cudaEventElapsedTime(&ms, b->ev_recon[0], b->ev_recon[1]));
		b->stats.recon_ms += ms;
	}
	if (!wave.empty()) {
		CUDA_CHECK(cudaEventSynchronize(b->ev_b));
		CUDA_CHECK(cudaEventElapsedTime(&ms, b->ev_a, b->ev_b));  // (beside the reconstruction: the two overlap)
		b->stats.parse_ms += ms;
		CUDA_CHECK(cudaEventElapsedTime(&ms, b->ev_a, b->ev_mid));
		b->stats.walk_ms += ms;
		if (b->trace.on) {
			float to_b = 0, to_recon = 0;
			CUDA_CHECK(cudaEventElapsedTime(&to_b, b->ev_a, b->ev_b));
			if (!steps.empty()) CUDA_CHECK(cudaEventElapsedTime(&to_recon, b->ev_a, b->ev_recon[1]));
			b->trace.device += std::max(to_b, to_recon);
		}
	}
	lap(b->trace.close, t);
	return consumed;
}

// decode_frames, once the rounds are queued: the odd edge of every RGBA frame opaque white (the epilogue never writes
// it), then the last RGBA frame into the stream's RGBA under OUT_RGBA, the last residual frame into its residual under
// OUT_RESIDUALS and the newest I/P picture's map frame into its set's map (decode_frames_into), in one batched copy; all
// on the reconstruct stream, behind the frames' stage 2.  The older I/P set's map is never read again before that set is
// rewritten (`prev` and get_accumulated read the newest), so one whose map is in a frame is left unwritten.
// decode_frames_display: the edge fill covers the store too, and the newest reconstructed picture's RGBA and residual are
// wherever it went, frame or store.  The map_at invariant: while the call runs, an I/P set's map_at is where that set's
// picture's map is now -- its frame, or the store while the picture is held there and until present_picture has queued
// its copy to its frame (the store is then free for the next held picture's map, and the next I/P picture's `prev` is
// read from the frame); so the newest set's map_at is what this copies back.
void finish_frames(Batch *b, const std::vector<FrameCursor> &frames, int flags) {
	std::vector<void *> dst, src;
	std::vector<size_t> size;
	for (size_t si = 0; si < frames.size(); si++) {
		const FrameCursor &f = frames[si];
		Stream &s = b->streams[si];
		if (f.made == 0) continue;
		if (f.rgba) {
			const size_t row = (size_t)s.width * 4, image = row * s.height;
			auto fill = [&](uint8_t *rgba, size_t n) {  // the odd edge of `n` images from `rgba`
				if (s.width & 1) CUDA_CHECK(cudaMemset2DAsync(rgba + row - 4, row, 0xff, 4, n * s.height, b->st_recon));
				if (s.height & 1) CUDA_CHECK(cudaMemset2DAsync(rgba + image - row, image, 0xff, row, n, b->st_recon));
			};
			if (f.n) fill(f.rgba, (size_t)f.n);
			if (f.stored) fill(s.hold.rgba.data(), 1);
			if (flags & JSMPEG_B200_OUT_RGBA) {
				dst.push_back(stream_rgba(b, s));
				src.push_back(f.last_rgba);
				size.push_back(image);
			}
		}
		if (f.res && (flags & JSMPEG_B200_OUT_RESIDUALS)) {
			const size_t planes = (size_t)s.coded_size * 3 / 2;
			dst.push_back(reserve_residuals(b, s));
			src.push_back(f.last_res);
			size.push_back(planes * sizeof(int16_t));
		}
		StreamSet &newest = s.sets[1 - s.cur], &older = s.sets[s.cur];
		if (newest.map_at) {
			dst.push_back(newest.map.data());
			src.push_back(const_cast<uint2 *>(newest.map_at));
			size.push_back((size_t)s.coded_size * 3 / 2 * sizeof(uint2));
			newest.map_at = nullptr;
		}
		if (older.map_at) {
			older.map_written = false;
			older.map_at = nullptr;
		}
	}
	if (!dst.empty()) copy_batch(b, dst, src, size, b->st_recon);
}

long batch_decode(Batch *b, int n_pictures, int flags, std::vector<FrameCursor> *frames = nullptr) {
	use_device(b);
	Batch::HostTrace &tr = b->trace;
	const bool trace_on = tr.on;
	tr = Batch::HostTrace{};
	tr.on = trace_on;
	HostClock::time_point t = HostClock::now();
	upload_all(b);
	lap(tr.upload, t);
	ensure_pool(b);
	const int S = (int)b->streams.size();
	std::vector<int> remaining(S, n_pictures), want(S), progress(S);
	std::vector<char> more(S, 1);
	long total = 0;
	int idle_rounds = 0;
	for (;;) {
		int active = 0;
		for (int i = 0; i < S; i++) if (more[i] && remaining[i] > 0 && b->streams[i].has_seq) active++;
		if (!active) break;
		// share the record slots between the active streams
		int cached = 0;
		for (auto &s : b->streams) cached += (int)s.cache.size();
		const int per_stream = std::max(1, (int)(b->free_slots.size() + cached) / active);
		for (int i = 0; i < S; i++)
			want[i] = (more[i] && b->streams[i].has_seq) ? std::min(remaining[i], per_stream) : 0;
		const long got = decode_round(b, want, progress, more, flags, frames);
		total += got;
		bool replanned = false;
		for (int i = 0; i < S; i++) {
			remaining[i] -= progress[i];
			if (want[i] > 0 && progress[i] < want[i] && more[i]) replanned = true;
		}
		if (got == 0 && (!replanned || ++idle_rounds > 2)) break;
		if (got) idle_rounds = 0;
	}
	t = HostClock::now();
	if (frames) finish_frames(b, *frames, flags);
	CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
	CUDA_CHECK(cudaStreamSynchronize(b->st_copy));
	CUDA_CHECK(cudaStreamSynchronize(b->st_main));
	lap(tr.close, t);
	b->recon_pending = false;
	if (tr.on)
		fprintf(stderr, "jsmpeg_b200 decode host_ms: upload=%.3f plan=%.3f stage1=%.3f infos=%.3f consume=%.3f stage2=%.3f close=%.3f device=%.3f\n",
		        tr.upload, tr.plan, tr.stage1, tr.infos, tr.consume, tr.stage2, tr.close, tr.device);
	return total;
}

// ---- decode_pictures / decode_intra: chosen pictures of any streams, each as a fresh decoder gives it from its chain
// start (DESIGN 3.6, 3.7) ------------------------------------------------------------------------------------------

// Picture k is closed when a later start code is resident whose fourth byte is no slice (01..AF), user data (B2) or
// extension (B5).  The parse of a closed picture stops at or before that code, so later bytes cannot change it.
bool picture_closed(const Stream &s, uint32_t k) {
	for (uint32_t c = s.pic_code[k] + 1; c < s.codes_classified; c++) {
		const uint8_t code = s.bb.bytes[s.codes[c] + 3u];
		if (!(code >= 0x01 && code <= 0xAF) && code != 0xB2 && code != 0xB5) return true;
	}
	return false;
}

// Whether the walks decode a picture (PIC_DECODED), by their rule (walk.cuh, walk_b.cuh): an I picture, a P picture with
// forward_f_code != 0, and when B pictures go to the B walk (b_walk) a B picture with both f_codes != 0
bool picture_decoded(const PictureHeader &h, bool b_walk) {
	if (h.type == 1) return true;
	if (h.type == 2) return h.forward_f_code != 0;
	return h.type == 3 && b_walk && h.forward_f_code != 0 && h.backward_f_code != 0;
}

// An entry of an index: picture `pic` (an index into s.pics) and its chain start
struct IndexEntry {
	uint32_t pic, chain_start;
};

// The random-access calls, by the index each serves
enum class Listing {
	Intra,        // decode_intra: the I pictures, each its own chain start
	Pictures,     // decode_pictures: the pictures decode() reconstructs under the current decode_b, with a chain start
	Macroblocks,  // decode_macroblocks: B pictures whatever decode_b says, no chain start needed (a picture's
	              // macroblock layer depends on its own bits only)
	Accumulated,  // decode_accumulated: the I and P pictures of Pictures, whatever decode_b says
};

// The pictures a random-access call can serve now: after the first sequence header, closed, decoded by the walks, and
// with a chain start where the call needs one -- the greatest I picture j <= k such that at least r(k) pictures of
// [j, k) are references (I, or P with forward_f_code != 0); r = 0 for I, 1 for P, 2 for B.
std::vector<IndexEntry> list_pictures(const Batch *b, const Stream &s, Listing what) {
	std::vector<IndexEntry> out;
	if (!s.has_seq) return out;
	std::vector<uint32_t> keys;      // the I pictures after the sequence header so far
	std::vector<uint32_t> refs_upto;  // refs_upto[k]: references among pictures [0, k)
	uint32_t refs = 0;
	for (uint32_t k = 0; k < s.pics.size(); k++) {
		refs_upto.push_back(refs);
		const PictureHeader h = picture_header(s, s.pics[k]);
		const bool after = s.pics[k] >= s.seq_floor;
		if (after && h.type == 1) keys.push_back(k);
		refs += h.type == 1 || (h.type == 2 && h.forward_f_code != 0);
		const bool listed = what == Listing::Intra         ? h.type == 1
		                    : what == Listing::Accumulated ? picture_decoded(h, false)
		                                                   : picture_decoded(h, what == Listing::Macroblocks || b->decode_b);
		if (!after || !listed || !picture_closed(s, k)) continue;
		if (what == Listing::Macroblocks) {
			out.push_back({k, k});
			continue;
		}
		const uint32_t need = h.type == 1 ? 0 : h.type - 1;
		// (every key is a reference: this looks at most three keys back)
		for (auto j = keys.rbegin(); j != keys.rend(); ++j)
			if (refs_upto[k] - refs_upto[*j] >= need) {
				out.push_back({k, *j});
				break;
			}
	}
	return out;
}

// What a random-access call reports per request (picture_info_t's status, n_present and error)
struct RequestInfo {
	std::vector<int32_t> status, n_present, error;
	explicit RequestInfo(int n) : status(n, 0), n_present(n, 0), error(n, 0) {}
	void set(int i, const picture_info_t &e) {
		status[i] = e.status;
		n_present[i] = e.n_present;
		error[i] = e.error;
	}
	// into the caller's arrays, those that are not nullptr
	void copy_out(int32_t *status_out, int32_t *n_present_out, int32_t *error_out) const {
		if (status_out) std::copy(status.begin(), status.end(), status_out);
		if (n_present_out) std::copy(n_present.begin(), n_present.end(), n_present_out);
		if (error_out) std::copy(error.begin(), error.end(), error_out);
	}
};

// One request: picture `pic` of stream `stream`, decoded by a fresh decoder from picture `from` (its chain start) on
struct PictureRequest {
	int stream;
	uint32_t pic, from;
};

// One chain of the random-access schedule: the requests with the same stream and chain start
struct Chain {
	int stream;
	uint32_t first, last;  // chain start, last requested picture
	uint32_t b_end;        // last requested B picture + 1; 0: none (B pictures after it are not reconstructed)
	int req_lo, req_hi;    // its requests: order[req_lo .. req_hi)
	int req_next;          // the first of them not consumed yet
	int n_sets;            // sets from the caller's pool: 0 (a leaf: its one picture goes to its destination), 2, 4
	uint8_t *set[4];       // (seek_pictures: none, its chains use their streams' sets)
	int cur, b_cur;        // as Stream::cur / b_cur
	const uint2 *map;      // decode_accumulated: the map of the newest reference picture (nullptr: none yet)
	uint32_t next;         // the picture decode() consumes next; beyond `last`: the chain is done
	std::vector<picture_info_t> info;  // per picture of the chain, once parsed
	std::vector<int> slot;
};

// The picture decode() consumes after the one whose info is `e`: the first picture start code at or after where its
// parse ended
uint32_t next_picture(const Stream &s, const picture_info_t &e) {
	return (uint32_t)(std::lower_bound(s.pics.begin(), s.pics.end(), (e.end_bit + 7) >> 3) - s.pics.begin());
}

// The requests in chain order (by stream, chain start and picture) and their chains, with n_sets 0 for a chain of one
// picture and 2 (4 with a B picture requested) otherwise
std::vector<Chain> make_chains(const Batch *b, const std::vector<PictureRequest> &req, std::vector<int> &order) {
	const int n = (int)req.size();
	order.resize(n);
	for (int i = 0; i < n; i++) order[i] = i;
	std::sort(order.begin(), order.end(), [&](int x, int y) {
		const PictureRequest &p = req[x], &q = req[y];
		return p.stream != q.stream ? p.stream < q.stream : p.from != q.from ? p.from < q.from : p.pic != q.pic ? p.pic < q.pic : x < y;
	});
	std::vector<Chain> chains;
	for (int lo = 0; lo < n;) {
		const PictureRequest &r = req[order[lo]];
		int hi = lo + 1;
		while (hi < n && req[order[hi]].stream == r.stream && req[order[hi]].from == r.from) hi++;
		const Stream &s = b->streams[r.stream];
		Chain c{};
		c.stream = r.stream;
		c.first = c.next = r.from;
		c.last = req[order[hi - 1]].pic;
		for (int i = lo; i < hi; i++)
			if (picture_header(s, s.pics[req[order[i]].pic]).type == 3) c.b_end = req[order[i]].pic + 1;
		c.req_lo = c.req_next = lo;
		c.req_hi = hi;
		c.n_sets = c.last == c.first ? 0 : (c.b_end ? 4 : 2);
		c.info.resize(c.last - c.first + 1);
		c.slot.resize(c.last - c.first + 1);
		chains.push_back(std::move(c));
		lo = hi;
	}
	return chains;
}

// What a caller of run_chains does with the pictures its chains consume
struct ChainWork {
	// picture e of chain `ch` (stream s) is consumed and decoded, the d-th of its chain in this wave: records in `slot`,
	// named by requests order[q_lo .. q_hi)
	virtual void picture(Chain &ch, const Stream &s, int slot, const picture_info_t &e, size_t d, int q_lo, int q_hi) = 0;
	// the wave's depths, one after the other on the reconstruct stream (run_steps)
	virtual void depths() = 0;
	virtual ~ChainWork() = default;
};

// Where run_chains takes each chain's n_sets plane or map sets from: `set_bytes` each out of `buf`, zeroed first when
// `zero`
struct SetPool {
	DeviceBuffer<uint8_t> &buf;
	size_t set_bytes;
	bool zero;
};

// The schedule behind decode_pictures, decode_intra, decode_accumulated and seek_pictures (DESIGN 3.7).  The chains'
// pictures [first, last] are parsed in waves over consecutive positions of every chain, consumed on the host by
// decode()'s rule (b_walk: B pictures go to the B walk, as decode_b; else they are skipped after their header) and
// handed to `work` by depth (depth d: the d-th decoded picture of every chain of the wave).  Chains run in groups of at
// most a wave's slots.  With a `pool`, each chain's sets come from it, a group's within half of the free device memory
// -- a request beyond the device is cut into groups, not refused; without one, `work` uses sets of its own.  The
// requests are valid (the caller checked them); on return the work is queued on the reconstruct stream, and the infos
// are the consumed pictures'.
RequestInfo run_chains(Batch *b, const std::vector<PictureRequest> &req, const std::vector<int> &order,
                       std::vector<Chain> &chains, bool b_walk, const SetPool *pool, ChainWork &work) {
	size_t n_tasks = 0;
	for (const Chain &c : chains) n_tasks += c.info.size();
	RequestInfo out((int)req.size());
	free_slots_for(b, n_tasks);
	const int wave_max = (int)b->free_slots.size();
	size_t max_sets = SIZE_MAX;
	if (pool) {
		size_t free_b = 0, total_b = 0;
		CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
		max_sets = std::max<size_t>(4, ((size_t)(0.5 * (double)free_b) + pool->buf.size()) / pool->set_bytes);
	}
	std::vector<std::pair<size_t, size_t>> groups;
	size_t most_sets = 0;
	for (size_t lo = 0; lo < chains.size();) {
		size_t hi = lo, sets = 0;
		while (hi < chains.size() && hi - lo < (size_t)wave_max && sets + chains[hi].n_sets <= max_sets) sets += chains[hi++].n_sets;
		groups.push_back({lo, hi});
		most_sets = std::max(most_sets, sets);
		lo = hi;
	}
	if (pool && most_sets * pool->set_bytes > pool->buf.size()) {
		if (pool->buf.data()) CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
		pool->buf.reserve(most_sets * pool->set_bytes);
	}
	for (const auto &[glo, ghi] : groups) {
		size_t sets = 0;
		if (pool)
			for (size_t c = glo; c < ghi; c++)
				for (int k = 0; k < chains[c].n_sets; k++) chains[c].set[k] = pool->buf.data() + pool->set_bytes * sets++;
		if (sets && pool->zero)  // (the previous group's copies are queued before)
			CUDA_CHECK(cudaMemsetAsync(pool->buf.data(), 0, pool->set_bytes * sets, b->st_recon));
		const uint32_t width = (uint32_t)std::max<size_t>(1, (size_t)wave_max / (ghi - glo));
		for (uint32_t lo = 0;; lo += width) {
			// ---- stage 1: positions [lo, lo + width) of every chain still consuming
			std::vector<WaveItem> wave;
			std::vector<int> wave_chain;  // the chain of each picture of the wave
			for (size_t c = glo; c < ghi; c++) {
				Chain &ch = chains[c];
				if (ch.next > ch.last) continue;
				for (uint32_t p = ch.first + lo; p <= ch.last && p - ch.first < lo + width; p++) {
					wave.push_back(take_slot(b, ch.stream, p, b_walk));
					ch.slot[p - ch.first] = wave.back().slot;
					wave_chain.push_back((int)c);
				}
			}
			if (wave.empty()) break;
			parse_wave(b, wave, true);
			for (size_t t = 0; t < wave.size(); t++) {
				Chain &ch = chains[wave_chain[t]];
				ch.info[wave[t].pic - ch.first] = b->h_info[t];
			}
			// ---- decode()'s consumption rule over the infos (decode_round): which pictures are decoded, at which depth
			for (size_t c = glo; c < ghi; c++) {
				Chain &ch = chains[c];
				const Stream &s = b->streams[ch.stream];
				const uint32_t parsed_end = std::min(ch.last + 1, ch.first + lo + width);
				size_t d = 0;
				while (ch.next < parsed_end) {
					const uint32_t k = ch.next;
					const picture_info_t &e = ch.info[k - ch.first];
					while (ch.req_next < ch.req_hi && req[order[ch.req_next]].pic < k) ch.req_next++;  // passed over: status 0
					const int q_lo = ch.req_next;
					while (ch.req_next < ch.req_hi && req[order[ch.req_next]].pic == k) ch.req_next++;
					const int q_hi = ch.req_next;
					for (int q = q_lo; q < q_hi; q++) out.set(order[q], e);
					const bool is_b = e.picture_type == 3;  // (only the B walk answers PIC_DECODED for one)
					if (e.status == PIC_DECODED && (!is_b || k < ch.b_end))
						work.picture(ch, s, ch.slot[k - ch.first], e, d++, q_lo, q_hi);
					ch.next = next_picture(s, e);
				}
			}
			// ---- stage 2 (run_steps), then the slots go back: the next wave's parse waits for ev_round
			work.depths();
			for (const WaveItem &w : wave) release_slot(b, w.slot);
		}
	}
	return out;
}

// decode_pictures and decode_intra: each depth is one launch_reconstruct, followed by the copies of its requested
// pictures.  A requested picture is copied to its destination right behind its launch -- or, in a chain that
// reconstructs nothing else, reconstructed straight into it.
struct PlaneWork : ChainWork {
	Batch *b;
	const std::vector<int> &order;
	void *const *planes_dst, *const *rgba_dst;
	bool rgba;
	std::vector<ReconStep> steps;
	PlaneWork(Batch *b, const std::vector<int> &order, void *const *planes_dst, void *const *rgba_dst, bool rgba)
	    : b(b), order(order), planes_dst(planes_dst), rgba_dst(rgba_dst), rgba(rgba) {}
	void picture(Chain &ch, const Stream &s, int slot, const picture_info_t &e, size_t d, int q_lo, int q_hi) override {
		const bool is_b = e.picture_type == 3;
		const bool leaf = ch.n_sets == 0;
		uint8_t *out_rgba = rgba && q_hi > q_lo ? static_cast<uint8_t *>(rgba_dst[order[q_lo]]) : nullptr;
		ReconTask t;
		if (is_b)  // the two I/P sets: `cur` the older (forward), `1 - cur` the newer (backward) reference
			t = recon_task(b, s, slot, ch.set[2 + ch.b_cur], ch.set[ch.cur], ch.set[1 - ch.cur], out_rgba);
		else if (leaf)  // into the destination, predicted (skipped macroblocks) from the zeroed scratch set
			t = recon_task(b, s, slot, static_cast<uint8_t *>(planes_dst[order[q_lo]]), b->d_intra_fwd.data(), nullptr, out_rgba);
		else
			t = recon_task(b, s, slot, ch.set[ch.cur], ch.set[1 - ch.cur], nullptr, out_rgba);
		if (steps.size() <= d) steps.emplace_back();
		ReconStep &dp = steps[d];
		dp.conceal(t, s, e, b->conceal && !leaf);  // (a leaf's forward set is the zeroed scratch and its destination is zeroed)
		dp.tasks.push_back(t);
		for (int q = q_lo; q < q_hi; q++) {  // the first request gets the picture, duplicates a copy of it
			if (!leaf || q > q_lo) dp.copy(planes_dst[order[q]], t.cur.y, (size_t)s.coded_size * 3 / 2);
			if (rgba && q > q_lo) dp.copy(rgba_dst[order[q]], t.rgba, (size_t)s.width * s.height * 4);
		}
		if (is_b) ch.b_cur ^= 1;
		else ch.cur ^= 1;
	}
	// (a set is overwritten two references later, by a later launch on the same stream)
	void depths() override {
		run_steps(b, steps, false);
		steps.clear();
	}
};

// decode_pictures and decode_intra (DESIGN 3.6, 3.7): run_chains with plane sets, B pictures as decode_b says
void decode_chains(Batch *b, const std::vector<PictureRequest> &req, void *const *planes_dst, void *const *rgba_dst,
                   bool rgba, int32_t *status_out, int32_t *n_present_out, int32_t *error_out) {
	ensure_pool(b);
	std::vector<int> order;
	std::vector<Chain> chains = make_chains(b, req, order);
	size_t set_bytes = 0;
	bool leaves = false;
	for (const Chain &c : chains) {
		const Stream &s = b->streams[c.stream];
		leaves |= c.n_sets == 0;
		// + coded_width + 64: parse_sequence_header's slack; a multiple of 256 keeps every set of the pool aligned
		set_bytes = std::max(set_bytes, ((size_t)s.coded_size * 3 / 2 + s.seq.coded_width + 64 + 255) & ~(size_t)255);
	}
	if (leaves && set_bytes > b->d_intra_fwd.size()) {
		if (b->d_intra_fwd.data()) CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
		b->d_intra_fwd.reserve(set_bytes);
		CUDA_CHECK(cudaMemsetAsync(b->d_intra_fwd.data(), 0, set_bytes, b->st_recon));
	}
	// what a request that is never consumed keeps: planes 0, RGBA opaque white.  A leaf is reconstructed into its
	// destination, whose absent macroblocks keep that 0; every other destination is written whole by a copy.
	for (const Chain &c : chains)
		for (int q = c.req_lo; q < c.req_hi; q++) {
			const int i = order[q];
			const Stream &s = b->streams[req[i].stream];
			if (c.n_sets == 0) CUDA_CHECK(cudaMemsetAsync(planes_dst[i], 0, (size_t)s.coded_size * 3 / 2, b->st_recon));
			if (rgba) CUDA_CHECK(cudaMemsetAsync(rgba_dst[i], 0xff, (size_t)s.width * s.height * 4, b->st_recon));
		}
	PlaneWork work(b, order, planes_dst, rgba_dst, rgba);
	// (a fresh decoder's planes start zeroed, the B sets too)
	const SetPool pool{b->d_chain_sets, set_bytes, true};
	const RequestInfo out = run_chains(b, req, order, chains, b->decode_b, &pool, work);
	for (const Chain &c : chains)  // never consumed: planes 0 (a copied destination was not zeroed)
		if (c.n_sets)
			for (int q = c.req_lo; q < c.req_hi; q++)
				if (out.status[order[q]] == 0) {
					const Stream &s = b->streams[c.stream];
					CUDA_CHECK(cudaMemsetAsync(planes_dst[order[q]], 0, (size_t)s.coded_size * 3 / 2, b->st_recon));
				}
	CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
	b->recon_pending = false;
	out.copy_out(status_out, n_present_out, error_out);
}

// seek_pictures' chain start for entry `e` of the picture index: the index's, except that under decode_b an I picture
// needs one reference in [j, k) -- the greatest I picture before it, or k itself where there is none -- so that the B
// pictures after it (of an open GOP) are decoded from both their references (DESIGN 3.12)
uint32_t seek_start(const Batch *b, const Stream &s, const IndexEntry &e) {
	if (!b->decode_b || e.pic != e.chain_start) return e.chain_start;
	for (uint32_t j = e.pic; j-- > 0;)
		if (s.pics[j] >= s.seq_floor && picture_header(s, s.pics[j]).type == 1) return j;
	return e.pic;
}

// The checks of a random-access call's requests, all before anything changes: the arrays are there; every request
// names a stream with a sequence header and a picture of its `what` listing; and the first `n_dst` of the destination
// arrays -- `dst` (seek_pictures has none) and an optional second one, `dst2` (decode_intra and decode_pictures under
// OUT_RGBA: the images; the exports: mb_dst) -- are there with every destination 16-byte aligned (stage 2 and the
// exports store 8 and 16 bytes at a time).  Fills `req` (with the chain starts) and returns true, or returns false.
bool check_requests(Batch *b, Listing what, int n, const int *streams, const uint32_t *pictures,
                    std::vector<PictureRequest> &req, int n_dst = 0, void *const *dst = nullptr, void *const *dst2 = nullptr) {
	void *const *const arrays[2] = {dst, dst2};
	for (int k = 0; k < n_dst; k++)
		if (n > 0 && !arrays[k]) return false;
	use_device(b);
	if (n < 0 || (n > 0 && (!streams || !pictures))) return false;
	upload_all(b);
	std::vector<std::vector<IndexEntry>> listed(b->streams.size());
	std::vector<char> indexed(b->streams.size(), 0);
	req.resize(n);
	for (int i = 0; i < n; i++) {
		const int si = streams[i];
		if (si < 0 || si >= (int)b->streams.size() || !b->streams[si].has_seq) return false;
		if (!indexed[si]) {
			listed[si] = list_pictures(b, b->streams[si], what);
			indexed[si] = 1;
		}
		auto e = std::lower_bound(listed[si].begin(), listed[si].end(), pictures[i],
		                          [](const IndexEntry &x, uint32_t k) { return x.pic < k; });
		if (e == listed[si].end() || e->pic != pictures[i]) return false;
		req[i] = {si, pictures[i], e->chain_start};
	}
	for (int k = 0; k < n_dst; k++)
		for (int i = 0; i < n; i++)
			if (!arrays[k][i] || ((uintptr_t)arrays[k][i] & 15u) != 0) return false;
	return true;
}

// decode_intra (`intra`: requests are looked up in the intra index) and decode_pictures (in the picture index)
long batch_decode_chosen(Batch *b, bool intra, int n, const int *streams, const uint32_t *pictures, void *const *planes_dst,
                         void *const *rgba_dst, int flags, int32_t *status_out, int32_t *n_present_out, int32_t *error_out) {
	const bool rgba = (flags & JSMPEG_B200_OUT_RGBA) != 0;
	std::vector<PictureRequest> req;
	const Listing what = intra ? Listing::Intra : Listing::Pictures;
	if (!check_requests(b, what, n, streams, pictures, req, rgba ? 2 : 1, planes_dst, rgba_dst)) return -2;
	if (n == 0) return 0;
	decode_chains(b, req, planes_dst, rgba_dst, rgba, status_out, n_present_out, error_out);
	return n;
}

// ---- decode_macroblocks, decode_coefficients, decode_residuals: the walks' records of chosen pictures of any streams,
// in the public layouts (DESIGN 3.8, 3.9, 3.10) ----

// What an export call writes into its required destinations
enum class Export { Macroblocks, Coefficients, Residuals };

// Each unique (stream, picture) of the requests takes a record slot; waves of as many as there are free slots (after
// flushing the look-ahead when they do not cover the call) run the walks alone -- or, for coefficients and residuals,
// the walks and the expand.  Each wave is then one stage-2 step without reconstruct tasks (run_steps): one export
// launch per destination kind, on the reconstruct stream behind the wave (ev_b), writes every request of the wave to
// its destination.  `dst` gets what `what` names; `mb_dst` (nullptr: none) gets the macroblock entries too.  The
// slots go back right after: the next wave's stage 1 waits for ev_round, so it rewrites them (records, dense records
// and -- through its walks and expands -- the compact planes) only after the exports read them.  The requests are
// valid (the caller checked them).
void decode_macroblocks(Batch *b, const std::vector<PictureRequest> &req, Export what, void *const *dst,
                        void *const *mb_dst, int32_t *n_present_out, int32_t *error_out) {
	const int n = (int)req.size();
	ensure_pool(b);
	std::vector<std::pair<int, uint32_t>> uniq(n);
	for (int i = 0; i < n; i++) uniq[i] = {req[i].stream, req[i].pic};
	std::sort(uniq.begin(), uniq.end());
	uniq.erase(std::unique(uniq.begin(), uniq.end()), uniq.end());
	std::vector<size_t> uniq_of(n);  // request i describes picture uniq[uniq_of[i]]
	for (int i = 0; i < n; i++)
		uniq_of[i] = std::lower_bound(uniq.begin(), uniq.end(), std::make_pair(req[i].stream, req[i].pic)) - uniq.begin();
	free_slots_for(b, uniq.size());
	void *const *entries_dst = what == Export::Macroblocks ? dst : mb_dst;
	const size_t wave_max = b->free_slots.size();
	RequestInfo out(n);
	for (size_t lo = 0; lo < uniq.size(); lo += wave_max) {
		const size_t hi = std::min(uniq.size(), lo + wave_max);
		std::vector<WaveItem> wave;
		for (size_t u = lo; u < hi; u++) wave.push_back(take_slot(b, uniq[u].first, uniq[u].second, true));
		parse_wave(b, wave, what != Export::Macroblocks);
		std::vector<ReconStep> steps(1);
		for (int i = 0; i < n; i++) {  // in request order: a duplicate gets tasks of its own
			if (uniq_of[i] < lo || uniq_of[i] >= hi) continue;
			const WaveItem &w = wave[uniq_of[i] - lo];
			const picture_info_t &info = b->h_info[uniq_of[i] - lo];
			out.set(i, info);
			const SeqParams &seq = b->streams[w.stream].seq;
			const SlotRecords sr = slot_records(b, w.slot);
			if (entries_dst) steps[0].entry(sr, seq.mb_size, info.picture_type, entries_dst[i]);
			if (what == Export::Coefficients) steps[0].coef(sr, seq.mb_size, dst[i]);
			if (what == Export::Residuals) steps[0].residual(sr, seq, static_cast<int16_t *>(dst[i]));
		}
		run_steps(b, steps, false);
		for (const WaveItem &w : wave) release_slot(b, w.slot);
	}
	CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
	b->recon_pending = false;
	out.copy_out(nullptr, n_present_out, error_out);
}

// The export calls' requests: pictures of the macroblock index, with the required destinations `dst` and the optional
// `mb_dst` (decode_coefficients, decode_residuals) checked as decode_pictures' are
long batch_decode_macroblocks(Batch *b, Export what, int n, const int *streams, const uint32_t *pictures, void *const *dst,
                              void *const *mb_dst, int32_t *n_present_out, int32_t *error_out) {
	std::vector<PictureRequest> req;
	if (!check_requests(b, Listing::Macroblocks, n, streams, pictures, req, mb_dst ? 2 : 1, dst, mb_dst)) return -2;
	if (n == 0) return 0;
	decode_macroblocks(b, req, what, dst, mb_dst, n_present_out, error_out);
	return n;
}

// ---- decode_accumulated: chosen I and P pictures traced back to their key picture (DESIGN 3.11) ------------------

// Each depth is one accumulate launch over the chains' pictures of that depth.  A requested picture's map is written
// straight into its first destination, duplicates get a copy of it; an unrequested one's goes to the chain's scratch set
// `cur` (the other set holds the map it reads, or an older one).  The next depth of the chain reads it where it is.
struct MapWork : ChainWork {
	Batch *b;
	const std::vector<int> &order;
	void *const *acc_dst;
	std::vector<ReconStep> steps;  // per depth: its maps and copies, no reconstruct task
	MapWork(Batch *b, const std::vector<int> &order, void *const *acc_dst) : b(b), order(order), acc_dst(acc_dst) {}
	void picture(Chain &ch, const Stream &s, int slot, const picture_info_t &, size_t d, int q_lo, int q_hi) override {
		uint2 *out;
		if (q_hi > q_lo) {
			out = static_cast<uint2 *>(acc_dst[order[q_lo]]);
		} else {
			out = reinterpret_cast<uint2 *>(ch.set[ch.cur]);
			ch.cur ^= 1;
		}
		if (steps.size() <= d) steps.emplace_back();
		steps[d].map(slot_records(b, slot), s.seq, ch.map, out);
		ch.map = out;
		for (int q = q_lo + 1; q < q_hi; q++) steps[d].copy(acc_dst[order[q]], out, (size_t)s.coded_size * 12);
	}
	void depths() override {
		run_steps(b, steps, false);
		steps.clear();
	}
};

// run_chains with two scratch map sets per chain (none for a chain of one picture) and B pictures skipped after their
// header, whatever decode_b says.  The requests are valid (the caller checked them).
void decode_accumulated(Batch *b, const std::vector<PictureRequest> &req, void *const *acc_dst, int32_t *status_out,
                        int32_t *n_present_out, int32_t *error_out) {
	ensure_pool(b);
	std::vector<int> order;
	std::vector<Chain> chains = make_chains(b, req, order);
	size_t set_bytes = 0;
	for (Chain &c : chains) {
		c.n_sets = c.n_sets ? 2 : 0;  // (no B picture is requested)
		set_bytes = std::max(set_bytes, ((size_t)b->streams[c.stream].coded_size * 12 + 255) & ~(size_t)255);
	}
	MapWork work(b, order, acc_dst);
	// (a scratch set is read only after the chain wrote it)
	const SetPool pool{b->d_map_sets, set_bytes, false};
	const RequestInfo out = run_chains(b, req, order, chains, false, &pool, work);
	for (int i = 0; i < (int)req.size(); i++)  // never consumed: every record untraced {0, 0, 0, -1}
		if (out.status[i] != PIC_DECODED)
			fill_untraced(static_cast<uint2 *>(acc_dst[i]), (size_t)b->streams[req[i].stream].coded_size * 3 / 2, b->st_recon);
	CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
	b->recon_pending = false;
	out.copy_out(status_out, n_present_out, error_out);
}

// decode_accumulated's requests: decode_pictures' checks over the I and P pictures, and no chain of more than 32,767
// reference pictures (`back` is int16)
long batch_decode_accumulated(Batch *b, int n, const int *streams, const uint32_t *pictures, void *const *acc_dst,
                              int32_t *status_out, int32_t *n_present_out, int32_t *error_out) {
	std::vector<PictureRequest> req;
	if (!check_requests(b, Listing::Accumulated, n, streams, pictures, req, 1, acc_dst)) return -2;
	std::map<std::pair<int, uint32_t>, uint32_t> chain_last;  // per (stream, chain start): the last picture requested
	for (const PictureRequest &r : req) {
		uint32_t &last = chain_last[{r.stream, r.from}];
		last = std::max(last, r.pic);
	}
	for (const auto &[key, last] : chain_last) {
		const Stream &s = b->streams[key.first];
		uint32_t refs = 0;
		for (uint32_t k = key.second; k <= last; k++) {
			const PictureHeader h = picture_header(s, s.pics[k]);
			refs += h.type == 1 || (h.type == 2 && h.forward_f_code != 0);
		}
		if (refs > 32767) return -2;
	}
	if (n == 0) return 0;
	decode_accumulated(b, req, acc_dst, status_out, n_present_out, error_out);
	return n;
}

// ---- seek_pictures: move decode() of chosen streams to a listed picture, each from its seek chain start (DESIGN 3.12)

// Each chain is consumed by decode()'s consume_picture into its stream's own sets, with the stream's rotation.  The last
// picture a chain consumes -- picture k, or on damaged input the picture whose walk ran across k -- is the visible one.
// No later launch of the call writes its set.
struct SeekWork : ChainWork {
	Batch *b;
	int flags;
	std::vector<ReconStep> steps;
	std::vector<TaskAt> newest;  // per stream: its newest picture of the wave (OUT_RESIDUALS)
	SeekWork(Batch *b, int flags) : b(b), flags(flags), newest(b->streams.size()) {}
	void picture(Chain &ch, const Stream &, int slot, const picture_info_t &e, size_t d, int, int) override {
		Stream &s = b->streams[ch.stream];
		consume_picture(b, s, steps, d, slot, e, flags, next_picture(s, e) > ch.last, newest[ch.stream]);  // (no stats)
	}
	void depths() override {
		for (size_t si = 0; si < newest.size(); si++) {  // as decode_round: each stream's newest picture of the wave
			if ((flags & JSMPEG_B200_OUT_RESIDUALS) && newest[si].step >= 0)
				steps[newest[si].step].tasks[newest[si].task].res = reserve_residuals(b, b->streams[si]);
			newest[si] = {};
		}
		run_steps(b, steps, (flags & JSMPEG_B200_OUT_HOST) != 0);
		steps.clear();
	}
};

// run_chains over the named streams' own plane sets, zeroed first with the rotation started over, then the commit of
// what else decode() observes: the bit index, last_picture and the flushed look-ahead.  The requests are valid and name
// distinct streams (the caller checked them).
void seek_pictures(Batch *b, std::vector<PictureRequest> &req, int flags, int32_t *status_out, int32_t *n_present_out,
                   int32_t *error_out) {
	ensure_pool(b);
	for (PictureRequest &r : req) r.from = seek_start(b, b->streams[r.stream], {r.pic, r.from});
	std::vector<int> order;
	std::vector<Chain> chains = make_chains(b, req, order);
	// copies of earlier decode() calls (OUT_HOST) may still read the sets; the zeroing and the chains queue behind
	// every earlier reconstruct launch on st_recon
	CUDA_CHECK(cudaStreamSynchronize(b->st_copy));
	for (Chain &c : chains) {
		Stream &s = b->streams[c.stream];
		flush_cache(b, s);
		if (b->decode_b) reserve_b_sets(b, s);
		if (flags & JSMPEG_B200_OUT_MACROBLOCKS) reserve_entries(b, s);
		if (flags & JSMPEG_B200_OUT_ACCUMULATED) reserve_maps(s);
		for (StreamSet &set : s.sets) {  // the fresh decoder's sets: zeroed planes, entries 0 until written, no map
			if (set.planes.data()) CUDA_CHECK(cudaMemsetAsync(set.planes.data(), 0, (size_t)s.coded_size * 3 / 2, b->st_recon));
			if (flags & JSMPEG_B200_OUT_MACROBLOCKS)
				CUDA_CHECK(cudaMemsetAsync(set.entries.data(), 0, set.entries.size(), b->st_recon));
			set.map_written = false;
		}
		s.cur = s.b_cur = 0;
		s.last = 1;
		s.hold.held = false;
		if (flags & JSMPEG_B200_OUT_RESIDUALS) {  // 0 unless the chain reconstructs a picture, like the entries
			reserve_residuals(b, s);
			CUDA_CHECK(cudaMemsetAsync(s.d_res.data(), 0, s.d_res.size() * sizeof(int16_t), b->st_recon));
		}
		c.b_end = c.last + 1;  // every B picture the fresh decoder reconstructs: a set's content is decode() state
	}
	SeekWork work(b, flags);
	RequestInfo out = run_chains(b, req, order, chains, b->decode_b, nullptr, work);
	for (const Chain &c : chains) {
		Stream &s = b->streams[c.stream];
		uint32_t k = c.first;  // the last picture the chain consumed, by decode()'s rule over its infos
		for (uint32_t next; (next = next_picture(s, c.info[k - c.first])) <= c.last;) k = next;
		const picture_info_t &e = c.info[k - c.first];
		s.bb.index = e.end_bit;
		s.last_type = e.picture_type;
		s.last_temporal = (uint64_t)s.pics[k] + 5 < s.bb.length ? picture_header(s, s.pics[k]).temporal_reference : 0;
		const int i = order[c.req_lo];  // (one request per chain)
		out.set(i, e);
		if (k != c.last) out.status[i] = 0;
	}
	CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
	CUDA_CHECK(cudaStreamSynchronize(b->st_copy));
	b->recon_pending = false;
	out.copy_out(status_out, n_present_out, error_out);
}

// seek_pictures' requests: decode_pictures' checks without destinations, and no stream named twice
long batch_seek_pictures(Batch *b, int n, const int *streams, const uint32_t *pictures, int flags, int32_t *status_out,
                         int32_t *n_present_out, int32_t *error_out) {
	std::vector<PictureRequest> req;
	if (!check_requests(b, Listing::Pictures, n, streams, pictures, req)) return -2;
	std::vector<char> named(b->streams.size(), 0);
	for (const PictureRequest &r : req) {
		if (named[r.stream]) return -2;
		named[r.stream] = 1;
	}
	if (n == 0) return 0;
	seek_pictures(b, req, flags, status_out, n_present_out, error_out);
	return n;
}

// The three *_index calls: the `what` listing of `stream`, its first n_max entries into the outputs that are not nullptr.
// Returns the listing's length, -2 for a stream out of range.
long write_index(Batch *b, int stream, Listing what, uint32_t *picture_out, uint32_t *byte_pos_out, int32_t *type_out,
                 int32_t *temporal_reference_out, uint32_t *chain_start_out, long n_max) {
	return guarded<long>(b, -1, [&]() -> long {
		if (stream < 0 || stream >= (int)b->streams.size()) return -2;
		use_device(b);
		upload_all(b);
		const Stream &s = b->streams[stream];
		const std::vector<IndexEntry> listed = list_pictures(b, s, what);
		for (long i = 0; i < std::min<long>((long)listed.size(), n_max); i++) {
			const uint32_t k = listed[i].pic;
			const PictureHeader h = picture_header(s, s.pics[k]);
			if (picture_out) picture_out[i] = k;
			if (byte_pos_out) byte_pos_out[i] = s.pics[k];
			if (type_out) type_out[i] = h.type;
			if (temporal_reference_out) temporal_reference_out[i] = h.temporal_reference;
			if (chain_start_out) chain_start_out[i] = listed[i].chain_start;
		}
		return (long)listed.size();
	});
}

// The planes of the stream's most recent picture: `forward` (mpeg1.c:841-851); with the B-picture extension it may be a
// B picture's own set
PlaneSet latest_planes(const Stream &s) { return plane_set(s, s.sets[s.last].planes.data()); }

int env_int(const char *name, int fallback) {
	const char *e = getenv(name);
	return e && *e ? atoi(e) : fallback;
}

// MPEG-TS in demux_many (tsdemux.cu, DESIGN 3.3): a request is staged only if it holds a whole packet, and owns one
// packet slot per 188 bytes, numbered over the call; a stream's PID table is made on its first TS write.
struct TsFormat {
	using Req = TsReq;
	using Out = TsReqOut;
	Batch *b;
	TsIo &io;
	uint32_t slots = 0;  // of the requests staged so far
	explicit TsFormat(Batch *b) : b(b), io(b->ts_io) {}

	// a partial packet, a resync that wanted more data (ts.js:25-41)
	static std::vector<uint8_t> &leftover(Stream &s) { return s.ts_leftover; }
	static bool stream_id_ok(int) { return true; }
	static bool fits(uint64_t all, uint64_t) { return all < 0xfffff000ull; }  // (positions are 32-bit; a header read may run a few bytes past a request)
	static uint64_t room(uint64_t len) { return len >= 188 ? len : 0; }  // (fewer bytes: not a packet yet, nothing to upload)
	TsReq request(Stream &s, uint32_t base, uint32_t len, int sid) {
		if (!s.ts_bound.data()) {  // the stream's first TS write: no PID bound yet
			s.ts_bound.reserve(8192);
			CUDA_CHECK(cudaMemsetAsync(s.ts_bound.data(), 0, 8192 * sizeof(int16_t), b->st_main));
		}
		const TsReq r{base, (uint32_t)room(len), slots, sid, s.ts_bound.data(), nullptr, 0, 0};
		slots += len / 188;
		return r;
	}
	uint32_t rows(uint32_t n, uint32_t base) {  // entry n carries the call's slot count
		io.h_req[n] = TsReq{base, 0, slots, 0, nullptr, nullptr, 0, 0};
		return n + 1;
	}
	void begin(uint32_t n, uint32_t) {
		if (!b->ts) b->ts.reset(ts_scratch_create());
		ts_call_begin(b->ts.get(), io, n, slots, (uint32_t)b->streams.size());
	}
	uint32_t measure() {
		const uint32_t launches = ts_call_measure(b->ts.get(), io, b->st_main);
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));
		return launches;
	}
	uint32_t gather() { return ts_call_gather(b->ts.get(), io, ES_PAD, b->st_main); }
	static uint32_t carry(Stream &, const TsReqOut &o) { return o.stop; }
};

// MPEG program streams in demux_many (psdemux.cu, DESIGN 3.5): every request is staged, at a 16-byte aligned offset
// (the candidate search reads 16-byte vectors), with its stream's in-sync state; the candidate counts size the
// rest of the measure step, so they come to the host first.
struct PsFormat {
	using Req = PsReq;
	using Out = PsReqOut;
	Batch *b;
	PsIo &io;
	explicit PsFormat(Batch *b) : b(b), io(b->ps_io) {}

	// an unfinished item, or the tail that may begin a pack header
	static std::vector<uint8_t> &leftover(Stream &s) { return s.ps_leftover; }
	static bool stream_id_ok(int sid) { return sid >= 0xE0 && sid <= 0xEF; }
	static bool fits(uint64_t all, uint64_t staged) { return all < 0xfffff000ull && staged < 0xfffff000ull; }  // (positions are 32-bit)
	static uint64_t room(uint64_t len) { return (len + 15) & ~15ull; }
	PsReq request(Stream &s, uint32_t base, uint32_t len, int sid) { return PsReq{base, len, sid, s.ps_in_sync ? 1u : 0u, nullptr, 0, 0}; }
	uint32_t rows(uint32_t n, uint32_t) { return n; }
	void begin(uint32_t n, uint32_t staged) {
		if (!b->ps) b->ps.reset(ps_scratch_create());
		ps_call_begin(b->ps.get(), n, staged);
	}
	uint32_t measure() {
		uint32_t launches = ps_call_candidates(b->ps.get(), io, b->st_main);
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));
		launches += ps_call_measure(b->ps.get(), io, b->st_main);
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));
		return launches;
	}
	uint32_t gather() { return ps_call_gather(b->ps.get(), io, ES_PAD, b->st_main); }
	static uint32_t carry(Stream &s, const PsReqOut &o) {  // bytes consumed; the stream's in-sync state after them
		s.ps_in_sync = o.in_sync != 0;
		return o.consumed;
	}
};

// jsmpeg_b200_batch_write_ts_many / _write_ps_many (include/jsmpeg_b200.h): request i appends to streams[i] what the
// format's one-request write would.  One pass for all requests (DESIGN 3.3): one batched upload of the staged bytes and
// the request table; the format's measure launches and synchronisation(s) for the per-request results; the host makes
// room in every stream (the write protocol, may expand or evict) and flushes its ordinary writes; one gather launch,
// one batched copy back of the new ES bytes and the PES list, one synchronisation.  The format F (TsFormat, PsFormat)
// says which requests are staged and where (room: a request's bytes in the staging buffer), fills their rows of the
// request table and queues its steps.
template <class F>
long demux_many(Batch *b, int n, const int *streams, const uint8_t *const *data, const size_t *n_bytes, const int *stream_ids,
                long *appended_out, uint64_t *pts_out, uint32_t *offset_out, long n_max, int32_t *n_pes_out) {
	if (n < 0 || (n > 0 && (!streams || !data || !n_bytes))) return -2;
	const int S = (int)b->streams.size();
	std::vector<char> named(S, 0);
	// a request's bytes: what its stream's last write left over, then the new ones
	uint64_t all = 0, staged = 0, left = 0;
	for (int i = 0; i < n; i++) {
		if (streams[i] < 0 || streams[i] >= S || named[streams[i]] || (!data[i] && n_bytes[i] > 0) ||
		    !F::stream_id_ok(stream_ids ? stream_ids[i] : 0xE0))
			return -2;
		named[streams[i]] = 1;
		const uint64_t lo = F::leftover(b->streams[streams[i]]).size();
		all += lo + n_bytes[i];
		staged += F::room(lo + n_bytes[i]);
		left += lo;
	}
	if (!F::fits(all, staged)) return -2;
	for (int i = 0; i < n; i++) {
		if (appended_out) appended_out[i] = 0;
		if (n_pes_out) n_pes_out[i] = 0;
	}
	std::vector<uint32_t> consumed(n, 0);
	long appended = 0;
	if (staged) {  // (else no request has bytes to demultiplex: no GPU work)
		use_device(b);
		F f(b);
		auto &io = f.io;
		io.begin(n + 1, staged, left);  // (TS's table has an entry n)
		std::vector<void *> dst, src;
		std::vector<size_t> size;
		uint32_t base = 0;
		size_t at_left = 0;
		for (int i = 0; i < n; i++) {
			Stream &s = b->streams[streams[i]];
			const std::vector<uint8_t> &lo = F::leftover(s);
			const uint32_t len = (uint32_t)(lo.size() + n_bytes[i]), room = (uint32_t)F::room(len);
			io.h_req[i] = f.request(s, base, len, stream_ids ? stream_ids[i] : 0xE0);
			if (!room) continue;
			// the left-over bytes go up from pinned memory: a left-over buffer is reallocated by nearly every call, and
			// a pageable source whose pages come and go between batched copies faulted the copy on the H100 (DESIGN 3.3)
			if (!lo.empty()) {
				memcpy(io.h_left.data() + at_left, lo.data(), lo.size());
				dst.push_back(io.stage.data() + base), src.push_back(io.h_left.data() + at_left), size.push_back(lo.size());
				at_left += lo.size();
			}
			if (n_bytes[i]) dst.push_back(io.stage.data() + base + lo.size()), src.push_back(const_cast<uint8_t *>(data[i])), size.push_back(n_bytes[i]);
			b->stats.h2d_bytes += len;
			base += room;
		}
		const uint32_t rows = f.rows(n, base);
		f.begin(n, (uint32_t)staged);  // (the format's scratch: every allocation of the call before the upload is queued)
		dst.push_back(io.req.data()), src.push_back(io.h_req.data()), size.push_back(rows * sizeof(typename F::Req));
		copy_batch(b, dst, src, size, b->st_main, cudaMemcpySrcAccessOrderDuringApiCall);
		b->stats.kernel_launches += f.measure();
		// room in every stream's host bit buffer and HBM mirror; its ordinary writes made resident first
		dst.clear(), src.clear(), size.clear();
		std::vector<uint8_t *> hdst(n, nullptr);
		uint32_t n_pes = 0;
		for (int i = 0; i < n; i++) {
			const typename F::Out &o = io.h_out[i];
			n_pes = std::max(n_pes, o.pes_first + o.pes);
			if (!o.total) continue;
			Stream &s = b->streams[streams[i]];
			hdst[i] = static_cast<uint8_t *>(stream_get_write_ptr(b, s, o.total));
			reserve_device_es(b, s, s.bb.length + o.total);
			if (s.d_valid < s.bb.length) {
				dst.push_back(s.d_es.data() + s.d_valid);
				src.push_back(s.bb.bytes + s.d_valid);
				size.push_back(s.bb.length - s.d_valid);
				b->stats.h2d_bytes += s.bb.length - s.d_valid;
				s.d_valid = s.bb.length;
			}
			io.h_req[i].dst = s.d_es.data() + s.bb.length;
			io.h_req[i].es_base = s.bb.length;
		}
		dst.push_back(io.req.data()), src.push_back(io.h_req.data()), size.push_back(rows * sizeof(typename F::Req));
		copy_batch(b, dst, src, size, b->st_main);
		b->stats.kernel_launches += f.gather();
		// the host keeps a mirror of the ES (sequence header parse, EVICT bookkeeping): the new bytes come back
		dst.clear(), src.clear(), size.clear();
		for (int i = 0; i < n; i++) {
			const uint32_t total = io.h_out[i].total;
			if (!total) continue;
			dst.push_back(hdst[i]), src.push_back(io.h_req[i].dst), size.push_back(total);
			b->stats.d2h_bytes += total;
		}
		if (n_pes && (pts_out || offset_out) && n_max > 0) {
			dst.push_back(io.h_pes_offset.data()), src.push_back(io.pes_offset.data()), size.push_back(n_pes * sizeof(uint32_t));
			dst.push_back(io.h_pes_pts.data()), src.push_back(io.pes_pts.data()), size.push_back(n_pes * sizeof(uint64_t));
		}
		if (!dst.empty()) copy_batch(b, dst, src, size, b->st_main);
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));
		long listed = 0;
		for (int i = 0; i < n; i++) {
			Stream &s = b->streams[streams[i]];
			const typename F::Out &o = io.h_out[i];
			consumed[i] = F::carry(s, o);
			if (!o.total) continue;
			stream_did_write(b, s, o.total);
			s.d_valid = s.bb.length;
			appended += o.total;
			if (appended_out) appended_out[i] = o.total;
			if (n_pes_out) n_pes_out[i] = (int32_t)o.pes;
			for (uint32_t k = 0; k < o.pes && listed < n_max; k++, listed++) {
				if (pts_out) pts_out[listed] = io.h_pes_pts[o.pes_first + k];
				if (offset_out) offset_out[listed] = io.h_pes_offset[o.pes_first + k];
			}
		}
	}
	// what the demuxer did not consume stays for the stream's next write
	for (int i = 0; i < n; i++) {
		std::vector<uint8_t> &lo = F::leftover(b->streams[streams[i]]);
		const size_t k = consumed[i];
		if (k <= lo.size()) {
			lo.erase(lo.begin(), lo.begin() + k);
			lo.insert(lo.end(), data[i], data[i] + n_bytes[i]);
		} else {
			lo.assign(data[i] + (k - lo.size()), data[i] + n_bytes[i]);
		}
	}
	return appended;
}

// jsmpeg_b200_batch_write_ts / _write_ps: one request of demux_many.  A stream id the format does not take is refused
// before anything changes; any other refusal (a stream out of range, 4 GiB or more) is a runtime error, `what` its message.
template <class F>
long write_one(Batch *b, int stream, const uint8_t *data, size_t n_bytes, int stream_id, uint64_t *pts_out, uint32_t *offset_out,
               int n_max, int *n_pes, const char *what) {
	if (n_pes) *n_pes = 0;
	return guarded<long>(b, -1, [&]() -> long {
		if (!F::stream_id_ok(stream_id)) return -2;
		int32_t count = 0;
		const long r = demux_many<F>(b, 1, &stream, &data, &n_bytes, &stream_id, nullptr, pts_out && offset_out ? pts_out : nullptr,
		                             pts_out && offset_out ? offset_out : nullptr, n_max, &count);
		if (r == -2) throw std::runtime_error(what);
		if (n_pes) *n_pes = count;
		return r;
	});
}

}  // namespace

// ================================================================================================
// C ABI, part 2 (batch)

extern "C" {

const char *jsmpeg_b200_version(void) { return "jsmpeg_b200 0.2 (sm_90a)"; }

jsmpeg_b200_batch_t *jsmpeg_b200_batch_create(int n_streams, int device, unsigned int max_slots) {
	Batch *b = new Batch();
	b->device = device;
	b->streams.resize(std::max(n_streams, 1));
	b->max_slots_req = max_slots;
	b->decode_b = env_int("JSMPEG_B200_DECODE_B", 0) != 0;
	b->slice_walk = env_int("JSMPEG_B200_SLICE_WALK", 0) != 0;
	b->trace.on = env_int("JSMPEG_B200_HOST_TRACE", 0) != 0;
	try {
		use_device(b);
		CUDA_CHECK(cudaStreamCreateWithFlags(&b->st_main, cudaStreamNonBlocking));
		CUDA_CHECK(cudaStreamCreateWithFlags(&b->st_recon, cudaStreamNonBlocking));
		CUDA_CHECK(cudaStreamCreateWithFlags(&b->st_info, cudaStreamNonBlocking));
		CUDA_CHECK(cudaStreamCreateWithFlags(&b->st_copy, cudaStreamNonBlocking));
		for (auto &st : b->st_side) CUDA_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
		cudaEvent_t *timed[] = {&b->ev_a, &b->ev_b, &b->ev_mid, &b->ev_recon[0], &b->ev_recon[1]};
		for (auto e : timed) CUDA_CHECK(cudaEventCreate(e));
		cudaEvent_t *untimed[] = {&b->ev_step, &b->ev_round, &b->ev_copied[0], &b->ev_copied[1], &b->ev_sfork, &b->ev_sjoin[0], &b->ev_sjoin[1], &b->ev_info};
		for (auto e : untimed) CUDA_CHECK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
		CUDA_CHECK(cudaEventCreateWithFlags(&b->fork.fork, cudaEventDisableTiming));
		for (int i = 0; i < PARSE_GROUPS; i++) {
			CUDA_CHECK(cudaStreamCreateWithFlags(&b->fork.side[i], cudaStreamNonBlocking));
			CUDA_CHECK(cudaEventCreateWithFlags(&b->fork.join[i], cudaEventDisableTiming));
			CUDA_CHECK(cudaEventCreateWithFlags(&b->fork.walked[i], cudaEventDisableTiming));
		}
	} catch (const std::exception &e) {
		mark_dead(b, e.what());  // no usable device: a decoder that answers false, not a dead process
	}
	return b;
}

void jsmpeg_b200_batch_destroy(jsmpeg_b200_batch_t *b) {
	if (!b) return;
	// best effort, nothing here may throw: the context may be the very thing that failed
	(void)cudaSetDevice(b->device);
	(void)cudaDeviceSynchronize();
	for (auto &s : b->streams) if (s.bb.bytes) kPinned.release(s.bb.bytes, kPinned.ctx);
	for (auto e : {b->ev_a, b->ev_b, b->ev_mid, b->ev_recon[0], b->ev_recon[1], b->ev_step, b->ev_round, b->ev_copied[0],
	               b->ev_copied[1], b->ev_sfork, b->ev_sjoin[0], b->ev_sjoin[1], b->fork.fork, b->ev_info}) if (e) cudaEventDestroy(e);
	for (int i = 0; i < PARSE_GROUPS; i++) {
		if (b->fork.join[i]) cudaEventDestroy(b->fork.join[i]);
		if (b->fork.walked[i]) cudaEventDestroy(b->fork.walked[i]);
		if (b->fork.side[i]) cudaStreamDestroy(b->fork.side[i]);
	}
	for (auto st : {b->st_main, b->st_recon, b->st_copy, b->st_info, b->st_side[0], b->st_side[1]}) if (st) cudaStreamDestroy(st);
	delete b;  // the buffers free themselves, after the synchronize above
	(void)cudaGetLastError();
}

const char *jsmpeg_b200_batch_last_error(jsmpeg_b200_batch_t *b) { return (b && b->dead) ? b->error.c_str() : nullptr; }

int jsmpeg_b200_batch_set_option(jsmpeg_b200_batch_t *b, const char *name, int value) {
	if (!b || !name) return -1;
	if (!strcmp(name, "lookahead")) { b->lookahead = std::max(1, value); return 0; }
	if (!strcmp(name, "slice_walk")) { b->slice_walk = value != 0; return 0; }  // (same records either way: nothing to flush)
	if (!strcmp(name, "conceal")) { b->conceal = value != 0; return 0; }  // (stage 2 only: from the next reconstruct step)
	if (!strcmp(name, "decode_b")) {
		if (b->decode_b != (value != 0))
			for (auto &st : b->streams) flush_cache(b, st);  // what was parsed ahead was parsed under the other rule
		b->decode_b = value != 0;
		return 0;
	}
	return -1;
}

void *jsmpeg_b200_batch_get_write_ptr(jsmpeg_b200_batch_t *b, int stream, unsigned int byte_size) {
	void *p = guarded<void *>(b, nullptr, [&]() -> void * {
		use_device(b);
		return stream_get_write_ptr(b, b->streams[stream], byte_size);
	});
	if (p) return p;
	// dead decoder: the caller's memcpy still needs somewhere to go
	b->dead_scratch.resize(std::max<size_t>(byte_size, 1));
	return b->dead_scratch.data();
}

void jsmpeg_b200_batch_did_write(jsmpeg_b200_batch_t *b, int stream, unsigned int byte_size) {
	guarded_void(b, [&] {
		use_device(b);
		stream_did_write(b, b->streams[stream], byte_size);
	});
}

int jsmpeg_b200_batch_get_index(jsmpeg_b200_batch_t *b, int stream) { return (int)b->streams[stream].bb.index; }

void jsmpeg_b200_batch_set_index(jsmpeg_b200_batch_t *b, int stream, unsigned int index) {
	Stream &s = b->streams[stream];
	s.bb.index = index;
	flush_cache(b, s);
	s.hold.held = false;
}

int jsmpeg_b200_batch_stream_info(jsmpeg_b200_batch_t *b, int stream, int *width, int *height, int *coded_size, float *frame_rate) {
	const Stream &s = b->streams[stream];
	if (width) *width = s.width;
	if (height) *height = s.height;
	if (coded_size) *coded_size = s.coded_size;
	if (frame_rate) *frame_rate = s.frame_rate;
	return s.has_seq ? 1 : 0;
}

long jsmpeg_b200_batch_upload(jsmpeg_b200_batch_t *b) {
	return guarded<long>(b, 0, [&] {
		use_device(b);
		return upload_all(b);
	});
}

void jsmpeg_b200_batch_rewind(jsmpeg_b200_batch_t *b) {
	for (auto &s : b->streams) {
		flush_cache(b, s);
		s.pics.clear();
		s.codes.clear();
		s.pic_code.clear();
		s.codes_classified = 0;
		s.scanned = 0;
		s.bb.index = s.has_seq ? s.seq_end_index : 0;  // where did_write left it (mpeg1.c:812-819)
		s.hold.held = false;
	}
}

void jsmpeg_b200_batch_reset(jsmpeg_b200_batch_t *b) {
	guarded_void(b, [&] {
		use_device(b);
		for (auto &s : b->streams) {
			forget_index(b, s);
			s.bb.length = 0;
			s.bb.index = 0;
			s.cur = s.b_cur = 0;
			s.last = 1;
			s.last_type = s.last_temporal = 0;
			s.h_head = -1;
			s.seq_floor = 0;
			s.hold.held = false;
			for (StreamSet &set : s.sets) {  // (zeroed sets: no picture, no map)
				if (set.planes.data()) CUDA_CHECK(cudaMemsetAsync(set.planes.data(), 0, (size_t)s.coded_size * 3 / 2, b->st_main));
				if (set.entries.data()) CUDA_CHECK(cudaMemsetAsync(set.entries.data(), 0, set.entries.size(), b->st_main));
				set.map_written = false;
			}
			for (HostSlot &h : s.ring)
				if (h.entries.data()) memset(h.entries.data(), 0, h.entries.size());
			if (s.d_res.data()) CUDA_CHECK(cudaMemsetAsync(s.d_res.data(), 0, s.d_res.size() * sizeof(int16_t), b->st_main));
		}
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));
	});
}

long jsmpeg_b200_batch_decode(jsmpeg_b200_batch_t *b, int n_pictures, int flags) {
	return guarded<long>(b, 0, [&] { return batch_decode(b, n_pictures, flags); });
}

long jsmpeg_b200_batch_decode_frames(jsmpeg_b200_batch_t *b, int n_pictures, int flags, void *const *planes_dst,
                                     void *const *rgba_dst, void *const *res_dst, void *const *mb_dst,
                                     jsmpeg_b200_frame_t *info_out, int32_t *n_frames_out) {
	const jsmpeg_b200_frame_dst_t dst{planes_dst, rgba_dst, res_dst, mb_dst, nullptr, nullptr};
	return jsmpeg_b200_batch_decode_frames_into(b, n_pictures, flags, &dst, info_out, n_frames_out);
}

namespace {

// The frame cursors of decode_frames_into, decode_frames_display and flush_frames for `dst`, info rows `stride` apart,
// or false -- before any work -- when dst is NULL, n_pictures < 0, a destination is not 16-byte aligned (stage 2 and the
// exports store 8 and 16 bytes at a time), a map destination is given where decode(n, flags) writes no maps, or
// (`display`) a stream holds a picture without a kind the call asks for
bool frame_cursors(const Batch *b, int n_pictures, int flags, const jsmpeg_b200_frame_dst_t *dst, jsmpeg_b200_frame_t *info_out,
                   size_t stride, bool display, std::vector<FrameCursor> &frames) {
	if (!dst || n_pictures < 0) return false;
	const size_t S = b->streams.size();
	auto aligned = [&](void *const *d) {
		for (size_t si = 0; d && si < S; si++)
			if ((uintptr_t)d[si] & 15u) return false;
		return true;
	};
	bool maps = false;
	for (size_t si = 0; dst->acc && si < S; si++) maps |= dst->acc[si] != nullptr;
	if (!aligned(dst->planes) || !aligned(dst->rgba) || !aligned(dst->res) || !aligned(dst->mb) || !aligned(dst->coef) ||
	    !aligned(dst->acc) || (maps && !(flags & JSMPEG_B200_OUT_ACCUMULATED)))
		return false;
	frames.assign(S, FrameCursor{});
	for (size_t si = 0; si < S; si++) {
		FrameCursor &f = frames[si];
		if (dst->planes) f.planes = static_cast<uint8_t *>(dst->planes[si]);
		if (dst->rgba) f.rgba = static_cast<uint8_t *>(dst->rgba[si]);
		if (dst->res) f.res = static_cast<int16_t *>(dst->res[si]);
		if (dst->mb) f.mb = static_cast<uint8_t *>(dst->mb[si]);
		if (dst->coef) f.coef = static_cast<int16_t *>(dst->coef[si]);
		if (dst->acc) f.acc = static_cast<uint2 *>(dst->acc[si]);
		if (info_out) f.info = info_out + si * stride;
		f.display = display;
		f.kinds = (f.planes ? KIND_PLANES : 0) | (f.rgba ? KIND_RGBA : 0) | (f.res ? KIND_RES : 0) | (f.mb ? KIND_MB : 0) |
		          (f.coef ? KIND_COEF : 0) | (f.acc ? KIND_ACC : 0);
		const FrameStore &h = b->streams[si].hold;
		if (display && h.held && (f.kinds & ~h.kinds)) return false;
	}
	return true;
}

}  // namespace

long jsmpeg_b200_batch_decode_frames_into(jsmpeg_b200_batch_t *b, int n_pictures, int flags, const jsmpeg_b200_frame_dst_t *dst,
                                          jsmpeg_b200_frame_t *info_out, int32_t *n_frames_out) {
	return guarded<long>(b, -1, [&]() -> long {
		std::vector<FrameCursor> frames;
		if (!frame_cursors(b, n_pictures, flags, dst, info_out, (size_t)n_pictures, false, frames)) return -2;
		const long got = batch_decode(b, n_pictures, flags, &frames);
		for (size_t si = 0; n_frames_out && si < frames.size(); si++) n_frames_out[si] = frames[si].n;
		return got;
	});
}

long jsmpeg_b200_batch_decode_frames_display(jsmpeg_b200_batch_t *b, int n_pictures, int flags, const jsmpeg_b200_frame_dst_t *dst,
                                             jsmpeg_b200_frame_t *info_out, int32_t *n_frames_out) {
	return guarded<long>(b, -1, [&]() -> long {
		std::vector<FrameCursor> frames;
		if (!frame_cursors(b, n_pictures, flags, dst, info_out, (size_t)n_pictures + 1, true, frames)) return -2;
		const long got = batch_decode(b, n_pictures, flags, &frames);
		for (size_t si = 0; n_frames_out && si < frames.size(); si++) n_frames_out[si] = frames[si].n;
		return got;
	});
}

long jsmpeg_b200_batch_flush_frames(jsmpeg_b200_batch_t *b, const jsmpeg_b200_frame_dst_t *dst, jsmpeg_b200_frame_t *info_out,
                                    int32_t *n_frames_out) {
	return guarded<long>(b, -1, [&]() -> long {
		std::vector<FrameCursor> frames;
		if (!frame_cursors(b, 0, JSMPEG_B200_OUT_ACCUMULATED, dst, info_out, 1, true, frames)) return -2;
		use_device(b);
		std::vector<void *> to, from;
		std::vector<size_t> size;
		long presented = 0;
		for (size_t si = 0; si < frames.size(); si++) {
			Stream &s = b->streams[si];
			FrameCursor &f = frames[si];
			if (!s.hold.held) continue;
			copy_held(s, s.hold.kinds, f.at(s, 0), to, from, size);
			if (f.info) f.info[0] = s.hold.info;
			s.hold.held = false;
			f.n = 1;
			presented++;
		}
		if (!to.empty()) copy_batch(b, to, from, size, b->st_recon);
		CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
		for (size_t si = 0; n_frames_out && si < frames.size(); si++) n_frames_out[si] = frames[si].n;
		return presented;
	});
}

long jsmpeg_b200_batch_intra_index(jsmpeg_b200_batch_t *b, int stream, uint32_t *picture_out, uint32_t *byte_pos_out,
                                   int32_t *temporal_reference_out, long n_max) {
	return write_index(b, stream, Listing::Intra, picture_out, byte_pos_out, nullptr, temporal_reference_out, nullptr, n_max);
}

long jsmpeg_b200_batch_decode_intra(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                    void *const *planes_dst, void *const *rgba_dst, int flags, int32_t *n_present_out,
                                    int32_t *error_out) {
	return guarded<long>(b, -1, [&] {
		return batch_decode_chosen(b, true, n, streams, pictures, planes_dst, rgba_dst, flags, nullptr, n_present_out, error_out);
	});
}

long jsmpeg_b200_batch_picture_index(jsmpeg_b200_batch_t *b, int stream, uint32_t *picture_out, uint32_t *byte_pos_out,
                                     int32_t *type_out, int32_t *temporal_reference_out, uint32_t *chain_start_out,
                                     long n_max) {
	return write_index(b, stream, Listing::Pictures, picture_out, byte_pos_out, type_out, temporal_reference_out,
	                   chain_start_out, n_max);
}

long jsmpeg_b200_batch_decode_pictures(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                       void *const *planes_dst, void *const *rgba_dst, int flags, int32_t *status_out,
                                       int32_t *n_present_out, int32_t *error_out) {
	return guarded<long>(b, -1, [&] {
		return batch_decode_chosen(b, false, n, streams, pictures, planes_dst, rgba_dst, flags, status_out, n_present_out, error_out);
	});
}

long jsmpeg_b200_batch_macroblock_index(jsmpeg_b200_batch_t *b, int stream, uint32_t *picture_out, uint32_t *byte_pos_out,
                                        int32_t *type_out, int32_t *temporal_reference_out, long n_max) {
	return write_index(b, stream, Listing::Macroblocks, picture_out, byte_pos_out, type_out, temporal_reference_out, nullptr,
	                   n_max);
}

long jsmpeg_b200_batch_decode_macroblocks(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                          void *const *mb_dst, int32_t *n_present_out, int32_t *error_out) {
	return guarded<long>(b, -1, [&] {
		return batch_decode_macroblocks(b, Export::Macroblocks, n, streams, pictures, mb_dst, nullptr, n_present_out, error_out);
	});
}

long jsmpeg_b200_batch_decode_coefficients(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                           void *const *coef_dst, void *const *mb_dst, int32_t *n_present_out,
                                           int32_t *error_out) {
	return guarded<long>(b, -1, [&] {
		return batch_decode_macroblocks(b, Export::Coefficients, n, streams, pictures, coef_dst, mb_dst, n_present_out, error_out);
	});
}

long jsmpeg_b200_batch_decode_residuals(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                        void *const *res_dst, void *const *mb_dst, int32_t *n_present_out,
                                        int32_t *error_out) {
	return guarded<long>(b, -1, [&] {
		return batch_decode_macroblocks(b, Export::Residuals, n, streams, pictures, res_dst, mb_dst, n_present_out, error_out);
	});
}

long jsmpeg_b200_batch_decode_accumulated(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                          void *const *acc_dst, int32_t *status_out, int32_t *n_present_out,
                                          int32_t *error_out) {
	return guarded<long>(b, -1, [&] {
		return batch_decode_accumulated(b, n, streams, pictures, acc_dst, status_out, n_present_out, error_out);
	});
}

long jsmpeg_b200_batch_seek_pictures(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures, int flags,
                                     int32_t *status_out, int32_t *n_present_out, int32_t *error_out) {
	return guarded<long>(b, -1, [&] {
		return batch_seek_pictures(b, n, streams, pictures, flags, status_out, n_present_out, error_out);
	});
}

int jsmpeg_b200_batch_get_planes(jsmpeg_b200_batch_t *b, int stream, void **y, void **cr, void **cb) {
	const Stream &s = b->streams[stream];
	if (!s.has_seq) return -1;
	PlaneSet p = latest_planes(s);
	if (y) *y = p.y;
	if (cr) *cr = p.cr;
	if (cb) *cb = p.cb;
	return 0;
}

int jsmpeg_b200_batch_get_host_planes(jsmpeg_b200_batch_t *b, int stream, void **y, void **cr, void **cb) {
	const Stream &s = b->streams[stream];
	if (!s.has_seq) return -1;
	PlaneSet p = plane_set(s, s.ring[s.h_head < 0 ? 0 : s.h_head].planes.data());
	if (y) *y = p.y;
	if (cr) *cr = p.cr;
	if (cb) *cb = p.cb;
	return 0;
}

int jsmpeg_b200_batch_get_rgba(jsmpeg_b200_batch_t *b, int stream, void **rgba) {
	const Stream &s = b->streams[stream];
	if (!s.has_seq || !s.d_rgba.data()) return -1;
	*rgba = s.d_rgba.data();
	return 0;
}

int jsmpeg_b200_batch_read_planes(jsmpeg_b200_batch_t *b, int stream, void *y, void *cr, void *cb) {
	return guarded<int>(b, -1, [&] {
		use_device(b);
		const Stream &s = b->streams[stream];
		if (!s.has_seq) return -1;
		PlaneSet p = latest_planes(s);
		if (y) CUDA_CHECK(cudaMemcpy(y, p.y, s.coded_size, cudaMemcpyDeviceToHost));
		if (cr) CUDA_CHECK(cudaMemcpy(cr, p.cr, s.coded_size >> 2, cudaMemcpyDeviceToHost));
		if (cb) CUDA_CHECK(cudaMemcpy(cb, p.cb, s.coded_size >> 2, cudaMemcpyDeviceToHost));
		return 0;
	});
}

long jsmpeg_b200_batch_write_ts(jsmpeg_b200_batch_t *b, int stream, const uint8_t *ts, size_t n_bytes, int stream_id,
                                uint64_t *pts_out, uint32_t *offset_out, int n_max, int *n_pes) {
	return write_one<TsFormat>(b, stream, ts, n_bytes, stream_id, pts_out, offset_out, n_max, n_pes,
	                           "jsmpeg_b200: write_ts: stream out of range, or a transport stream buffer of 4 GiB or more");
}

long jsmpeg_b200_batch_write_ts_many(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint8_t *const *ts,
                                     const size_t *n_bytes, const int *stream_ids, long *appended_out, uint64_t *pts_out,
                                     uint32_t *offset_out, long n_max, int32_t *n_pes_out) {
	return guarded<long>(b, -1, [&] {
		return demux_many<TsFormat>(b, n, streams, ts, n_bytes, stream_ids, appended_out, pts_out, offset_out, n_max, n_pes_out);
	});
}

long jsmpeg_b200_batch_write_ps(jsmpeg_b200_batch_t *b, int stream, const uint8_t *ps, size_t n_bytes, int stream_id,
                                uint64_t *pts_out, uint32_t *offset_out, int n_max, int *n_pes) {
	return write_one<PsFormat>(b, stream, ps, n_bytes, stream_id, pts_out, offset_out, n_max, n_pes,
	                           "jsmpeg_b200: write_ps: stream out of range, or a program stream buffer of 4 GiB or more");
}

long jsmpeg_b200_batch_write_ps_many(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint8_t *const *ps,
                                     const size_t *n_bytes, const int *stream_ids, long *appended_out, uint64_t *pts_out,
                                     uint32_t *offset_out, long n_max, int32_t *n_pes_out) {
	return guarded<long>(b, -1, [&] {
		return demux_many<PsFormat>(b, n, streams, ps, n_bytes, stream_ids, appended_out, pts_out, offset_out, n_max, n_pes_out);
	});
}

int jsmpeg_b200_batch_read_rgba(jsmpeg_b200_batch_t *b, int stream, void *rgba) {
	return guarded<int>(b, -1, [&] {
		use_device(b);
		const Stream &s = b->streams[stream];
		if (!s.has_seq || !s.d_rgba.data()) return -1;
		CUDA_CHECK(cudaMemcpy(rgba, s.d_rgba.data(), (size_t)s.width * s.height * 4, cudaMemcpyDeviceToHost));
		return 0;
	});
}

// The stream whose entries the three *_macroblocks calls hand out, its entry buffers made (nullptr: out of range or
// no sequence header yet)
static Stream *entries_stream(Batch *b, int stream) {
	if (stream < 0 || stream >= (int)b->streams.size() || !b->streams[stream].has_seq) return nullptr;
	Stream &s = b->streams[stream];
	if (!s.sets[0].entries.data()) {
		use_device(b);
		reserve_entries(b, s);
		CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
	}
	return &s;
}

int jsmpeg_b200_batch_get_macroblocks(jsmpeg_b200_batch_t *b, int stream, void **entries) {
	return guarded<int>(b, -1, [&] {
		const Stream *s = entries_stream(b, stream);
		if (!s) return -1;
		if (entries) *entries = s->sets[s->last].entries.data();
		return 0;
	});
}

int jsmpeg_b200_batch_read_macroblocks(jsmpeg_b200_batch_t *b, int stream, void *dst) {
	return guarded<int>(b, -1, [&] {
		const Stream *s = entries_stream(b, stream);
		if (!s) return -1;
		if (dst) CUDA_CHECK(cudaMemcpy(dst, s->sets[s->last].entries.data(), (size_t)s->seq.mb_size * sizeof(jsmpeg_b200_macroblock_t),
		                               cudaMemcpyDeviceToHost));
		return 0;
	});
}

int jsmpeg_b200_batch_get_host_macroblocks(jsmpeg_b200_batch_t *b, int stream, void **entries) {
	return guarded<int>(b, -1, [&] {
		const Stream *s = entries_stream(b, stream);
		if (!s) return -1;
		if (entries) *entries = s->ring[s->h_head < 0 ? 0 : s->h_head].entries.data();
		return 0;
	});
}

// The residual get / read_residuals hand out, made zeroed on first use (nullptr: stream out of range or no sequence
// header yet)
static int16_t *stream_residuals(Batch *b, int stream) {
	if (stream < 0 || stream >= (int)b->streams.size() || !b->streams[stream].has_seq) return nullptr;
	Stream &s = b->streams[stream];
	use_device(b);
	if (!s.d_res.data()) {
		reserve_residuals(b, s);
		CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
	}
	return s.d_res.data();
}

int jsmpeg_b200_batch_get_residuals(jsmpeg_b200_batch_t *b, int stream, void **res) {
	return guarded<int>(b, -1, [&] {
		int16_t *r = stream_residuals(b, stream);
		if (!r) return -1;
		if (res) *res = r;
		return 0;
	});
}

int jsmpeg_b200_batch_read_residuals(jsmpeg_b200_batch_t *b, int stream, void *dst) {
	return guarded<int>(b, -1, [&] {
		int16_t *r = stream_residuals(b, stream);
		if (!r) return -1;
		if (dst) CUDA_CHECK(cudaMemcpy(dst, r, b->streams[stream].d_res.size() * sizeof(int16_t), cudaMemcpyDeviceToHost));
		return 0;
	});
}

// The map get / read_accumulated hand out: the one beside the set of the stream's newest I/P picture, made on first use
// and filled untraced unless a call with the flag wrote it for that picture (nullptr: stream out of range or no
// sequence header yet)
static uint2 *newest_map(Batch *b, int stream) {
	if (stream < 0 || stream >= (int)b->streams.size() || !b->streams[stream].has_seq) return nullptr;
	Stream &s = b->streams[stream];
	use_device(b);
	reserve_maps(s);
	StreamSet &set = s.sets[1 - s.cur];
	if (!set.map_written) {  // (the earlier calls have synchronised their streams)
		fill_untraced(set.map.data(), set.map.size(), b->st_recon);
		CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
	}
	return set.map.data();
}

int jsmpeg_b200_batch_get_accumulated(jsmpeg_b200_batch_t *b, int stream, void **map) {
	return guarded<int>(b, -1, [&] {
		uint2 *m = newest_map(b, stream);
		if (!m) return -1;
		if (map) *map = m;
		return 0;
	});
}

int jsmpeg_b200_batch_read_accumulated(jsmpeg_b200_batch_t *b, int stream, void *dst) {
	return guarded<int>(b, -1, [&] {
		const uint2 *m = newest_map(b, stream);
		if (!m) return -1;
		if (dst) CUDA_CHECK(cudaMemcpy(dst, m, (size_t)b->streams[stream].coded_size * 3 / 2 * sizeof(uint2), cudaMemcpyDeviceToHost));
		return 0;
	});
}

int jsmpeg_b200_batch_last_picture(jsmpeg_b200_batch_t *b, int stream, int *picture_type, int *temporal_reference) {
	const Stream &s = b->streams[stream];
	if (picture_type) *picture_type = s.last_type;
	if (temporal_reference) *temporal_reference = s.last_temporal;
	return s.last_type ? 0 : -1;
}

void jsmpeg_b200_batch_get_stats(jsmpeg_b200_batch_t *b, jsmpeg_b200_stats_t *out) { *out = b->stats; }
void jsmpeg_b200_batch_reset_stats(jsmpeg_b200_batch_t *b) { b->stats = jsmpeg_b200_stats_t{}; }

// ================================================================================================
// C ABI, part 1 (reference ABI): one stream, synchronous, host-visible planes

struct mpeg1_decoder_t {
	jsmpeg_b200_batch_t *b;
	bool macroblocks = false;  // the "macroblocks" option: decode() also copies the picture's entries to the host
};

// Host placement.  The pinned bit buffers and plane rings of a decoder are touched by the host threads
// that drive it and by the GPU's copy engines; on a two-socket host a GPU hangs off ONE socket, and a
// ring on the other socket costs every D2H byte a trip over the socket interconnect.  This binds the CALLING THREAD -- and with it the threads it
// creates and the pages it first touches from now on -- to the CPUs of the NUMA node of `device`
// (sysfs: /sys/bus/pci/devices/<id>/numa_node, /sys/devices/system/node/node<k>/cpulist), intersected
// with the affinity it already has.  Returns the number of CPUs bound to, 0 if the node is unknown
// (nothing changed), -1 on error.  node_out (may be NULL) receives the node.
int jsmpeg_b200_bind_host_to_device(int device, int *node_out) {
	if (node_out) *node_out = -1;
	char id[32] = {0};
	if (cudaDeviceGetPCIBusId(id, sizeof id, device) != cudaSuccess) { (void)cudaGetLastError(); return -1; }
	for (char *c = id; *c; c++) if (*c >= 'A' && *c <= 'F') *c += 'a' - 'A';
	char path[128];
	snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", id);
	FILE *f = fopen(path, "r");
	int node = -1;
	if (f) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
	if (node < 0) return 0;
	snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
	f = fopen(path, "r");
	if (!f) return 0;
	cpu_set_t want, have, both;
	CPU_ZERO(&want);
	int lo, hi;
	while (fscanf(f, "%d", &lo) == 1) {  // "0-31,64-95"
		hi = lo;
		int ch = fgetc(f);
		if (ch == '-') { if (fscanf(f, "%d", &hi) != 1) hi = lo; ch = fgetc(f); }
		for (int c = lo; c <= hi && c < CPU_SETSIZE; c++) CPU_SET(c, &want);
		if (ch != ',') break;
	}
	fclose(f);
	if (sched_getaffinity(0, sizeof have, &have) != 0) return -1;
	CPU_AND(&both, &want, &have);
	const int n = CPU_COUNT(&both);
	if (n == 0) return 0;
	if (sched_setaffinity(0, sizeof both, &both) != 0) return -1;
	if (node_out) *node_out = node;
	return n;
}

static int g_default_device = -1;  // -1: JSMPEG_B200_DEVICE or 0
void jsmpeg_b200_set_default_device(int device) { g_default_device = device; }

mpeg1_decoder_t *mpeg1_decoder_create(unsigned int buffer_size, bit_buffer_mode_t buffer_mode) {
	int lookahead = env_int("JSMPEG_B200_LOOKAHEAD", 16);
	if (lookahead < 1) lookahead = 1;
	mpeg1_decoder_t *d = new mpeg1_decoder_t();
	d->b = jsmpeg_b200_batch_create(1, g_default_device >= 0 ? g_default_device : env_int("JSMPEG_B200_DEVICE", 0), (unsigned)lookahead + 1);
	d->b->lookahead = lookahead;
	Stream &s = d->b->streams[0];
	s.bb.mode = buffer_mode;
	guarded_void(d->b, [&] {
		if (!bitbuffer::resize(s.bb, buffer_size ? buffer_size : 1, kPinned)) throw std::runtime_error("jsmpeg_b200: bit buffer allocation failed");
	});
	return d;
}

void mpeg1_decoder_destroy(mpeg1_decoder_t *self) {
	if (!self) return;
	jsmpeg_b200_batch_destroy(self->b);
	delete self;
}

const char *jsmpeg_b200_decoder_last_error(mpeg1_decoder_t *self) { return self ? jsmpeg_b200_batch_last_error(self->b) : nullptr; }
int jsmpeg_b200_decoder_set_option(mpeg1_decoder_t *self, const char *name, int value) {
	if (self && name && !strcmp(name, "macroblocks")) {
		self->macroblocks = value != 0;
		return 0;
	}
	return self ? jsmpeg_b200_batch_set_option(self->b, name, value) : -1;
}
void *jsmpeg_b200_decoder_get_macroblocks(mpeg1_decoder_t *self) {
	void *p = nullptr;
	return self && jsmpeg_b200_batch_get_host_macroblocks(self->b, 0, &p) == 0 ? p : nullptr;
}
int jsmpeg_b200_decoder_last_picture(mpeg1_decoder_t *self, int *picture_type, int *temporal_reference) {
	return self ? jsmpeg_b200_batch_last_picture(self->b, 0, picture_type, temporal_reference) : -1;
}

void *mpeg1_decoder_get_write_ptr(mpeg1_decoder_t *self, unsigned int byte_size) {
	return jsmpeg_b200_batch_get_write_ptr(self->b, 0, byte_size);
}
int mpeg1_decoder_get_index(mpeg1_decoder_t *self) { return jsmpeg_b200_batch_get_index(self->b, 0); }
void mpeg1_decoder_set_index(mpeg1_decoder_t *self, unsigned int index) { jsmpeg_b200_batch_set_index(self->b, 0, index); }
void mpeg1_decoder_did_write(mpeg1_decoder_t *self, unsigned int byte_size) { jsmpeg_b200_batch_did_write(self->b, 0, byte_size); }
int mpeg1_decoder_has_sequence_header(mpeg1_decoder_t *self) { return self->b->streams[0].has_seq ? 1 : 0; }
float mpeg1_decoder_get_frame_rate(mpeg1_decoder_t *self) { return self->b->streams[0].frame_rate; }
int mpeg1_decoder_get_coded_size(mpeg1_decoder_t *self) { return self->b->streams[0].coded_size; }
int mpeg1_decoder_get_width(mpeg1_decoder_t *self) { return self->b->streams[0].width; }
int mpeg1_decoder_get_height(mpeg1_decoder_t *self) { return self->b->streams[0].height; }

static void *host_plane(mpeg1_decoder_t *self, int which) {
	void *p[3] = {nullptr, nullptr, nullptr};
	if (jsmpeg_b200_batch_get_host_planes(self->b, 0, &p[0], &p[1], &p[2]) != 0) return nullptr;
	return p[which];
}
void *mpeg1_decoder_get_y_ptr(mpeg1_decoder_t *self) { return host_plane(self, 0); }
void *mpeg1_decoder_get_cr_ptr(mpeg1_decoder_t *self) { return host_plane(self, 1); }
void *mpeg1_decoder_get_cb_ptr(mpeg1_decoder_t *self) { return host_plane(self, 2); }

bool mpeg1_decoder_decode(mpeg1_decoder_t *self) {
	if (!self->b->streams[0].has_seq) return false;
	return jsmpeg_b200_batch_decode(self->b, 1, JSMPEG_B200_OUT_HOST | (self->macroblocks ? JSMPEG_B200_OUT_MACROBLOCKS : 0)) > 0;
}

// ================================================================================================
// test hooks

long jsmpeg_b200_debug_read_es(jsmpeg_b200_batch_t *b, int stream, void *dst, size_t cap) {
	return guarded<long>(b, -1, [&]() -> long {
		use_device(b);
		const Stream &s = b->streams[stream];
		const size_t n = std::min<size_t>(cap, s.d_valid);
		if (n) CUDA_CHECK(cudaMemcpy(dst, s.d_es.data(), n, cudaMemcpyDeviceToHost));
		return (long)s.d_valid;
	});
}

int jsmpeg_b200_debug_parse_picture(const uint8_t *es, uint32_t es_len, uint32_t start_byte, int mb_width,
                                    int mb_height, const uint8_t *intra_q, const uint8_t *non_intra_q,
                                    void *info_out, void *hdr_out, void *coef_out) {
	try {
		SeqParams sp{};
		sp.mb_width = mb_width; sp.mb_height = mb_height; sp.mb_size = mb_width * mb_height;
		sp.coded_width = mb_width * 16; sp.coded_height = mb_height * 16;
		memcpy(sp.intra_q, intra_q, 64);
		memcpy(sp.non_intra_q, non_intra_q, 64);
		seq_fill_xq(sp);
		const size_t n_mb = sp.mb_size;
		DeviceBuffer<uint8_t> d_es(es_len + ES_PAD);
		DeviceBuffer<SeqParams> d_seq(1);
		DeviceBuffer<mb_record_t> d_hdr(n_mb);
		DeviceBuffer<int16_t> d_coef(n_mb * MB_COEF_INT16);
		DeviceBuffer<uint2> d_park(n_mb * 6);
		DeviceBuffer<uint4> d_stage((size_t)stage_entries_for(sp.mb_size) * 4);
		DeviceBuffer<picture_info_t> d_info(1);
		DeviceBuffer<ParseTask> d_task(1);
		CUDA_CHECK(cudaMemcpy(d_es.data(), es, es_len, cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemset(d_es.data() + es_len, 0, ES_PAD));
		CUDA_CHECK(cudaMemcpy(d_seq.data(), &sp, sizeof(sp), cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemset(d_coef.data(), 0, n_mb * MB_COEF_INT16 * sizeof(int16_t)));
		ParseTask t{};
		t.es = d_es.data(); t.es_len = es_len; t.start_byte = start_byte; t.seq = d_seq.data(); t.hdr = d_hdr.data();
		t.coef = d_coef.data(); t.info = d_info.data(); t.park = d_park.data(); t.mb_width = mb_width; t.mb_size = sp.mb_size;
		t.stage = d_stage.data(); t.stage_entries = stage_entries_for(sp.mb_size);
		t.codes = nullptr; t.n_codes = 0; t.code_hint = 0;  // this hook lets the walk search the slice end itself
		CUDA_CHECK(cudaMemcpy(d_task.data(), &t, sizeof(t), cudaMemcpyHostToDevice));
		launch_parse_pictures(WALK_LANES, d_task.data(), 1, sp.mb_size, true, 0);
		CUDA_CHECK(cudaGetLastError());
		CUDA_CHECK(cudaDeviceSynchronize());
		CUDA_CHECK(cudaMemcpy(info_out, d_info.data(), sizeof(picture_info_t), cudaMemcpyDeviceToHost));
		CUDA_CHECK(cudaMemcpy(hdr_out, d_hdr.data(), n_mb * sizeof(mb_record_t), cudaMemcpyDeviceToHost));
		CUDA_CHECK(cudaMemcpy(coef_out, d_coef.data(), n_mb * MB_COEF_INT16 * sizeof(int16_t), cudaMemcpyDeviceToHost));
		// stage 1b left most blocks as compact records in the staging area: the caller gets them dense
		std::vector<coef_record_t> compact(n_mb * 6);
		CUDA_CHECK(cudaMemcpy(compact.data(), d_stage.data(), compact.size() * sizeof(coef_record_t), cudaMemcpyDeviceToHost));
		const mb_record_t *hdr = static_cast<const mb_record_t *>(hdr_out);
		for (size_t slot = 0; slot < n_mb * 6; slot++) {
			const mb_record_t &r = hdr[slot / 6];
			if ((r.flags & MBF_PRESENT) && (r.cbp & (0x20 >> (slot % 6))) && compact[slot].mask != COEF_RECORD_DENSE)
				coef_record_unpack(compact[slot], static_cast<int16_t *>(coef_out) + slot * 64);
		}
		return 0;
	} catch (const std::exception &e) {
		fprintf(stderr, "%s\n", e.what());
		return -1;
	}
}

int jsmpeg_b200_debug_reconstruct(int mb_width, int mb_height, const void *hdr, const void *coef,
                                  const uint8_t *fwd_y, const uint8_t *fwd_cr, const uint8_t *fwd_cb,
                                  uint8_t *cur_y, uint8_t *cur_cr, uint8_t *cur_cb) {
	try {
		const size_t n_mb = (size_t)mb_width * mb_height;
		const size_t ysz = n_mb * 256, csz = ysz / 4, total = ysz + 2 * csz;
		DeviceBuffer<mb_record_t> d_hdr(n_mb);
		DeviceBuffer<int16_t> d_coef(n_mb * MB_COEF_INT16);
		// the caller's dense blocks as stage 1b would hand them over: compact records where they fit
		std::vector<coef_record_t> compact(n_mb * 6);
		for (size_t slot = 0; slot < n_mb * 6; slot++) {
			const int16_t *blk = static_cast<const int16_t *>(coef) + slot * 64;
			const uint64_t pos = coef_nonzero_positions(blk);
			if (coef_record_fits(pos)) compact[slot] = coef_record_pack(pos, blk);
			else compact[slot].mask = COEF_RECORD_DENSE;
		}
		DeviceBuffer<coef_record_t> d_compact(n_mb * 6);
		CUDA_CHECK(cudaMemcpy(d_compact.data(), compact.data(), compact.size() * sizeof(coef_record_t), cudaMemcpyHostToDevice));
		const size_t pad = (size_t)mb_width * 16 + 64;
		DeviceBuffer<uint8_t> fwd_buf(total + pad), cur_buf(total + pad);
		uint8_t *d_fwd = fwd_buf.data(), *d_cur = cur_buf.data();
		CUDA_CHECK(cudaMemset(d_fwd + total, 0, pad));
		CUDA_CHECK(cudaMemcpy(d_hdr.data(), hdr, n_mb * sizeof(mb_record_t), cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_coef.data(), coef, n_mb * MB_COEF_INT16 * sizeof(int16_t), cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_fwd, fwd_y, ysz, cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_fwd + ysz, fwd_cr, csz, cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_fwd + ysz + csz, fwd_cb, csz, cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_cur, cur_y, ysz, cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_cur + ysz, cur_cr, csz, cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_cur + ysz + csz, cur_cb, csz, cudaMemcpyHostToDevice));
		ReconTask t{};
		t.hdr = d_hdr.data(); t.coef = d_coef.data(); t.compact = d_compact.data();
		t.cur = PlaneSet{d_cur, d_cur + ysz, d_cur + ysz + csz};
		t.fwd = PlaneSet{d_fwd, d_fwd + ysz, d_fwd + ysz + csz};
		t.mb_width = mb_width; t.mb_size = (int)n_mb;
		t.coded_width = mb_width * 16; t.coded_height = mb_height * 16;
		launch_reconstruct(&t, 1, 0);
		CUDA_CHECK(cudaGetLastError());
		CUDA_CHECK(cudaDeviceSynchronize());
		CUDA_CHECK(cudaMemcpy(cur_y, d_cur, ysz, cudaMemcpyDeviceToHost));
		CUDA_CHECK(cudaMemcpy(cur_cr, d_cur + ysz, csz, cudaMemcpyDeviceToHost));
		CUDA_CHECK(cudaMemcpy(cur_cb, d_cur + ysz + csz, csz, cudaMemcpyDeviceToHost));
		return 0;
	} catch (const std::exception &e) {
		fprintf(stderr, "%s\n", e.what());
		return -1;
	}
}

}  // extern "C"
