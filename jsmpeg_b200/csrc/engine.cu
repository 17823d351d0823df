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
// queues one reconstruct step per picture depth (ReconStep, launch_step) on the reconstruct stream.
// Cutting the wave into chunks to overlap stage 1 with stage 2 was measured not to pay (DESIGN 8).
// decode_macroblocks runs the same waves walk-only (no expand, no reconstruct) and exports the records (DESIGN 3.8).
#include <sched.h>

#include <algorithm>
#include <cstring>
#include <deque>
#include <string>
#include <vector>

#include "bitbuffer.h"
#include "common.cuh"
#include "../../include/jsmpeg_b200.h"

namespace {

constexpr int HOST_RING = 4;
constexpr uint32_t ES_PAD = 512;  // readable, zeroed slack after the ES mirror (the walk's ring prefetches 64 bytes ahead)

template <typename T>
T *dev_alloc(size_t n) {
	T *p = nullptr;
	CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)));
	return p;
}
template <typename T>
T *pinned_alloc(size_t n) {
	T *p = nullptr;
	CUDA_CHECK(cudaHostAlloc(&p, std::max<size_t>(n, 1) * sizeof(T), cudaHostAllocDefault));
	return p;
}

// the bit buffer lives in pinned host memory (H2D copies of new bytes run at PCIe speed)
void *bb_pinned_alloc(size_t n, void *) { return pinned_alloc<uint8_t>(n); }
void bb_pinned_release(void *p, void *) { (void)cudaFreeHost(p); }
const bitbuffer::Allocator kPinned = {bb_pinned_alloc, bb_pinned_release, nullptr};

struct Parsed {
	uint32_t pos;           // byte position of the 00 00 01 00 start code
	uint32_t len_at_parse;  // buffer length the parse saw
	int slot;
	picture_info_t info;
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
	SeqParams *d_seq = nullptr;
	// ES mirror in HBM + start-code index
	uint8_t *d_es = nullptr;
	uint32_t d_capacity = 0, d_valid = 0;
	std::vector<uint32_t> pics;  // sorted byte positions of picture start codes (00 00 01 00)
	std::vector<uint32_t> codes, pic_code;  // every start-code prefix (00 00 01), sorted; pics[k] == codes[pic_code[k]]
	uint32_t codes_classified = 0;          // codes[0 .. codes_classified) have had their fourth byte looked at
	uint32_t scanned = 0;        // every prefix with pos + 2 < scanned is in `codes`
	uint32_t scan_from = 0;      // the span a pending scan covers starts here
	bool scan_pending = false;
	// planes: two sets in HBM (ping-pong like mpeg1.js:221-246), a host ring for OUT_HOST
	uint8_t *d_planes[2] = {nullptr, nullptr};
	int cur = 0;  // set written by the next I/P picture; forward = 1 - cur
	uint8_t *h_planes[HOST_RING] = {};
	int h_head = -1;
	// B-picture extension ("decode_b"): two more sets in HBM, written in turn -- a B picture is no reference, the
	// ping-pong above is untouched by it; d_last = the set holding the most recently decoded picture
	uint8_t *d_planes_b[2] = {nullptr, nullptr};
	int b_cur = 0;
	uint8_t *d_last = nullptr;
	int last_type = 0, last_temporal = 0;  // picture_coding_type / temporal_reference of the last picture decode() consumed
	uint8_t *d_rgba = nullptr;
	std::vector<int16_t> ts_bound;     // device TS demux: the stream id every PID is bound to, 0 = none (ts.js pidsToStreamIds)
	std::vector<uint8_t> ts_leftover;  // ... and the bytes the last write_ts left over (ts.js leftoverBytes)
	std::vector<uint8_t> ps_leftover;  // device PS demux: the bytes the last write_ps left over
	bool ps_in_sync = false;           // ... and whether they continue the item chain (else: look for a pack header)
	// parsed-ahead pictures, consecutive, front = next picture decode() consumes
	std::deque<Parsed> cache;
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
	ScanSpan *d_spans = nullptr, *h_spans = nullptr;
	uint32_t *d_scan_counts = nullptr, *h_scan_counts = nullptr, *d_scan_pos = nullptr, *h_scan_pos = nullptr;
	uint32_t scan_rows = 0, scan_seg = 0;       // room: spans, positions per span
	uint32_t *d_codes = nullptr, *h_codes = nullptr;
	uint32_t codes_rows = 0, codes_stride = 0;  // rows = streams, stride = entries per row
	cudaStream_t st_main = nullptr, st_recon = nullptr, st_copy = nullptr;  // uploads + scan + parse | reconstruct | copy-out
	cudaEvent_t ev_a = nullptr, ev_b = nullptr, ev_mid = nullptr, ev_step = nullptr, ev_round = nullptr, ev_copied[2] = {nullptr, nullptr};
	cudaEvent_t ev_recon[2] = {nullptr, nullptr};  // around a round's reconstruct launches (timing)
	// record slots
	unsigned max_slots_req = 0;
	int slot_mb = 0, n_slots = 0;
	mb_record_t *d_hdr = nullptr;
	int16_t *d_coef = nullptr;
	uint2 *d_park = nullptr;
	uint4 *d_stage = nullptr;  // per slot: stage_entries_for(slot_mb) x 64 B (lane-parallel walk, relative records)
	picture_info_t *d_info = nullptr, *h_info = nullptr;
	std::vector<int> free_slots;
	int lookahead = 1;
	bool decode_b = false;       // the B-picture extension: off = B pictures are skipped like the reference does (mpeg1.js:181-184)
	bool slice_walk = false;     // I/P pictures of >= SLICE_WALK_MIN_SLICES slices go to the one-lane-per-slice walk (walk_slices.cuh)
	// pictures with a walk kernel of their own (B pictures; with "slice_walk", I/P pictures of many slices) are
	// walked beside the others, on these streams
	cudaStream_t st_side[2] = {nullptr, nullptr};
	cudaEvent_t ev_sfork = nullptr, ev_sjoin[2] = {nullptr, nullptr};
	bool recon_pending = false;  // reconstruct launches of an earlier round may still read record slots
	// parse task staging
	ParseTask *h_ptasks = nullptr, *d_ptasks = nullptr;
	int ptask_cap = 0;
	uint64_t copy_steps = 0;  // reconstruct launches with a copy-out so far (event parity)
	ParseFork fork{};
	bool batch_copy_ok = true;
	TsScratch *ts = nullptr;
	PsScratch *ps = nullptr;
	// decode_pictures / decode_intra: the forward plane set a chain of one picture names, zeroed and never written
	// (DESIGN 3.6); and the pool of the other chains' plane sets, zeroed per chain group (DESIGN 3.7)
	uint8_t *d_intra_fwd = nullptr;
	size_t intra_fwd_bytes = 0;
	uint8_t *d_chain_sets = nullptr;
	size_t chain_sets_bytes = 0;
	// decode_macroblocks: the export tasks of a wave (DESIGN 3.8)
	MbExportTask *h_xtasks = nullptr, *d_xtasks = nullptr;
	int xtask_cap = 0;
	jsmpeg_b200_stats_t stats{};
};

namespace {

using Batch = jsmpeg_b200_batch_t;

void use_device(Batch *b) { CUDA_CHECK(cudaSetDevice(b->device)); }

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

// MSB-first reader for the (tiny, once-per-stream) sequence header on the host
struct HostBits {
	const uint8_t *p;
	uint32_t len, idx;
	uint32_t read(int n) {
		uint32_t v = 0;
		for (int i = 0; i < n; i++, idx++) {
			uint32_t byte = idx >> 3;
			v = (v << 1) | (byte < len ? (p[byte] >> (7 - (idx & 7))) & 1u : 0u);
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
	s.bb.index = hb.idx;
	s.seq_end_index = hb.idx;
	s.seq_floor = (hb.idx + 7) >> 3;  // where decode() starts looking for the first picture
	s.seq.mb_width = (s.width + 15) >> 4;
	s.seq.mb_height = (s.height + 15) >> 4;
	s.seq.mb_size = s.seq.mb_width * s.seq.mb_height;
	s.seq.coded_width = s.seq.mb_width << 4;
	s.seq.coded_height = s.seq.mb_height << 4;
	s.coded_size = s.seq.coded_width * s.seq.coded_height;
	s.has_seq = true;

	const size_t plane_bytes = (size_t)s.coded_size * 3 / 2;
	s.d_seq = dev_alloc<SeqParams>(1);
	CUDA_CHECK(cudaMemcpyAsync(s.d_seq, &s.seq, sizeof(SeqParams), cudaMemcpyHostToDevice, b->st_main));
	for (int i = 0; i < 2; i++) {
		// + coded_width + 64: stage 2's row loads may touch (never use) up to one row past a plane set's end
		s.d_planes[i] = dev_alloc<uint8_t>(plane_bytes + s.seq.coded_width + 64);
		CUDA_CHECK(cudaMemsetAsync(s.d_planes[i], 0, plane_bytes + s.seq.coded_width + 64, b->st_main));  // JS typed arrays start zeroed
	}
	for (int i = 0; i < HOST_RING; i++) {
		s.h_planes[i] = pinned_alloc<uint8_t>(plane_bytes);
		memset(s.h_planes[i], 0, plane_bytes);
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
	if ((uint64_t)need + ES_PAD <= s.d_capacity) return;
	uint64_t cap = std::max<uint64_t>((uint64_t)need + ES_PAD, (uint64_t)s.d_capacity * 2);
	cap = std::min<uint64_t>((cap + 255u) & ~255ull, 0xffffff00ull);
	uint8_t *n = dev_alloc<uint8_t>(cap);
	if (s.d_es) {
		if (s.d_valid) CUDA_CHECK(cudaMemcpyAsync(n, s.d_es, s.d_valid, cudaMemcpyDeviceToDevice, b->st_main));
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));
		CUDA_CHECK(cudaFree(s.d_es));
	}
	s.d_es = n;
	s.d_capacity = (uint32_t)cap;
}

// Room for `rows` spans with `seg` positions each (contents are per scan: nothing to keep).
void reserve_scan(Batch *b, uint32_t rows, uint32_t seg) {
	if (rows <= b->scan_rows && seg <= b->scan_seg) return;
	rows = std::max(rows, b->scan_rows);
	seg = std::max(seg, b->scan_seg);
	if (b->d_spans) CUDA_CHECK(cudaFree(b->d_spans));
	if (b->d_scan_counts) CUDA_CHECK(cudaFree(b->d_scan_counts));
	if (b->d_scan_pos) CUDA_CHECK(cudaFree(b->d_scan_pos));
	if (b->h_spans) CUDA_CHECK(cudaFreeHost(b->h_spans));
	if (b->h_scan_counts) CUDA_CHECK(cudaFreeHost(b->h_scan_counts));
	if (b->h_scan_pos) CUDA_CHECK(cudaFreeHost(b->h_scan_pos));
	b->d_spans = nullptr; b->d_scan_counts = nullptr; b->d_scan_pos = nullptr;
	b->h_spans = nullptr; b->h_scan_counts = nullptr; b->h_scan_pos = nullptr;
	b->scan_rows = b->scan_seg = 0;
	b->d_spans = dev_alloc<ScanSpan>(rows);
	b->h_spans = pinned_alloc<ScanSpan>(rows);
	b->d_scan_counts = dev_alloc<uint32_t>(rows);
	b->h_scan_counts = pinned_alloc<uint32_t>(rows);
	b->d_scan_pos = dev_alloc<uint32_t>((size_t)rows * seg);
	b->h_scan_pos = pinned_alloc<uint32_t>((size_t)rows * seg);
	b->scan_rows = rows;
	b->scan_seg = seg;
}

// One launch over the pending spans (h_spans[0 .. n)); the counts come back to h_scan_counts.
void launch_scan(Batch *b, int n, uint32_t longest) {
	CUDA_CHECK(cudaMemcpyAsync(b->d_spans, b->h_spans, n * sizeof(ScanSpan), cudaMemcpyHostToDevice, b->st_main));
	CUDA_CHECK(cudaMemsetAsync(b->d_scan_counts, 0, n * sizeof(uint32_t), b->st_main));
	launch_scan_start_codes(b->d_spans, n, longest, b->d_scan_pos, b->scan_seg, b->d_scan_counts, b->st_main);
	b->stats.kernel_launches++;
	CUDA_CHECK(cudaMemcpyAsync(b->h_scan_counts, b->d_scan_counts, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, b->st_main));
}

// The device's copy of every stream's prefix list: row si = streams[si].codes.  The host has them all, so a
// change of geometry (more streams, a longer list) just stages everything again.  Returns true if rebuilt.
bool reserve_codes(Batch *b, uint32_t rows, uint32_t entries) {
	if (rows == b->codes_rows && entries <= b->codes_stride) return false;
	const uint32_t stride = std::max<uint32_t>(std::max<uint32_t>(2 * b->codes_stride, entries + 256u), 1024u);
	if (b->d_codes) {
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));  // (tasks of an earlier round may still name the old rows)
		CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
		CUDA_CHECK(cudaFree(b->d_codes));
	}
	if (b->h_codes) CUDA_CHECK(cudaFreeHost(b->h_codes));
	b->d_codes = nullptr; b->h_codes = nullptr;
	b->codes_rows = b->codes_stride = 0;
	b->d_codes = dev_alloc<uint32_t>((size_t)rows * stride);
	b->h_codes = pinned_alloc<uint32_t>((size_t)rows * stride);
	b->codes_rows = rows;
	b->codes_stride = stride;
	return true;
}

void begin_upload(Batch *b, Stream &s) {
	s.scan_pending = false;
	if (s.d_valid >= s.bb.length && s.scanned >= s.bb.length) return;
	reserve_device_es(b, s, s.bb.length);
	if (s.d_valid < s.bb.length) {
		uint32_t from = s.d_valid & ~15u;
		CUDA_CHECK(cudaMemcpyAsync(s.d_es + from, s.bb.bytes + from, s.bb.length - from, cudaMemcpyHostToDevice, b->st_main));
		b->stats.h2d_bytes += s.bb.length - from;
		s.d_valid = s.bb.length;
		// the kernels rely on zeros right after the data (bytes past the end read as 0, like JS)
		CUDA_CHECK(cudaMemsetAsync(s.d_es + s.bb.length, 0, ES_PAD, b->st_main));
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
			b->h_spans[k] = ScanSpan{s.d_es, s.scan_from, s.bb.length};
		}
		launch_scan(b, n, longest);
		CUDA_CHECK(cudaEventRecord(b->ev_b, b->st_main));
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));
		float ms = 0;
		CUDA_CHECK(cudaEventElapsedTime(&ms, b->ev_a, b->ev_b));
		b->stats.scan_ms += ms;
		uint32_t most = *std::max_element(b->h_scan_counts, b->h_scan_counts + n);
		if (most > b->scan_seg) {
			// a list overflowed (hostile input: start codes cannot overlap, so at most length / 3 of them): once
			// more, with room for the count the kernel reported
			reserve_scan(b, (uint32_t)n, most + 16u);
			for (int k = 0; k < n; k++) {  // (the pinned span list was reallocated)
				const Stream &s = b->streams[pending[k]];
				b->h_spans[k] = ScanSpan{s.d_es, s.scan_from, s.bb.length};
			}
			launch_scan(b, n, longest);
			CUDA_CHECK(cudaStreamSynchronize(b->st_main));
			most = *std::max_element(b->h_scan_counts, b->h_scan_counts + n);
			if (most > b->scan_seg) throw std::runtime_error("jsmpeg_b200: start-code index overflow after a rescan");
		}
		if (most) {  // the positions of all spans in one (strided) copy
			CUDA_CHECK(cudaMemcpy2DAsync(b->h_scan_pos, (size_t)b->scan_seg * sizeof(uint32_t), b->d_scan_pos,
			                             (size_t)b->scan_seg * sizeof(uint32_t), (size_t)most * sizeof(uint32_t), (size_t)n,
			                             cudaMemcpyDeviceToHost, b->st_main));
			b->stats.d2h_bytes += (uint64_t)most * n * sizeof(uint32_t);
			CUDA_CHECK(cudaStreamSynchronize(b->st_main));
		}
		bool grew = false;
		for (int k = 0; k < n; k++) {
			Stream &s = b->streams[pending[k]];
			uint32_t *hits = b->h_scan_pos + (size_t)k * b->scan_seg;
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
			const bool rebuilt = reserve_codes(b, (uint32_t)S, (uint32_t)longest_list);
			for (int si = 0; si < S; si++) {
				const Stream &s = b->streams[si];
				// (a rewound stream's list starts over: staging whole rows keeps this free of bookkeeping; they are short)
				if (!s.codes.empty() && (rebuilt || std::find(pending.begin(), pending.end(), si) != pending.end()))
					memcpy(b->h_codes + (size_t)si * b->codes_stride, s.codes.data(), s.codes.size() * sizeof(uint32_t));
			}
			CUDA_CHECK(cudaMemcpy2DAsync(b->d_codes, (size_t)b->codes_stride * sizeof(uint32_t), b->h_codes,
			                             (size_t)b->codes_stride * sizeof(uint32_t), longest_list * sizeof(uint32_t), (size_t)S,
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
	if (b->d_hdr) { CUDA_CHECK(cudaFree(b->d_hdr)); b->d_hdr = nullptr; }
	if (b->d_coef) { CUDA_CHECK(cudaFree(b->d_coef)); b->d_coef = nullptr; }
	if (b->d_park) { CUDA_CHECK(cudaFree(b->d_park)); b->d_park = nullptr; }
	if (b->d_stage) { CUDA_CHECK(cudaFree(b->d_stage)); b->d_stage = nullptr; }
	if (b->d_info) { CUDA_CHECK(cudaFree(b->d_info)); b->d_info = nullptr; }
	if (b->h_info) { CUDA_CHECK(cudaFreeHost(b->h_info)); b->h_info = nullptr; }
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
	b->d_hdr = dev_alloc<mb_record_t>(n * need_mb);
	b->d_coef = dev_alloc<int16_t>(n * need_mb * MB_COEF_INT16);
	b->d_park = dev_alloc<uint2>(n * need_mb * 6);
	b->d_stage = dev_alloc<uint4>(n * (size_t)stage_entries_for(need_mb) * 4);
	b->d_info = dev_alloc<picture_info_t>(n);
	b->h_info = pinned_alloc<picture_info_t>(n);
	b->slot_mb = need_mb;
	b->n_slots = (int)n;
	for (int i = (int)n - 1; i >= 0; i--) b->free_slots.push_back(i);
}

void ensure_task_caps(Batch *b, int n_parse) {
	if (n_parse <= b->ptask_cap) return;
	if (b->h_ptasks) { CUDA_CHECK(cudaFreeHost(b->h_ptasks)); b->h_ptasks = nullptr; }
	if (b->d_ptasks) { CUDA_CHECK(cudaFree(b->d_ptasks)); b->d_ptasks = nullptr; }
	const int cap = std::max(n_parse, b->ptask_cap * 2);
	b->ptask_cap = 0;
	b->h_ptasks = pinned_alloc<ParseTask>(cap);
	b->d_ptasks = dev_alloc<ParseTask>(cap);
	b->ptask_cap = cap;
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
// where the driver has no batched copy
void copy_batch(Batch *b, std::vector<void *> &dst, std::vector<void *> &src, std::vector<size_t> &size, cudaStream_t st) {
	const size_t n_copy = dst.size();
	bool batched = false;
	if (b->batch_copy_ok && n_copy > 1) {
		cudaMemcpyAttributes attr{};
		attr.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
		size_t attr_idx = 0, fail_idx = 0;
		cudaError_t e = cudaMemcpyBatchAsync(dst.data(), src.data(), size.data(), n_copy, &attr, &attr_idx, 1, &fail_idx, st);
		if (e == cudaSuccess) batched = true;
		else { (void)cudaGetLastError(); b->batch_copy_ok = false; }  // older driver: plain copies from now on
	}
	if (!batched)
		for (size_t i = 0; i < n_copy; i++) CUDA_CHECK(cudaMemcpyAsync(dst[i], src[i], size[i], cudaMemcpyDefault, st));
}

// The reconstruct launches of one step of decode() (or one depth of decode_chains), by kernel: I/P and B pictures,
// each without and with the fused RGBA conversion; and the copies of its pictures that follow them
struct ReconStep {
	std::vector<ReconTask> ip, ip_rgba, bi, bi_rgba;
	std::vector<void *> dst, src;
	std::vector<size_t> size;
	void add(const ReconTask &t) { (t.bwd.y ? (t.rgba ? bi_rgba : bi) : (t.rgba ? ip_rgba : ip)).push_back(t); }
	void copy(void *to, void *from, size_t n) {
		dst.push_back(to);
		src.push_back(from);
		size.push_back(n);
	}
};

// Queues a step's reconstruct launches on `st`; returns the number of kernels launched
int launch_step(const ReconStep &r, cudaStream_t st) {
	int n = launch_reconstruct(r.ip.data(), (int)r.ip.size(), st);
	n += launch_reconstruct_rgba(r.ip_rgba.data(), (int)r.ip_rgba.size(), st);
	n += launch_reconstruct_b(r.bi.data(), (int)r.bi.size(), false, st);
	n += launch_reconstruct_b(r.bi_rgba.data(), (int)r.bi_rgba.size(), true, st);
	return n;
}

// The copy-out of one step's pictures (OUT_HOST) on the copy stream, behind the step's launches
void copy_out_step(Batch *b, ReconStep &r) {
	CUDA_CHECK(cudaEventRecord(b->ev_step, b->st_recon));
	CUDA_CHECK(cudaStreamWaitEvent(b->st_copy, b->ev_step, 0));
	copy_batch(b, r.dst, r.src, r.size, b->st_copy);  // all pictures of the step leave in one batched copy call
	CUDA_CHECK(cudaEventRecord(b->ev_copied[b->copy_steps & 1], b->st_copy));
	b->copy_steps++;
}

// picture_coding_type of picture `pic` of a stream (ISO 11172-2 2.4.2.5: 10 bits temporal_reference, 3 bits
// picture_coding_type); 0 while its header byte is not in the buffer yet
int picture_type_of(const Stream &s, uint32_t pic) {
	const uint32_t pos = s.pics[pic];
	return (uint64_t)pos + 5 < s.bb.length ? (s.bb.bytes[pos + 5] >> 3) & 7 : 0;
}

// Which walk kernel takes picture `pic` of a stream: 0 the lane-parallel walk, 1 the slice walk, 2 the B-picture walk.
// b_walk: a type 3 picture goes to the B-picture walk (decode() and decode_pictures: the decode_b option); everything
// else, and everything without it, to the I/P walk
int walk_kind(const Batch *b, const Stream &s, uint32_t pic, bool b_walk) {
	const int type = picture_type_of(s, pic);
	int kind = (b_walk && type == 3) ? 2 : 0;
	if (b->slice_walk && (type == 1 || type == 2)) {  // enough slice start codes between this picture's and the next one's?
		const uint32_t hi = pic + 1 < s.pic_code.size() ? s.pic_code[pic + 1] : (uint32_t)s.codes.size();
		int n_slices = 0;
		for (uint32_t k = s.pic_code[pic] + 1; k < hi && n_slices < SLICE_WALK_MIN_SLICES; k++) {
			const uint32_t q = s.codes[k];
			if (q + 3u < s.bb.length && s.bb.bytes[q + 3u] >= 0x01 && s.bb.bytes[q + 3u] <= 0xAF) n_slices++;
		}
		if (n_slices >= SLICE_WALK_MIN_SLICES) kind = 1;
	}
	return kind;
}

// The stage-1 task of picture `pic` of stream `si`: records into `slot`, its info into d_info[info_idx]
ParseTask parse_task(const Batch *b, int si, uint32_t pic, int slot, int info_idx) {
	const Stream &s = b->streams[si];
	ParseTask t{};
	t.es = s.d_es;
	t.es_len = s.bb.length;
	t.start_byte = s.pics[pic] + 4;
	t.seq = s.d_seq;
	t.hdr = b->d_hdr + (size_t)slot * b->slot_mb;
	t.coef = b->d_coef + (size_t)slot * b->slot_mb * MB_COEF_INT16;
	t.park = b->d_park + (size_t)slot * b->slot_mb * 6;
	t.info = b->d_info + info_idx;
	t.mb_width = s.seq.mb_width;
	t.mb_size = s.seq.mb_size;
	t.stage = b->d_stage + (size_t)slot * stage_entries_for(b->slot_mb) * 4;
	t.stage_entries = stage_entries_for(b->slot_mb);
	t.codes = b->d_codes ? b->d_codes + (size_t)si * b->codes_stride : nullptr;
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
	int kind;
	uint32_t bytes;
};

// Stage 1 of `wave` as one wave, for decode(), decode_chains and decode_macroblocks alike; expand = false runs the walks
// alone (records without coefficients: decode_macroblocks).  The tasks are grouped by walk kernel and,
// within a kernel, longest first: a CTA's warps, and consecutive CTAs (which land on different SMs), then carry
// similar amounts of work and the walk ends without a long tail.  The first kernel present runs on the main stream;
// the others have walk kernels of their own (one warp per picture, latency-bound like every walk) and run beside it on
// side streams, forked after the upload and joined before the infos are read.  On return the infos are on the host,
// b->h_info[i] that of wave[i], and ev_a / ev_mid / ev_b bracket the wave and its lane-parallel walk.  Returns the
// number of kernels launched.
int parse_wave(Batch *b, const std::vector<WaveItem> &wave, bool expand) {
	const int n = (int)wave.size();
	std::vector<int> order(n);
	for (int i = 0; i < n; i++) order[i] = i;
	std::stable_sort(order.begin(), order.end(), [&](int x, int y) {
		return wave[x].kind != wave[y].kind ? wave[x].kind < wave[y].kind : wave[x].bytes > wave[y].bytes;
	});
	ensure_task_caps(b, n);
	int cnt[3] = {0, 0, 0};
	for (int j = 0; j < n; j++) {
		const WaveItem &w = wave[order[j]];
		b->h_ptasks[j] = parse_task(b, w.stream, w.pic, w.slot, order[j]);
		cnt[w.kind]++;
	}
	if (b->recon_pending) {  // slots freed by an earlier round or wave may still be read by its reconstruct launches
		CUDA_CHECK(cudaStreamWaitEvent(b->st_main, b->ev_round, 0));
		b->recon_pending = false;
	}
	CUDA_CHECK(cudaMemcpyAsync(b->d_ptasks, b->h_ptasks, n * sizeof(ParseTask), cudaMemcpyHostToDevice, b->st_main));
	CUDA_CHECK(cudaEventRecord(b->ev_a, b->st_main));
	int primary = 0;
	while (cnt[primary] == 0) primary++;
	if (cnt[primary] < n) CUDA_CHECK(cudaEventRecord(b->ev_sfork, b->st_main));
	// the wave's pictures by walk kernel: [0, cnt[0]) lane-parallel walk, then the slice walk's, then the B pictures
	const int off[3] = {0, cnt[0], cnt[0] + cnt[1]};
	int launches = 0, n_side = 0;
	for (int kind = 0; kind < 3; kind++) {
		if (cnt[kind] == 0) continue;
		cudaStream_t st = b->st_main;
		if (kind != primary) {
			st = b->st_side[n_side];
			CUDA_CHECK(cudaStreamWaitEvent(st, b->ev_sfork, 0));
		}
		if (kind == 0) launches += launch_parse_pictures(b->d_ptasks, cnt[0], b->slot_mb, expand, st, b->ev_mid, &b->fork);
		else if (kind == 1) launches += launch_parse_pictures_slices(b->d_ptasks + off[1], cnt[1], b->slot_mb, expand, st);
		else launches += launch_parse_pictures_b(b->d_ptasks + off[2], cnt[2], b->slot_mb, expand, st);
		if (kind != primary) {
			CUDA_CHECK(cudaEventRecord(b->ev_sjoin[n_side], st));
			CUDA_CHECK(cudaStreamWaitEvent(b->st_main, b->ev_sjoin[n_side], 0));
			n_side++;
		}
	}
	CUDA_CHECK(cudaMemcpyAsync(b->h_info, b->d_info, n * sizeof(picture_info_t), cudaMemcpyDeviceToHost, b->st_main));
	if (cnt[0] == 0) CUDA_CHECK(cudaEventRecord(b->ev_mid, b->st_main));  // (a wave without the lane-parallel walk)
	CUDA_CHECK(cudaEventRecord(b->ev_b, b->st_main));
	CUDA_CHECK(cudaEventSynchronize(b->ev_b));
	return launches;
}

// The reconstruct task of a picture of `s` whose records are in `slot`: written into the plane set at `cur`, predicted
// from `fwd` (and, for a B picture, `bwd`), with the fused RGBA conversion into `rgba` unless that is nullptr
ReconTask recon_task(const Batch *b, const Stream &s, int slot, uint8_t *cur, uint8_t *fwd, uint8_t *bwd, uint8_t *rgba) {
	ReconTask t{};
	t.hdr = b->d_hdr + (size_t)slot * b->slot_mb;
	t.coef = b->d_coef + (size_t)slot * b->slot_mb * MB_COEF_INT16;
	t.compact = compact_plane(b->d_stage + (size_t)slot * stage_entries_for(b->slot_mb) * 4);  // (stage 1b wrote it: parse_task)
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

// One round: parse ahead what is missing in one wave, then consume up to want[s] pictures per stream in decode()
// order and queue their reconstruction.  Returns pictures consumed; `progress[s]` gets the per-stream count, `more[s]`
// whether the stream may have further pictures.
long decode_round(Batch *b, const std::vector<int> &want, std::vector<int> &progress, std::vector<char> &more, int flags) {
	const int S = (int)b->streams.size();
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
			Parsed p{};
			p.pos = *next;
			p.len_at_parse = s.bb.length;
			p.slot = b->free_slots.back();
			b->free_slots.pop_back();
			s.cache.push_back(p);
			++next;
			const uint32_t pic = (uint32_t)(next - 1 - s.pics.begin());
			wave.push_back({si, pic, p.slot, walk_kind(b, s, pic, b->decode_b), (next < s.pics.end() ? *next : s.bb.length) - p.pos});
		}
	}
	// ---- 2. stage 1: the wave, every picture's info on the host before consumption starts
	if (!wave.empty()) {
		b->stats.kernel_launches += parse_wave(b, wave, true);
		for (size_t i = 0; i < wave.size(); i++) {  // a stream's pictures are in the wave in cache order
			const int si = wave[i].stream;
			Parsed &p = b->streams[si].cache[fresh[si]++];
			p.info = b->h_info[i];
			if (p.info.error == PARSE_ERR_INVALID_VLC) b->stats.parse_errors++;
			if (p.info.reserved[0]) b->stats.lane_walk_pictures++;
		}
		b->stats.h2d_bytes += wave.size() * sizeof(ParseTask);
		b->stats.d2h_bytes += wave.size() * sizeof(picture_info_t);
		float ms = 0;
		CUDA_CHECK(cudaEventElapsedTime(&ms, b->ev_a, b->ev_b));
		b->stats.parse_ms += ms;
		CUDA_CHECK(cudaEventElapsedTime(&ms, b->ev_a, b->ev_mid));
		b->stats.walk_ms += ms;
	}
	// ---- 3. consume in decode() order; the j-th reconstructed picture of a stream goes to step j
	long consumed = 0;
	std::vector<ReconStep> steps;
	for (int si = 0; si < S; si++) {
		if (!more[si]) continue;
		Stream &s = b->streams[si];
		size_t step = 0;
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
			s.last_temporal = (uint64_t)e.pos + 5 < s.bb.length ? (s.bb.bytes[e.pos + 4] << 2 | s.bb.bytes[e.pos + 5] >> 6) : 0;
			if (e.info.status == PIC_DECODED) {
				const bool is_b = e.info.picture_type == 3;  // (only the extension's walk answers PIC_DECODED for one)
				uint8_t *rgba = nullptr;
				if (flags & JSMPEG_B200_OUT_RGBA) {
					if (!s.d_rgba) {  // opaque white, like the canvas the reference creates (canvas2d.js:24-29): the odd edge keeps it
						s.d_rgba = dev_alloc<uint8_t>((size_t)s.width * s.height * 4);
						CUDA_CHECK(cudaMemsetAsync(s.d_rgba, 0xff, (size_t)s.width * s.height * 4, b->st_recon));
					}
					rgba = s.d_rgba;
				}
				ReconTask t;
				if (is_b) {
					// after the swaps `cur` holds the older and `1 - cur` the newer of the two most recent I/P pictures:
					// the B picture's forward (past) and backward (future) reference.  It goes to a set of its own.
					if (!s.d_planes_b[0]) {
						const size_t bytes = (size_t)s.coded_size * 3 / 2 + s.seq.coded_width + 64;
						for (auto &pb : s.d_planes_b) {
							pb = dev_alloc<uint8_t>(bytes);
							CUDA_CHECK(cudaMemsetAsync(pb, 0, bytes, b->st_recon));
						}
					}
					t = recon_task(b, s, e.slot, s.d_planes_b[s.b_cur], s.d_planes[s.cur], s.d_planes[1 - s.cur], rgba);
					s.b_cur ^= 1;  // no reference: the I/P ping-pong stays as it is
				} else {
					t = recon_task(b, s, e.slot, s.d_planes[s.cur], s.d_planes[1 - s.cur], nullptr, rgba);
					s.cur ^= 1;  // mpeg1.js:221-246: the picture just decoded becomes `forward`
				}
				s.d_last = t.cur.y;
				const uint64_t planes = (uint64_t)s.coded_size * 3 / 2;
				if (steps.size() <= step) steps.emplace_back();
				steps[step].add(t);
				if (flags & JSMPEG_B200_OUT_HOST) {  // into the next slot of the stream's host ring
					s.h_head = (s.h_head + 1) % HOST_RING;
					steps[step].copy(s.h_planes[s.h_head], t.cur.y, planes);
					b->stats.d2h_bytes += planes;
				}
				step++;
				b->stats.pictures_decoded++;
				b->stats.coded_blocks += e.info.n_coded_blocks;
				b->stats.macroblocks += e.info.n_present;
				b->stats.algorithmic_bytes += planes + (e.info.picture_type == 2 ? planes : (is_b ? 2 * planes : 0)) +
				                              (uint64_t)s.seq.mb_size * sizeof(mb_record_t) + (uint64_t)e.info.n_coded_blocks * sizeof(coef_record_t);
			}
			release_slot(b, e.slot);  // reused by the NEXT round's parse, which waits for this round's reconstruction (ev_round)
		}
	}
	// ---- 4. reconstruction, one step after the other on the reconstruct stream
	if (!steps.empty()) {
		CUDA_CHECK(cudaEventRecord(b->ev_recon[0], b->st_recon));
		for (ReconStep &r : steps) {
			// A launch overwrites, per stream, the plane set written two of that stream's pictures ago, i.e. by
			// a launch at least two copy-out launches back: the copy-out recorded two launches ago must be done
			// (the copy stream is in order, so that covers every earlier one).
			if ((flags & JSMPEG_B200_OUT_HOST) && b->copy_steps >= 2)
				CUDA_CHECK(cudaStreamWaitEvent(b->st_recon, b->ev_copied[b->copy_steps & 1], 0));
			b->stats.kernel_launches += launch_step(r, b->st_recon);
			b->stats.recon_launches++;
			if (flags & JSMPEG_B200_OUT_HOST) copy_out_step(b, r);  // while the next step reconstructs
		}
		CUDA_CHECK(cudaEventRecord(b->ev_recon[1], b->st_recon));
		CUDA_CHECK(cudaEventRecord(b->ev_round, b->st_recon));
		b->recon_pending = true;
		CUDA_CHECK(cudaEventSynchronize(b->ev_recon[1]));
		float ms = 0;
		CUDA_CHECK(cudaEventElapsedTime(&ms, b->ev_recon[0], b->ev_recon[1]));
		b->stats.recon_ms += ms;
	}
	return consumed;
}

long batch_decode(Batch *b, int n_pictures, int flags) {
	use_device(b);
	upload_all(b);
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
		const long got = decode_round(b, want, progress, more, flags);
		total += got;
		bool replanned = false;
		for (int i = 0; i < S; i++) {
			remaining[i] -= progress[i];
			if (want[i] > 0 && progress[i] < want[i] && more[i]) replanned = true;
		}
		if (got == 0 && (!replanned || ++idle_rounds > 2)) break;
		if (got) idle_rounds = 0;
	}
	CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
	CUDA_CHECK(cudaStreamSynchronize(b->st_copy));
	CUDA_CHECK(cudaStreamSynchronize(b->st_main));
	b->recon_pending = false;
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

// An entry of an index: picture `pic` (an index into s.pics) and its chain start
struct IndexEntry {
	uint32_t pic, chain_start;
};

// The pictures decode_intra can decode now: after the first sequence header, picture_coding_type 1, and closed.  Each
// is its own chain start.
std::vector<IndexEntry> intra_index(const Stream &s) {
	std::vector<IndexEntry> out;
	if (!s.has_seq) return out;
	for (uint32_t k = 0; k < s.pics.size(); k++)
		if (s.pics[k] >= s.seq_floor && picture_type_of(s, k) == 1 && picture_closed(s, k)) out.push_back({k, k});
	return out;
}

// `n` bits of picture `pic`'s header, from bit `bit` after its start code (ISO 11172-2 2.4.2.5: temporal_reference 10,
// picture_coding_type 3, vbv_delay 16, full_pel_forward_vector 1, forward_f_code 3, full_pel_backward_vector 1,
// backward_f_code 3).  Bytes beyond the buffer read as 0, as they do to the walks.
uint32_t picture_header_bits(const Stream &s, uint32_t pic, int bit, int n) {
	uint32_t v = 0;
	for (int i = 0; i < n; i++, bit++) {
		const uint64_t byte = (uint64_t)s.pics[pic] + 4 + (bit >> 3);
		v = v << 1 | (byte < s.bb.length ? (s.bb.bytes[byte] >> (7 - (bit & 7))) & 1u : 0u);
	}
	return v;
}

// Whether the walks decode picture k (PIC_DECODED), by their rule (walk.cuh, walk_b.cuh): an I picture, a P picture with
// forward_f_code != 0, and when B pictures go to the B walk (decode_b) a B picture with both f_codes != 0
bool picture_decoded(const Stream &s, uint32_t k, bool decode_b) {
	const int type = picture_type_of(s, k);
	if (type == 1) return true;
	if (type == 2) return picture_header_bits(s, k, 30, 3) != 0;
	return type == 3 && decode_b && picture_header_bits(s, k, 30, 3) != 0 && picture_header_bits(s, k, 34, 3) != 0;
}

// The pictures decode_pictures can decode now: after the first sequence header, closed, reconstructed by decode(),
// and with a chain start -- the greatest picture j <= k of the intra index such that at least r(k) pictures of
// [j, k) are references (I, or P with forward_f_code != 0); r = 0 for I, 1 for P, 2 for B.
std::vector<IndexEntry> picture_index(const Batch *b, const Stream &s) {
	std::vector<IndexEntry> out;
	if (!s.has_seq) return out;
	std::vector<uint32_t> keys;      // the I pictures after the sequence header so far
	std::vector<uint32_t> refs_upto;  // refs_upto[k]: references among pictures [0, k)
	uint32_t refs = 0;
	for (uint32_t k = 0; k < s.pics.size(); k++) {
		refs_upto.push_back(refs);
		const int type = picture_type_of(s, k);
		const bool after = s.pics[k] >= s.seq_floor;
		if (after && type == 1) keys.push_back(k);
		refs += type == 1 || (type == 2 && picture_header_bits(s, k, 30, 3) != 0);
		if (!after || !picture_decoded(s, k, b->decode_b) || !picture_closed(s, k)) continue;
		const uint32_t need = type == 1 ? 0 : type - 1;
		// (every key is a reference: this looks at most three keys back)
		for (auto j = keys.rbegin(); j != keys.rend(); ++j)
			if (refs_upto[k] - refs_upto[*j] >= need) {
				out.push_back({k, *j});
				break;
			}
	}
	return out;
}

// One request: picture `pic` of stream `stream`, decoded by a fresh decoder from picture `from` (its chain start) on
struct PictureRequest {
	int stream;
	uint32_t pic, from;
};

// The schedule behind decode_pictures and decode_intra (DESIGN 3.7).  Requests with the same stream and chain start
// form a chain: pictures [first, last], parsed in waves over consecutive positions of every chain, consumed on the
// host by decode()'s rule and reconstructed in launches by depth (launch d: the d-th reconstructed picture of every
// chain of the wave).  A requested picture is copied to its destination right behind its launch -- or, in a chain
// that reconstructs nothing else, reconstructed straight into it.  The requests are valid (the caller checked them).
void decode_chains(Batch *b, const std::vector<PictureRequest> &req, void *const *planes_dst, void *const *rgba_dst,
                   bool rgba, int32_t *status_out, int32_t *n_present_out, int32_t *error_out) {
	const int n = (int)req.size();
	ensure_pool(b);
	std::vector<int> order(n);  // the requests by stream, chain start and picture
	for (int i = 0; i < n; i++) order[i] = i;
	std::sort(order.begin(), order.end(), [&](int x, int y) {
		const PictureRequest &p = req[x], &q = req[y];
		return p.stream != q.stream ? p.stream < q.stream : p.from != q.from ? p.from < q.from : p.pic != q.pic ? p.pic < q.pic : x < y;
	});
	struct Chain {
		int stream;
		uint32_t first, last;  // chain start, last requested picture
		uint32_t b_end;        // last requested B picture + 1; 0: none (B pictures after it are not reconstructed)
		int req_lo, req_hi;    // its requests: order[req_lo .. req_hi)
		int req_next;          // the first of them not consumed yet
		int n_sets;            // plane sets: 0 (a leaf: it reconstructs the one picture requested), 2 (I/P), 4 (+ B)
		uint8_t *set[4];
		int cur, b_cur;        // as Stream::cur / b_cur
		uint32_t next;         // the picture decode() consumes next; beyond `last`: the chain is done
		std::vector<picture_info_t> info;  // per picture of the chain, once parsed
		std::vector<int> slot;
	};
	std::vector<Chain> chains;
	size_t set_bytes = 0, n_tasks = 0;
	bool leaves = false;
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
			if (picture_type_of(s, req[order[i]].pic) == 3) c.b_end = req[order[i]].pic + 1;
		c.req_lo = c.req_next = lo;
		c.req_hi = hi;
		c.n_sets = c.last == c.first ? 0 : (c.b_end ? 4 : 2);
		c.info.resize(c.last - c.first + 1);
		c.slot.resize(c.last - c.first + 1);
		leaves |= c.n_sets == 0;
		// + coded_width + 64: parse_sequence_header's slack; a multiple of 256 keeps every set of the pool aligned
		set_bytes = std::max(set_bytes, ((size_t)s.coded_size * 3 / 2 + s.seq.coded_width + 64 + 255) & ~(size_t)255);
		n_tasks += c.info.size();
		chains.push_back(std::move(c));
		lo = hi;
	}
	if (leaves && set_bytes > b->intra_fwd_bytes) {
		if (b->d_intra_fwd) {
			CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
			CUDA_CHECK(cudaFree(b->d_intra_fwd));
			b->d_intra_fwd = nullptr;
			b->intra_fwd_bytes = 0;
		}
		b->d_intra_fwd = dev_alloc<uint8_t>(set_bytes);
		CUDA_CHECK(cudaMemsetAsync(b->d_intra_fwd, 0, set_bytes, b->st_recon));
		b->intra_fwd_bytes = set_bytes;
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
	std::vector<int32_t> status(n, 0), n_present(n, 0), error(n, 0);
	// record slots: the free ones; when they do not cover the call, the look-ahead's too (decode() parses those again)
	if (b->free_slots.size() < n_tasks)
		for (auto &s : b->streams) flush_cache(b, s);
	const int wave_max = (int)b->free_slots.size();
	// chain groups: at most wave_max chains (a wave parses at least one picture of each), and plane sets within half
	// of the free device memory -- a request beyond the device is cut into groups, not refused
	size_t free_b = 0, total_b = 0;
	CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
	const size_t max_sets = std::max<size_t>(4, ((size_t)(0.5 * (double)free_b) + b->chain_sets_bytes) / set_bytes);
	std::vector<std::pair<size_t, size_t>> groups;
	size_t most_sets = 0;
	for (size_t lo = 0; lo < chains.size();) {
		size_t hi = lo, sets = 0;
		while (hi < chains.size() && hi - lo < (size_t)wave_max && sets + chains[hi].n_sets <= max_sets) sets += chains[hi++].n_sets;
		groups.push_back({lo, hi});
		most_sets = std::max(most_sets, sets);
		lo = hi;
	}
	if (most_sets * set_bytes > b->chain_sets_bytes) {
		if (b->d_chain_sets) {
			CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
			CUDA_CHECK(cudaFree(b->d_chain_sets));
			b->d_chain_sets = nullptr;
			b->chain_sets_bytes = 0;
		}
		b->d_chain_sets = dev_alloc<uint8_t>(most_sets * set_bytes);
		b->chain_sets_bytes = most_sets * set_bytes;
	}
	for (const auto &[glo, ghi] : groups) {
		size_t sets = 0;
		for (size_t c = glo; c < ghi; c++)
			for (int k = 0; k < chains[c].n_sets; k++) chains[c].set[k] = b->d_chain_sets + set_bytes * sets++;
		if (sets)  // a fresh decoder's planes start zeroed, the B sets too (the previous group's copies are queued before)
			CUDA_CHECK(cudaMemsetAsync(b->d_chain_sets, 0, set_bytes * sets, b->st_recon));
		const uint32_t width = (uint32_t)std::max<size_t>(1, (size_t)wave_max / (ghi - glo));
		for (uint32_t lo = 0;; lo += width) {
			// ---- stage 1: positions [lo, lo + width) of every chain still consuming
			std::vector<WaveItem> wave;
			std::vector<int> wave_chain;  // the chain of each picture of the wave
			for (size_t c = glo; c < ghi; c++) {
				Chain &ch = chains[c];
				if (ch.next > ch.last) continue;
				const Stream &s = b->streams[ch.stream];
				for (uint32_t p = ch.first + lo; p <= ch.last && p - ch.first < lo + width; p++) {
					const uint32_t end = p + 1 < s.pics.size() ? s.pics[p + 1] : s.bb.length;
					const int slot = b->free_slots.back();
					b->free_slots.pop_back();
					ch.slot[p - ch.first] = slot;
					wave.push_back({ch.stream, p, slot, walk_kind(b, s, p, b->decode_b), end - s.pics[p]});
					wave_chain.push_back((int)c);
				}
			}
			if (wave.empty()) break;
			parse_wave(b, wave, true);
			for (size_t t = 0; t < wave.size(); t++) {
				Chain &ch = chains[wave_chain[t]];
				ch.info[wave[t].pic - ch.first] = b->h_info[t];
			}
			// ---- decode()'s consumption rule over the infos (decode_round): which pictures reconstruct, at which depth
			std::vector<ReconStep> depths;
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
					for (int q = q_lo; q < q_hi; q++) {
						status[order[q]] = e.status;
						n_present[order[q]] = e.n_present;
						error[order[q]] = e.error;
					}
					const bool is_b = e.picture_type == 3;  // (only the B walk answers PIC_DECODED for one)
					if (e.status == PIC_DECODED && (!is_b || k < ch.b_end)) {
						const int slot = ch.slot[k - ch.first];
						const bool leaf = ch.n_sets == 0;
						uint8_t *out_rgba = rgba && q_hi > q_lo ? static_cast<uint8_t *>(rgba_dst[order[q_lo]]) : nullptr;
						ReconTask t;
						if (is_b)  // the two I/P sets: `cur` the older (forward), `1 - cur` the newer (backward) reference
							t = recon_task(b, s, slot, ch.set[2 + ch.b_cur], ch.set[ch.cur], ch.set[1 - ch.cur], out_rgba);
						else if (leaf)  // into the destination, predicted (skipped macroblocks) from the zeroed scratch set
							t = recon_task(b, s, slot, static_cast<uint8_t *>(planes_dst[order[q_lo]]), b->d_intra_fwd, nullptr, out_rgba);
						else
							t = recon_task(b, s, slot, ch.set[ch.cur], ch.set[1 - ch.cur], nullptr, out_rgba);
						if (depths.size() <= d) depths.emplace_back();
						ReconStep &dp = depths[d++];
						dp.add(t);
						for (int q = q_lo; q < q_hi; q++) {  // the first request gets the picture, duplicates a copy of it
							if (!leaf || q > q_lo) dp.copy(planes_dst[order[q]], t.cur.y, (size_t)s.coded_size * 3 / 2);
							if (rgba && q > q_lo) dp.copy(rgba_dst[order[q]], t.rgba, (size_t)s.width * s.height * 4);
						}
						if (is_b) ch.b_cur ^= 1;
						else ch.cur ^= 1;
					}
					// the next picture: the first picture start code at or after where this one's parse ended
					ch.next = (uint32_t)(std::lower_bound(s.pics.begin(), s.pics.end(), (e.end_bit + 7) >> 3) - s.pics.begin());
				}
			}
			// ---- stage 2: one depth after the other on the reconstruct stream, each followed by its copies (a set is
			// overwritten two references later, by a later launch on the same stream)
			for (ReconStep &dp : depths) {
				launch_step(dp, b->st_recon);
				if (!dp.dst.empty()) copy_batch(b, dp.dst, dp.src, dp.size, b->st_recon);
			}
			CUDA_CHECK(cudaEventRecord(b->ev_round, b->st_recon));
			b->recon_pending = true;
			for (const WaveItem &w : wave) release_slot(b, w.slot);  // reused by the next wave's parse, which waits for ev_round
		}
		for (size_t c = glo; c < ghi; c++)  // never consumed: planes 0 (a copied destination was not zeroed)
			if (chains[c].n_sets)
				for (int q = chains[c].req_lo; q < chains[c].req_hi; q++)
					if (status[order[q]] == 0) {
						const Stream &s = b->streams[chains[c].stream];
						CUDA_CHECK(cudaMemsetAsync(planes_dst[order[q]], 0, (size_t)s.coded_size * 3 / 2, b->st_recon));
					}
	}
	CUDA_CHECK(cudaStreamSynchronize(b->st_recon));
	b->recon_pending = false;
	for (int i = 0; i < n; i++) {
		if (status_out) status_out[i] = status[i];
		if (n_present_out) n_present_out[i] = n_present[i];
		if (error_out) error_out[i] = error[i];
	}
}

// The checks both front ends make of a request before anything changes: stream, sequence header, destinations
bool request_valid(const Batch *b, int si, void *planes, void *image, bool rgba) {
	auto aligned = [](const void *p) { return ((uintptr_t)p & 15u) == 0; };  // stage 2 stores 8 and 16 bytes at a time
	if (si < 0 || si >= (int)b->streams.size() || !b->streams[si].has_seq || !planes || !aligned(planes)) return false;
	return !rgba || (image && aligned(image));
}

// decode_intra (`intra`: requests are looked up in the intra index) and decode_pictures (in the picture index)
long batch_decode_chosen(Batch *b, bool intra, int n, const int *streams, const uint32_t *pictures, void *const *planes_dst,
                         void *const *rgba_dst, int flags, int32_t *status_out, int32_t *n_present_out, int32_t *error_out) {
	use_device(b);
	const bool rgba = (flags & JSMPEG_B200_OUT_RGBA) != 0;
	if (n < 0 || (n > 0 && (!streams || !pictures || !planes_dst || (rgba && !rgba_dst)))) return -2;
	upload_all(b);
	// ---- every request is checked before anything changes
	std::vector<std::vector<IndexEntry>> listed(b->streams.size());
	std::vector<char> indexed(b->streams.size(), 0);
	std::vector<PictureRequest> req(n);
	for (int i = 0; i < n; i++) {
		const int si = streams[i];
		if (!request_valid(b, si, planes_dst[i], rgba ? rgba_dst[i] : nullptr, rgba)) return -2;
		if (!indexed[si]) {
			listed[si] = intra ? intra_index(b->streams[si]) : picture_index(b, b->streams[si]);
			indexed[si] = 1;
		}
		auto e = std::lower_bound(listed[si].begin(), listed[si].end(), pictures[i],
		                          [](const IndexEntry &x, uint32_t k) { return x.pic < k; });
		if (e == listed[si].end() || e->pic != pictures[i]) return -2;
		req[i] = {si, pictures[i], e->chain_start};
	}
	if (n == 0) return 0;
	decode_chains(b, req, planes_dst, rgba_dst, rgba, status_out, n_present_out, error_out);
	return n;
}

// ---- decode_macroblocks: the walks' records of chosen pictures of any streams, in the public layout (DESIGN 3.8) ----

// The pictures decode_macroblocks can describe now: after the first sequence header, closed, and decoded by the walks
// with B pictures going to the B walk whatever decode_b says.  No chain start: a picture's macroblock layer depends on
// its own bits only.
std::vector<uint32_t> macroblock_index(const Stream &s) {
	std::vector<uint32_t> out;
	if (!s.has_seq) return out;
	for (uint32_t k = 0; k < s.pics.size(); k++)
		if (s.pics[k] >= s.seq_floor && picture_decoded(s, k, true) && picture_closed(s, k)) out.push_back(k);
	return out;
}

// Each unique (stream, picture) of the requests takes a record slot; waves of as many as there are free slots (after
// flushing the look-ahead when they do not cover the call) run the walks alone, and one export launch per wave, on the
// main stream behind the walks and before the slots are released, writes every request of the wave to its
// destination.  The next wave's walks are queued behind it.  The requests are valid (the caller checked them).
void decode_macroblocks(Batch *b, int n, const int *streams, const uint32_t *pictures, void *const *dst,
                        int32_t *n_present_out, int32_t *error_out) {
	ensure_pool(b);
	std::vector<std::pair<int, uint32_t>> uniq(n);
	for (int i = 0; i < n; i++) uniq[i] = {streams[i], pictures[i]};
	std::sort(uniq.begin(), uniq.end());
	uniq.erase(std::unique(uniq.begin(), uniq.end()), uniq.end());
	std::vector<size_t> uniq_of(n);  // request i describes picture uniq[uniq_of[i]]
	for (int i = 0; i < n; i++)
		uniq_of[i] = std::lower_bound(uniq.begin(), uniq.end(), std::make_pair(streams[i], pictures[i])) - uniq.begin();
	if (b->free_slots.size() < uniq.size())  // decode() parses the look-ahead again
		for (auto &s : b->streams) flush_cache(b, s);
	if (n > b->xtask_cap) {
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));
		if (b->h_xtasks) { CUDA_CHECK(cudaFreeHost(b->h_xtasks)); b->h_xtasks = nullptr; }
		if (b->d_xtasks) { CUDA_CHECK(cudaFree(b->d_xtasks)); b->d_xtasks = nullptr; }
		b->xtask_cap = 0;
		b->h_xtasks = pinned_alloc<MbExportTask>(n);
		b->d_xtasks = dev_alloc<MbExportTask>(n);
		b->xtask_cap = n;
	}
	const size_t wave_max = b->free_slots.size();
	std::vector<int32_t> n_present(n, 0), error(n, 0);
	for (size_t lo = 0; lo < uniq.size(); lo += wave_max) {
		const size_t hi = std::min(uniq.size(), lo + wave_max);
		std::vector<WaveItem> wave;
		for (size_t u = lo; u < hi; u++) {
			const Stream &s = b->streams[uniq[u].first];
			const uint32_t p = uniq[u].second;
			const uint32_t end = p + 1 < s.pics.size() ? s.pics[p + 1] : s.bb.length;
			const int slot = b->free_slots.back();
			b->free_slots.pop_back();
			wave.push_back({uniq[u].first, p, slot, walk_kind(b, s, p, true), end - s.pics[p]});
		}
		// (parse_wave waits for the infos, which also means the previous wave's task upload has read h_xtasks)
		parse_wave(b, wave, false);
		int m = 0;
		uint32_t total = 0;
		for (int i = 0; i < n; i++) {
			if (uniq_of[i] < lo || uniq_of[i] >= hi) continue;
			const WaveItem &w = wave[uniq_of[i] - lo];
			const picture_info_t &info = b->h_info[uniq_of[i] - lo];
			n_present[i] = info.n_present;
			error[i] = info.error;
			const int mb_size = b->streams[w.stream].seq.mb_size;
			b->h_xtasks[m++] = MbExportTask{b->d_hdr + (size_t)w.slot * b->slot_mb, dst[i], total, mb_size, info.picture_type, 0};
			total += (uint32_t)mb_size;
		}
		CUDA_CHECK(cudaMemcpyAsync(b->d_xtasks, b->h_xtasks, m * sizeof(MbExportTask), cudaMemcpyHostToDevice, b->st_main));
		launch_export_macroblocks(b->d_xtasks, m, total, b->st_main);
		for (const WaveItem &w : wave) release_slot(b, w.slot);  // the next wave's walks queue behind the export
	}
	CUDA_CHECK(cudaStreamSynchronize(b->st_main));
	for (int i = 0; i < n; i++) {
		if (n_present_out) n_present_out[i] = n_present[i];
		if (error_out) error_out[i] = error[i];
	}
}

long batch_decode_macroblocks(Batch *b, int n, const int *streams, const uint32_t *pictures, void *const *mb_dst,
                              int32_t *n_present_out, int32_t *error_out) {
	use_device(b);
	if (n < 0 || (n > 0 && (!streams || !pictures || !mb_dst))) return -2;
	upload_all(b);
	// ---- every request is checked before anything changes
	std::vector<std::vector<uint32_t>> listed(b->streams.size());
	std::vector<char> indexed(b->streams.size(), 0);
	for (int i = 0; i < n; i++) {
		const int si = streams[i];
		if (!request_valid(b, si, mb_dst[i], nullptr, false)) return -2;
		if (!indexed[si]) {
			listed[si] = macroblock_index(b->streams[si]);
			indexed[si] = 1;
		}
		if (!std::binary_search(listed[si].begin(), listed[si].end(), pictures[i])) return -2;
	}
	if (n == 0) return 0;
	decode_macroblocks(b, n, streams, pictures, mb_dst, n_present_out, error_out);
	return n;
}

int env_int(const char *name, int fallback) {
	const char *e = getenv(name);
	return e && *e ? atoi(e) : fallback;
}

// The tail of a device demux (write_ts, write_ps): `total` ES bytes that gather(es_base) writes to the HBM
// mirror at s.d_es + es_base are appended to the stream as if written with get_write_ptr / did_write.
// gather returns the number of PES starts it listed in pts_out / offset_out (unordered).
template <typename F>
long append_demuxed(Batch *b, Stream &s, uint32_t total, F &&gather, uint64_t *pts_out, uint32_t *offset_out, int n_max, int *n_pes) {
	// room in the host bit buffer (the reference's write protocol, may expand or evict) and in HBM
	uint8_t *hdst = static_cast<uint8_t *>(stream_get_write_ptr(b, s, total));
	reserve_device_es(b, s, s.bb.length + total);
	if (s.d_valid < s.bb.length) {  // bytes written the ordinary way that are not resident yet
		CUDA_CHECK(cudaMemcpyAsync(s.d_es + s.d_valid, s.bb.bytes + s.d_valid, s.bb.length - s.d_valid, cudaMemcpyHostToDevice, b->st_main));
		b->stats.h2d_bytes += s.bb.length - s.d_valid;
		s.d_valid = s.bb.length;
	}
	const int count = gather(s.bb.length);
	// the host keeps a mirror of the ES (sequence header parse, EVICT bookkeeping): copy the new bytes back
	CUDA_CHECK(cudaMemcpyAsync(hdst, s.d_es + s.bb.length, (size_t)total, cudaMemcpyDeviceToHost, b->st_main));
	CUDA_CHECK(cudaMemsetAsync(s.d_es + s.bb.length + total, 0, ES_PAD, b->st_main));
	CUDA_CHECK(cudaStreamSynchronize(b->st_main));
	b->stats.d2h_bytes += (uint64_t)total;
	stream_did_write(b, s, total);
	s.d_valid = s.bb.length;
	if (n_pes) *n_pes = count;
	if (pts_out && offset_out && count > 1) {  // the device appends PES starts unordered: sort by offset
		const int m = std::min(count, n_max);
		std::vector<std::pair<uint32_t, uint64_t>> v(m);
		for (int i = 0; i < m; i++) v[i] = {offset_out[i], pts_out[i]};
		std::sort(v.begin(), v.end());
		for (int i = 0; i < m; i++) { offset_out[i] = v[i].first; pts_out[i] = v[i].second; }
	}
	return total;
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
	try {
		use_device(b);
		CUDA_CHECK(cudaStreamCreateWithFlags(&b->st_main, cudaStreamNonBlocking));
		CUDA_CHECK(cudaStreamCreateWithFlags(&b->st_recon, cudaStreamNonBlocking));
		CUDA_CHECK(cudaStreamCreateWithFlags(&b->st_copy, cudaStreamNonBlocking));
		for (auto &st : b->st_side) CUDA_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
		cudaEvent_t *timed[] = {&b->ev_a, &b->ev_b, &b->ev_mid, &b->ev_recon[0], &b->ev_recon[1]};
		for (auto e : timed) CUDA_CHECK(cudaEventCreate(e));
		cudaEvent_t *untimed[] = {&b->ev_step, &b->ev_round, &b->ev_copied[0], &b->ev_copied[1], &b->ev_sfork, &b->ev_sjoin[0], &b->ev_sjoin[1]};
		for (auto e : untimed) CUDA_CHECK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
		CUDA_CHECK(cudaEventCreateWithFlags(&b->fork.fork, cudaEventDisableTiming));
		for (int i = 0; i < PARSE_GROUPS; i++) {
			CUDA_CHECK(cudaStreamCreateWithFlags(&b->fork.side[i], cudaStreamNonBlocking));
			CUDA_CHECK(cudaEventCreateWithFlags(&b->fork.join[i], cudaEventDisableTiming));
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
	for (auto &s : b->streams) {
		if (s.bb.bytes) cudaFreeHost(s.bb.bytes);
		if (s.d_seq) cudaFree(s.d_seq);
		if (s.d_es) cudaFree(s.d_es);
		if (s.d_rgba) cudaFree(s.d_rgba);
		for (auto p : s.d_planes) if (p) cudaFree(p);
		for (auto p : s.d_planes_b) if (p) cudaFree(p);
		for (auto p : s.h_planes) if (p) cudaFreeHost(p);
	}
	if (b->d_spans) cudaFree(b->d_spans);
	if (b->h_spans) cudaFreeHost(b->h_spans);
	if (b->d_scan_counts) cudaFree(b->d_scan_counts);
	if (b->h_scan_counts) cudaFreeHost(b->h_scan_counts);
	if (b->d_scan_pos) cudaFree(b->d_scan_pos);
	if (b->h_scan_pos) cudaFreeHost(b->h_scan_pos);
	if (b->d_codes) cudaFree(b->d_codes);
	if (b->h_codes) cudaFreeHost(b->h_codes);
	if (b->d_hdr) cudaFree(b->d_hdr);
	if (b->d_coef) cudaFree(b->d_coef);
	if (b->d_park) cudaFree(b->d_park);
	if (b->d_stage) cudaFree(b->d_stage);
	if (b->d_info) cudaFree(b->d_info);
	if (b->h_info) cudaFreeHost(b->h_info);
	if (b->h_ptasks) cudaFreeHost(b->h_ptasks);
	if (b->d_ptasks) cudaFree(b->d_ptasks);
	if (b->d_intra_fwd) cudaFree(b->d_intra_fwd);
	if (b->d_chain_sets) cudaFree(b->d_chain_sets);
	if (b->h_xtasks) cudaFreeHost(b->h_xtasks);
	if (b->d_xtasks) cudaFree(b->d_xtasks);
	ts_scratch_destroy(b->ts);
	ps_scratch_destroy(b->ps);
	for (auto e : {b->ev_a, b->ev_b, b->ev_mid, b->ev_recon[0], b->ev_recon[1], b->ev_step, b->ev_round, b->ev_copied[0],
	               b->ev_copied[1], b->ev_sfork, b->ev_sjoin[0], b->ev_sjoin[1], b->fork.fork}) if (e) cudaEventDestroy(e);
	for (int i = 0; i < PARSE_GROUPS; i++) {
		if (b->fork.join[i]) cudaEventDestroy(b->fork.join[i]);
		if (b->fork.side[i]) cudaStreamDestroy(b->fork.side[i]);
	}
	for (auto st : {b->st_main, b->st_recon, b->st_copy, b->st_side[0], b->st_side[1]}) if (st) cudaStreamDestroy(st);
	(void)cudaGetLastError();
	delete b;
}

const char *jsmpeg_b200_batch_last_error(jsmpeg_b200_batch_t *b) { return (b && b->dead) ? b->error.c_str() : nullptr; }

int jsmpeg_b200_batch_set_option(jsmpeg_b200_batch_t *b, const char *name, int value) {
	if (!b || !name) return -1;
	if (!strcmp(name, "lookahead")) { b->lookahead = std::max(1, value); return 0; }
	if (!strcmp(name, "slice_walk")) { b->slice_walk = value != 0; return 0; }  // (same records either way: nothing to flush)
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
	}
}

void jsmpeg_b200_batch_reset(jsmpeg_b200_batch_t *b) {
	guarded_void(b, [&] {
		use_device(b);
		for (auto &s : b->streams) {
			forget_index(b, s);
			s.bb.length = 0;
			s.bb.index = 0;
			s.cur = 0;
			s.b_cur = 0;
			s.d_last = nullptr;
			s.last_type = s.last_temporal = 0;
			s.h_head = -1;
			s.seq_floor = 0;
			if (s.has_seq) {
				for (auto p : s.d_planes) CUDA_CHECK(cudaMemsetAsync(p, 0, (size_t)s.coded_size * 3 / 2, b->st_main));
				for (auto p : s.d_planes_b) if (p) CUDA_CHECK(cudaMemsetAsync(p, 0, (size_t)s.coded_size * 3 / 2, b->st_main));
			}
		}
		CUDA_CHECK(cudaStreamSynchronize(b->st_main));
	});
}

long jsmpeg_b200_batch_decode(jsmpeg_b200_batch_t *b, int n_pictures, int flags) {
	return guarded<long>(b, 0, [&] { return batch_decode(b, n_pictures, flags); });
}

long jsmpeg_b200_batch_intra_index(jsmpeg_b200_batch_t *b, int stream, uint32_t *picture_out, uint32_t *byte_pos_out,
                                   int32_t *temporal_reference_out, long n_max) {
	return guarded<long>(b, -1, [&]() -> long {
		if (stream < 0 || stream >= (int)b->streams.size()) return -2;
		use_device(b);
		upload_all(b);
		const Stream &s = b->streams[stream];
		const std::vector<IndexEntry> listed = intra_index(s);
		for (long i = 0; i < std::min<long>((long)listed.size(), n_max); i++) {
			const uint32_t pos = s.pics[listed[i].pic];
			if (picture_out) picture_out[i] = listed[i].pic;
			if (byte_pos_out) byte_pos_out[i] = pos;
			if (temporal_reference_out) temporal_reference_out[i] = s.bb.bytes[pos + 4] << 2 | s.bb.bytes[pos + 5] >> 6;
		}
		return (long)listed.size();
	});
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
	return guarded<long>(b, -1, [&]() -> long {
		if (stream < 0 || stream >= (int)b->streams.size()) return -2;
		use_device(b);
		upload_all(b);
		const Stream &s = b->streams[stream];
		const std::vector<IndexEntry> listed = picture_index(b, s);
		for (long i = 0; i < std::min<long>((long)listed.size(), n_max); i++) {
			const uint32_t k = listed[i].pic;
			if (picture_out) picture_out[i] = k;
			if (byte_pos_out) byte_pos_out[i] = s.pics[k];
			if (type_out) type_out[i] = picture_type_of(s, k);
			if (temporal_reference_out) temporal_reference_out[i] = (int32_t)picture_header_bits(s, k, 0, 10);
			if (chain_start_out) chain_start_out[i] = listed[i].chain_start;
		}
		return (long)listed.size();
	});
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
	return guarded<long>(b, -1, [&]() -> long {
		if (stream < 0 || stream >= (int)b->streams.size()) return -2;
		use_device(b);
		upload_all(b);
		const Stream &s = b->streams[stream];
		const std::vector<uint32_t> listed = macroblock_index(s);
		for (long i = 0; i < std::min<long>((long)listed.size(), n_max); i++) {
			const uint32_t k = listed[i];
			if (picture_out) picture_out[i] = k;
			if (byte_pos_out) byte_pos_out[i] = s.pics[k];
			if (type_out) type_out[i] = picture_type_of(s, k);
			if (temporal_reference_out) temporal_reference_out[i] = (int32_t)picture_header_bits(s, k, 0, 10);
		}
		return (long)listed.size();
	});
}

long jsmpeg_b200_batch_decode_macroblocks(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                          void *const *mb_dst, int32_t *n_present_out, int32_t *error_out) {
	return guarded<long>(b, -1, [&] { return batch_decode_macroblocks(b, n, streams, pictures, mb_dst, n_present_out, error_out); });
}

int jsmpeg_b200_batch_get_planes(jsmpeg_b200_batch_t *b, int stream, void **y, void **cr, void **cb) {
	const Stream &s = b->streams[stream];
	if (!s.has_seq) return -1;
	// most recent picture = forward (mpeg1.c:841-851); with the B-picture extension it may be a B picture's own set
	PlaneSet p = plane_set(s, s.d_last ? s.d_last : s.d_planes[1 - s.cur]);
	if (y) *y = p.y;
	if (cr) *cr = p.cr;
	if (cb) *cb = p.cb;
	return 0;
}

int jsmpeg_b200_batch_get_host_planes(jsmpeg_b200_batch_t *b, int stream, void **y, void **cr, void **cb) {
	const Stream &s = b->streams[stream];
	if (!s.has_seq) return -1;
	PlaneSet p = plane_set(s, s.h_planes[s.h_head < 0 ? 0 : s.h_head]);
	if (y) *y = p.y;
	if (cr) *cr = p.cr;
	if (cb) *cb = p.cb;
	return 0;
}

int jsmpeg_b200_batch_get_rgba(jsmpeg_b200_batch_t *b, int stream, void **rgba) {
	const Stream &s = b->streams[stream];
	if (!s.has_seq || !s.d_rgba) return -1;
	*rgba = s.d_rgba;
	return 0;
}

int jsmpeg_b200_batch_read_planes(jsmpeg_b200_batch_t *b, int stream, void *y, void *cr, void *cb) {
	return guarded<int>(b, -1, [&] {
		use_device(b);
		const Stream &s = b->streams[stream];
		if (!s.has_seq) return -1;
		PlaneSet p = plane_set(s, s.d_last ? s.d_last : s.d_planes[1 - s.cur]);
		if (y) CUDA_CHECK(cudaMemcpy(y, p.y, s.coded_size, cudaMemcpyDeviceToHost));
		if (cr) CUDA_CHECK(cudaMemcpy(cr, p.cr, s.coded_size >> 2, cudaMemcpyDeviceToHost));
		if (cb) CUDA_CHECK(cudaMemcpy(cb, p.cb, s.coded_size >> 2, cudaMemcpyDeviceToHost));
		return 0;
	});
}

long jsmpeg_b200_batch_write_ts(jsmpeg_b200_batch_t *b, int stream, const uint8_t *ts, size_t n_bytes, int stream_id,
                                uint64_t *pts_out, uint32_t *offset_out, int n_max, int *n_pes) {
	if (n_pes) *n_pes = 0;
	return guarded<long>(b, -1, [&]() -> long {
		use_device(b);
		Stream &s = b->streams[stream];
		if (!b->ts) b->ts = ts_scratch_create();
		if (s.ts_bound.empty()) s.ts_bound.assign(8192, 0);
		// what the previous call left over comes first (a partial packet, a resync that wanted more data: ts.js:25-41)
		const uint8_t *data = ts;
		size_t n_data = n_bytes;
		if (!s.ts_leftover.empty()) {
			s.ts_leftover.insert(s.ts_leftover.end(), ts, ts + n_bytes);
			data = s.ts_leftover.data();
			n_data = s.ts_leftover.size();
		}
		size_t consumed = 0;
		const long total = ts_demux_measure(b->ts, data, n_data, stream_id, s.ts_bound.data(), &consumed, b->st_main);
		std::vector<uint8_t> rest(data + consumed, data + n_data);  // (data may alias ts_leftover)
		s.ts_leftover.swap(rest);
		if (total <= 0) return total;
		b->stats.kernel_launches += 7;
		b->stats.h2d_bytes += n_data;
		return append_demuxed(b, s, (uint32_t)total, [&](uint32_t es_base) {
			return ts_demux_gather(b->ts, s.d_es, es_base, pts_out, offset_out, n_max, b->st_main);
		}, pts_out, offset_out, n_max, n_pes);
	});
}

long jsmpeg_b200_batch_write_ps(jsmpeg_b200_batch_t *b, int stream, const uint8_t *ps, size_t n_bytes, int stream_id,
                                uint64_t *pts_out, uint32_t *offset_out, int n_max, int *n_pes) {
	if (n_pes) *n_pes = 0;
	return guarded<long>(b, -1, [&]() -> long {
		if (stream_id < 0xE0 || stream_id > 0xEF) return -2;  // not a video stream id: the caller's mistake, nothing changes
		use_device(b);
		Stream &s = b->streams[stream];
		if (!b->ps) b->ps = ps_scratch_create();
		// what the previous call left over comes first: an unfinished item, or the tail that may begin a pack header
		const uint8_t *data = ps;
		size_t n_data = n_bytes;
		if (!s.ps_leftover.empty()) {
			s.ps_leftover.insert(s.ps_leftover.end(), ps, ps + n_bytes);
			data = s.ps_leftover.data();
			n_data = s.ps_leftover.size();
		}
		size_t consumed = 0;
		const long total = ps_demux_measure(b->ps, data, n_data, stream_id, &s.ps_in_sync, &consumed, b->st_main);
		std::vector<uint8_t> rest(data + consumed, data + n_data);  // (data may alias ps_leftover)
		s.ps_leftover.swap(rest);
		b->stats.h2d_bytes += n_data;
		long r = total;
		if (total > 0)
			r = append_demuxed(b, s, (uint32_t)total, [&](uint32_t es_base) {
				return ps_demux_gather(b->ps, s.d_es, es_base, pts_out, offset_out, n_max, b->st_main);
			}, pts_out, offset_out, n_max, n_pes);
		b->stats.kernel_launches += ps_demux_launches(b->ps);
		return r;
	});
}

int jsmpeg_b200_batch_read_rgba(jsmpeg_b200_batch_t *b, int stream, void *rgba) {
	return guarded<int>(b, -1, [&] {
		use_device(b);
		const Stream &s = b->streams[stream];
		if (!s.has_seq || !s.d_rgba) return -1;
		CUDA_CHECK(cudaMemcpy(rgba, s.d_rgba, (size_t)s.width * s.height * 4, cudaMemcpyDeviceToHost));
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
	return self ? jsmpeg_b200_batch_set_option(self->b, name, value) : -1;
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
	return jsmpeg_b200_batch_decode(self->b, 1, JSMPEG_B200_OUT_HOST) > 0;
}

// ================================================================================================
// test hooks

long jsmpeg_b200_debug_read_es(jsmpeg_b200_batch_t *b, int stream, void *dst, size_t cap) {
	return guarded<long>(b, -1, [&]() -> long {
		use_device(b);
		const Stream &s = b->streams[stream];
		const size_t n = std::min<size_t>(cap, s.d_valid);
		if (n) CUDA_CHECK(cudaMemcpy(dst, s.d_es, n, cudaMemcpyDeviceToHost));
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
		uint8_t *d_es = dev_alloc<uint8_t>(es_len + ES_PAD);
		SeqParams *d_seq = dev_alloc<SeqParams>(1);
		mb_record_t *d_hdr = dev_alloc<mb_record_t>(n_mb);
		int16_t *d_coef = dev_alloc<int16_t>(n_mb * MB_COEF_INT16);
		uint2 *d_park = dev_alloc<uint2>(n_mb * 6);
		uint4 *d_stage = dev_alloc<uint4>((size_t)stage_entries_for(sp.mb_size) * 4);
		picture_info_t *d_info = dev_alloc<picture_info_t>(1);
		ParseTask *d_task = dev_alloc<ParseTask>(1);
		CUDA_CHECK(cudaMemcpy(d_es, es, es_len, cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemset(d_es + es_len, 0, ES_PAD));
		CUDA_CHECK(cudaMemcpy(d_seq, &sp, sizeof(sp), cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemset(d_coef, 0, n_mb * MB_COEF_INT16 * sizeof(int16_t)));
		ParseTask t{};
		t.es = d_es; t.es_len = es_len; t.start_byte = start_byte; t.seq = d_seq; t.hdr = d_hdr; t.coef = d_coef; t.info = d_info;
		t.park = d_park; t.mb_width = mb_width; t.mb_size = sp.mb_size;
		t.stage = d_stage; t.stage_entries = stage_entries_for(sp.mb_size);
		t.codes = nullptr; t.n_codes = 0; t.code_hint = 0;  // this hook lets the walk search the slice end itself
		CUDA_CHECK(cudaMemcpy(d_task, &t, sizeof(t), cudaMemcpyHostToDevice));
		launch_parse_pictures(d_task, 1, sp.mb_size, true, 0);
		CUDA_CHECK(cudaGetLastError());
		CUDA_CHECK(cudaDeviceSynchronize());
		CUDA_CHECK(cudaMemcpy(info_out, d_info, sizeof(picture_info_t), cudaMemcpyDeviceToHost));
		CUDA_CHECK(cudaMemcpy(hdr_out, d_hdr, n_mb * sizeof(mb_record_t), cudaMemcpyDeviceToHost));
		CUDA_CHECK(cudaMemcpy(coef_out, d_coef, n_mb * MB_COEF_INT16 * sizeof(int16_t), cudaMemcpyDeviceToHost));
		// stage 1b left most blocks as compact records in the staging area: the caller gets them dense
		std::vector<coef_record_t> compact(n_mb * 6);
		CUDA_CHECK(cudaMemcpy(compact.data(), d_stage, compact.size() * sizeof(coef_record_t), cudaMemcpyDeviceToHost));
		const mb_record_t *hdr = static_cast<const mb_record_t *>(hdr_out);
		for (size_t slot = 0; slot < n_mb * 6; slot++) {
			const mb_record_t &r = hdr[slot / 6];
			if ((r.flags & MBF_PRESENT) && (r.cbp & (0x20 >> (slot % 6))) && compact[slot].mask != COEF_RECORD_DENSE)
				coef_record_unpack(compact[slot], static_cast<int16_t *>(coef_out) + slot * 64);
		}
		cudaFree(d_es); cudaFree(d_seq); cudaFree(d_hdr); cudaFree(d_coef); cudaFree(d_park); cudaFree(d_stage); cudaFree(d_info); cudaFree(d_task);
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
		mb_record_t *d_hdr = dev_alloc<mb_record_t>(n_mb);
		int16_t *d_coef = dev_alloc<int16_t>(n_mb * MB_COEF_INT16);
		// the caller's dense blocks as stage 1b would hand them over: compact records where they fit
		std::vector<coef_record_t> compact(n_mb * 6);
		for (size_t slot = 0; slot < n_mb * 6; slot++) {
			const int16_t *blk = static_cast<const int16_t *>(coef) + slot * 64;
			const uint64_t pos = coef_nonzero_positions(blk);
			if (coef_record_fits(pos)) compact[slot] = coef_record_pack(pos, blk);
			else compact[slot].mask = COEF_RECORD_DENSE;
		}
		coef_record_t *d_compact = dev_alloc<coef_record_t>(n_mb * 6);
		CUDA_CHECK(cudaMemcpy(d_compact, compact.data(), compact.size() * sizeof(coef_record_t), cudaMemcpyHostToDevice));
		const size_t pad = (size_t)mb_width * 16 + 64;
		uint8_t *d_fwd = dev_alloc<uint8_t>(total + pad), *d_cur = dev_alloc<uint8_t>(total + pad);
		CUDA_CHECK(cudaMemset(d_fwd + total, 0, pad));
		CUDA_CHECK(cudaMemcpy(d_hdr, hdr, n_mb * sizeof(mb_record_t), cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_coef, coef, n_mb * MB_COEF_INT16 * sizeof(int16_t), cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_fwd, fwd_y, ysz, cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_fwd + ysz, fwd_cr, csz, cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_fwd + ysz + csz, fwd_cb, csz, cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_cur, cur_y, ysz, cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_cur + ysz, cur_cr, csz, cudaMemcpyHostToDevice));
		CUDA_CHECK(cudaMemcpy(d_cur + ysz + csz, cur_cb, csz, cudaMemcpyHostToDevice));
		ReconTask t{};
		t.hdr = d_hdr; t.coef = d_coef; t.compact = d_compact;
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
		cudaFree(d_hdr); cudaFree(d_coef); cudaFree(d_compact); cudaFree(d_fwd); cudaFree(d_cur);
		return 0;
	} catch (const std::exception &e) {
		fprintf(stderr, "%s\n", e.what());
		return -1;
	}
}

}  // extern "C"
