// ts_many_check.cpp -- the segmented MPEG-TS pass of tsdemux.cu run sequentially on the host with the device's
// per-packet arithmetic (jsmpeg_b200/csrc/tsdemux.cuh), for tests/test_ts_many_emu.py.
//
//   ts_many_check IN OUT
// IN: u32 n_streams, u32 n_calls; per call u32 n_req, per request i32 stream, i32 stream_id, u32 len, len bytes.
// OUT: per call and request u32 appended, u32 n_pes, u32 left-over bytes after it; then per stream u32 es_len, the ES,
// u32 n_pes, (u32 offset, u64 pts) each, u32 leftover_len, the bytes, u32 n_bound, (u32 pid, i32 stream id) each.
// Every step is the kernel's loop body over its threads, in the kernel order of ts_call_measure / ts_call_gather.
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "../../jsmpeg_b200/csrc/tsdemux.cuh"

struct StreamState {
	std::vector<uint8_t> es, leftover;
	std::vector<int16_t> bound = std::vector<int16_t>(8192, 0);
	std::vector<std::pair<uint32_t, uint64_t>> pes;
};

static uint32_t request_of(const std::vector<TsReq> &req, uint32_t n_req, uint32_t slot) {
	uint32_t r = 0;
	while (r + 1 < n_req && req[r + 1].slot0 <= slot) r++;
	return r;
}

static void call(std::vector<StreamState> &st, const std::vector<int> &streams, const std::vector<int> &sids,
                 const std::vector<std::vector<uint8_t>> &bufs, std::vector<uint32_t> &out_rows) {
	const uint32_t n = (uint32_t)streams.size();
	std::vector<uint8_t> stage;
	std::vector<TsReq> req(n + 1);
	uint32_t slot = 0;
	for (uint32_t i = 0; i < n; i++) {
		StreamState &s = st[streams[i]];
		const uint32_t len = (uint32_t)(s.leftover.size() + bufs[i].size());
		const bool whole = len >= 188;
		req[i] = TsReq{(uint32_t)stage.size(), whole ? len : 0, slot, sids[i], s.bound.data(), nullptr, 0, 0};
		if (!whole) continue;
		stage.insert(stage.end(), s.leftover.begin(), s.leftover.end());
		stage.insert(stage.end(), bufs[i].begin(), bufs[i].end());
		slot += len / 188;
	}
	req[n] = TsReq{(uint32_t)stage.size(), 0, slot, 0, nullptr, nullptr, 0, 0};
	const uint32_t m = slot;
	std::vector<TsReqOut> out(n, TsReqOut{0, 0, 0, 0, 0, 0});
	std::vector<uint32_t> grid(m + 1);
	// check grid
	for (uint32_t i = 0; i < m; i++) {
		const uint32_t r = request_of(req, n, i);
		if (stage[req[r].base + (i - req[r].slot0) * 188u] != 0x47) out[r].misaligned = 1;
	}
	// walk grid: the warp's steps one packet at a time
	for (uint32_t r = 0; r < n; r++) {
		const uint32_t len = req[r].n, cap = req[r + 1].slot0 - req[r].slot0;
		if (!out[r].misaligned) { out[r].count = cap; out[r].stop = cap * 188u; continue; }
		const uint8_t *ts = stage.data() + req[r].base;
		uint32_t pos = 0, count = 0;
		while (len - pos >= 188u) {
			if (ts[pos] == 0x47) { grid[req[r].slot0 + count++] = pos; pos += 188; continue; }
			pos += 1;
			if (len - pos < TS_RESYNC_BYTES) break;
			int found = -1;
			for (uint32_t i = 0; i < 187 && found < 0; i++) if (ts_resync_at(ts, pos, i)) found = (int)i;
			if (found < 0) { pos += 187; break; }
			grid[req[r].slot0 + count++] = pos + (uint32_t)found;
			pos = pos + (uint32_t)found + 188u;
		}
		out[r].count = count;
		out[r].stop = pos;
	}
	// classify
	std::vector<TsPacketInfo> info(m);
	std::vector<uint64_t> pts(m), key(m);
	std::vector<uint32_t> val(m);
	for (uint32_t i = 0; i < m; i++) {
		const uint32_t r = request_of(req, n, i), k = i - req[r].slot0;
		TsPacketInfo pi{0, 0, 0, 188, 0};
		uint64_t t = 0;
		if (k < out[r].count) pi = ts_classify(stage.data() + req[r].base, req[r].n, out[r].misaligned ? grid[i] : k * 188u, &t);
		info[i] = pi;
		pts[i] = t;
		key[i] = (pi.flags & 2) ? ts_event_key(r, pi.pid, i) : TS_NO_EVENT;
		val[i] = pi.sid;
	}
	// sort the events (stable, like the radix sort)
	std::vector<uint32_t> order(m);
	for (uint32_t i = 0; i < m; i++) order[i] = i;
	std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
	std::vector<uint64_t> skey(m);
	std::vector<uint32_t> sval(m);
	for (uint32_t i = 0; i < m; i++) { skey[i] = key[order[i]]; sval[i] = val[order[i]]; }
	// bind (every slot reads the tables before carry writes them)
	std::vector<TsPacketUse> use(m);
	std::vector<uint64_t> lenpes(m + 1, 0);
	for (uint32_t i = 0; i < m; i++) {
		TsPacketUse u{0, 0};
		int pes = 0;
		if (info[i].flags & 1) {
			const uint32_t r = request_of(req, n, i);
			u = ts_use(info[i], ts_binding(skey.data(), sval.data(), m, r, info[i].pid, i, req[r].bound), req[r].stream_id, &pes);
		}
		use[i] = u;
		lenpes[i] = (uint64_t)u.len << 32 | (uint64_t)pes;
	}
	// carry
	for (uint32_t e = 0; e < m; e++) {
		if (skey[e] == TS_NO_EVENT) continue;
		const uint64_t group = skey[e] >> TS_SLOT_BITS;
		if (e + 1 == m || (skey[e + 1] >> TS_SLOT_BITS) != group)
			req[(uint32_t)(group >> TS_PID_BITS)].bound[group & 8191u] = (int16_t)sval[e];
	}
	// scan, totals
	std::vector<uint64_t> scan(m + 1, 0);
	for (uint32_t i = 0; i < m; i++) scan[i + 1] = scan[i] + lenpes[i];
	for (uint32_t r = 0; r < n; r++) {
		const uint64_t a = scan[req[r].slot0], b = scan[req[r + 1].slot0];
		out[r].total = (uint32_t)(b >> 32) - (uint32_t)(a >> 32);
		out[r].pes = (uint32_t)b - (uint32_t)a;
		out[r].pes_first = (uint32_t)a;
	}
	// the host makes room, the gather places the payloads (the stream's ES grows in place here)
	std::vector<uint32_t> pes_offset(m), es_base(n);
	std::vector<uint64_t> pes_pts(m);
	for (uint32_t r = 0; r < n; r++) {
		StreamState &s = st[streams[r]];
		es_base[r] = (uint32_t)s.es.size();
		if (out[r].total) s.es.resize(s.es.size() + out[r].total);
	}
	for (uint32_t w = 0; w < m; w++) {
		const uint32_t r = request_of(req, n, w), k = w - req[r].slot0;
		if (k >= out[r].count || !out[r].total) continue;
		const uint32_t off = (uint32_t)(scan[w] >> 32) - (uint32_t)(scan[req[r].slot0] >> 32);
		if ((uint32_t)scan[w + 1] != (uint32_t)scan[w]) {
			pes_offset[(uint32_t)scan[w]] = es_base[r] + off;
			pes_pts[(uint32_t)scan[w]] = pts[w];
		}
		const uint8_t *src = stage.data() + req[r].base + (out[r].misaligned ? grid[w] : k * 188u) + use[w].start;
		std::copy(src, src + use[w].len, st[streams[r]].es.begin() + es_base[r] + off);
	}
	for (uint32_t r = 0; r < n; r++) {
		StreamState &s = st[streams[r]];
		if (out[r].total)
			for (uint32_t k = 0; k < out[r].pes; k++) s.pes.push_back({pes_offset[out[r].pes_first + k], pes_pts[out[r].pes_first + k]});
		std::vector<uint8_t> data = s.leftover;
		data.insert(data.end(), bufs[r].begin(), bufs[r].end());
		s.leftover.assign(data.begin() + out[r].stop, data.end());
		out_rows.push_back(out[r].total);
		out_rows.push_back(out[r].total ? out[r].pes : 0);
		out_rows.push_back((uint32_t)s.leftover.size());
	}
}

static uint32_t rd32(FILE *f) {
	uint32_t v;
	if (fread(&v, 4, 1, f) != 1) { fprintf(stderr, "short input\n"); exit(2); }
	return v;
}

int main(int argc, char **argv) {
	if (argc != 3) { fprintf(stderr, "usage: ts_many_check IN OUT\n"); return 2; }
	FILE *in = fopen(argv[1], "rb");
	if (!in) return 2;
	const uint32_t n_streams = rd32(in), n_calls = rd32(in);
	std::vector<StreamState> st(n_streams);
	std::vector<uint32_t> rows;
	for (uint32_t c = 0; c < n_calls; c++) {
		const uint32_t n = rd32(in);
		std::vector<int> streams(n), sids(n);
		std::vector<std::vector<uint8_t>> bufs(n);
		for (uint32_t i = 0; i < n; i++) {
			streams[i] = (int)rd32(in);
			sids[i] = (int)rd32(in);
			bufs[i].resize(rd32(in));
			if (!bufs[i].empty() && fread(bufs[i].data(), 1, bufs[i].size(), in) != bufs[i].size()) return 2;
		}
		call(st, streams, sids, bufs, rows);
	}
	fclose(in);
	FILE *o = fopen(argv[2], "wb");
	if (!o) return 2;
	fwrite(rows.data(), 4, rows.size(), o);
	for (const StreamState &s : st) {
		uint32_t k = (uint32_t)s.es.size();
		fwrite(&k, 4, 1, o);
		fwrite(s.es.data(), 1, k, o);
		k = (uint32_t)s.pes.size();
		fwrite(&k, 4, 1, o);
		for (auto &p : s.pes) { fwrite(&p.first, 4, 1, o); fwrite(&p.second, 8, 1, o); }
		k = (uint32_t)s.leftover.size();
		fwrite(&k, 4, 1, o);
		fwrite(s.leftover.data(), 1, k, o);
		std::vector<std::pair<uint32_t, int32_t>> b;
		for (uint32_t pid = 0; pid < 8192; pid++) if (s.bound[pid]) b.push_back({pid, s.bound[pid]});
		k = (uint32_t)b.size();
		fwrite(&k, 4, 1, o);
		for (auto &p : b) { fwrite(&p.first, 4, 1, o); fwrite(&p.second, 4, 1, o); }
	}
	fclose(o);
	return 0;
}
