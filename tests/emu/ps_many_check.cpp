// ps_many_check.cpp -- the many-request program stream pass of psdemux.cu run sequentially on the host with the
// device's step functions (jsmpeg_b200/csrc/psdemux.cuh), for tests/test_ps_many_emu.py.
//
//   ps_many_check IN OUT
// IN: u32 n_streams, u32 n_calls; per call u32 n_req, per request i32 stream, i32 stream_id, u32 len, len bytes.
// OUT: per call and request u32 appended, u32 n_pes, u32 left-over bytes after it, u32 in_sync after it, u32 k and the
// k positions (relative to the request) of the whole items its chain marked; then per stream u32 es_len, the ES,
// u32 n_pes, (u32 offset, u64 pts) each, u32 leftover_len, the bytes, u32 in_sync.
// Every step is the kernel's loop body over its threads, in the kernel order of ps_call_candidates / ps_call_measure /
// ps_call_gather.  The alignment padding between requests is filled with pack-header bytes, and the candidates are
// listed in a scrambled order before the sort, as the device's atomics may list them.
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <random>
#include <vector>

#include "../../jsmpeg_b200/csrc/psdemux.cuh"

struct StreamState {
	std::vector<uint8_t> es, leftover;
	bool in_sync = false;
	std::vector<std::pair<uint32_t, uint64_t>> pes;
};

static uint32_t request_at(const std::vector<PsReq> &req, uint32_t g) {
	uint32_t r = PS_NONE;
	for (uint32_t k = 0; k < req.size(); k++)
		if (req[k].base <= g) r = k;
	return r != PS_NONE && g - req[r].base < req[r].n ? r : PS_NONE;
}

static std::mt19937 scramble(12345);

static void call(std::vector<StreamState> &st, const std::vector<int> &streams, const std::vector<int> &sids,
                 const std::vector<std::vector<uint8_t>> &bufs, std::vector<uint32_t> &rows) {
	const uint32_t n = (uint32_t)streams.size();
	std::vector<uint8_t> stage;
	std::vector<PsReq> req(n);
	const uint8_t fill[5] = {0x00, 0x00, 0x01, 0xBA, 0x21};
	for (uint32_t i = 0; i < n; i++) {
		StreamState &s = st[streams[i]];
		req[i] = PsReq{(uint32_t)stage.size(), (uint32_t)(s.leftover.size() + bufs[i].size()), sids[i], s.in_sync ? 1u : 0u, nullptr, 0, 0};
		stage.insert(stage.end(), s.leftover.begin(), s.leftover.end());
		stage.insert(stage.end(), bufs[i].begin(), bufs[i].end());
		for (uint32_t k = 0; stage.size() % 16; k++) stage.push_back(fill[k % 5]);
	}
	const uint32_t staged = (uint32_t)stage.size();
	stage.insert(stage.end(), 32, 0);
	// candidates
	std::vector<PsReqOut> out(n, PsReqOut{0, 0, 0, 0, 0, 0, 0, 0, 0, 0});
	std::vector<uint32_t> sel;
	uint32_t most = 0;
	for (uint32_t g = 0; g + 2 < staged; g++) {
		if (stage[g] != 0 || stage[g + 1] != 0 || stage[g + 2] != 1) continue;
		const uint32_t r = request_at(req, g);
		if (r == PS_NONE || !ps_keep(stage.data() + req[r].base, req[r].n, g - req[r].base)) continue;
		sel.push_back(g);
		most = std::max(most, ++out[r].count);
	}
	std::shuffle(sel.begin(), sel.end(), scramble);
	const uint32_t m = (uint32_t)sel.size();
	int levels = 1;
	while ((1u << levels) < most) levels++;
	// sort
	std::vector<uint32_t> pos = sel;
	std::sort(pos.begin(), pos.end());
	// pack: rev and every request's first candidate; then the suffix minimum
	std::vector<uint32_t> rev(m), npr(m);
	for (uint32_t i = 0; i < m; i++) {
		const uint32_t r = request_at(req, pos[i]);
		rev[m - 1 - i] = ps_is_pack(stage.data() + req[r].base, req[r].n, pos[i] - req[r].base) ? i : PS_NONE;
	}
	for (uint32_t r = 0; r < n; r++) out[r].c0 = ps_lower(pos.data(), 0, m, req[r].base);
	for (uint32_t k = 0; k < m; k++) npr[k] = k ? std::min(npr[k - 1], rev[k]) : rev[k];
	auto cands = [&](uint32_t r) { return PsCands{pos.data(), npr.data(), m, out[r].c0, out[r].c0 + out[r].count, req[r].base}; };
	// link
	std::vector<std::vector<uint32_t>> jump(levels + 1, std::vector<uint32_t>(m));
	std::vector<uint32_t> term_kind(m), term_stop(m);
	for (uint32_t i = 0; i < m; i++) {
		const uint32_t r = request_at(req, pos[i]);
		const PsStep s = ps_link(stage.data() + req[r].base, req[r].n, cands(r), i);
		if (s.kind == PS_T_LINK && (s.next <= i || s.next >= out[r].c0 + out[r].count)) { fprintf(stderr, "link leaves its request\n"); exit(3); }
		jump[0][i] = s.kind == PS_T_LINK ? s.next : i;
		term_kind[i] = s.kind;
		term_stop[i] = s.stop;
	}
	// doubling
	for (int k = 0; k < levels; k++)
		for (uint32_t i = 0; i < m; i++) jump[k + 1][i] = jump[k][jump[k][i]];
	// heads
	std::vector<uint8_t> marked(m, 0);
	for (uint32_t r = 0; r < n; r++) {
		const PsStep s = ps_head(stage.data() + req[r].base, req[r].n, cands(r), req[r].in_sync != 0);
		if (s.kind == PS_T_LINK) {
			out[r].head = s.next;
			marked[s.next] = 1;
		} else {
			out[r].head = PS_NONE;
			out[r].kind = s.kind;
			out[r].stop = s.stop;
		}
	}
	// marking
	for (int k = levels; k >= 0; k--)
		for (uint32_t i = 0; i < m; i++)
			if (marked[i]) marked[jump[k][i]] = 1;
	// classify
	std::vector<uint64_t> key(m + 1, 0), pts(m, 0);
	std::vector<uint32_t> src(m, 0);
	for (uint32_t i = 0; i < m; i++) {
		if (!marked[i]) continue;
		const uint32_t r = request_at(req, pos[i]);
		uint32_t start;
		uint64_t t;
		key[i] = ps_place_key(stage.data() + req[r].base, req[r].n, pos[i] - req[r].base, req[r].stream_id, &start, &t);
		src[i] = req[r].base + start;
		pts[i] = t;
	}
	// scan, totals
	std::vector<uint64_t> scan(m + 1, 0);
	for (uint32_t i = 0; i < m; i++) scan[i + 1] = scan[i] + key[i];
	for (uint32_t r = 0; r < n; r++) {
		PsReqOut &o = out[r];
		if (o.head != PS_NONE) {
			const uint32_t j = jump[levels][o.head];
			if (term_kind[j] == PS_T_LINK) { fprintf(stderr, "chain longer than the doubling\n"); exit(3); }
			o.kind = term_kind[j];
			o.stop = term_stop[j];
		}
		ps_finish(o.kind, o.stop, req[r].n, &o.consumed, &o.in_sync);
		const uint64_t a = scan[o.c0], b = scan[o.c0 + o.count];
		o.total = (uint32_t)(b >> 32) - (uint32_t)(a >> 32);
		o.pes = (uint32_t)b - (uint32_t)a;
		o.pes_first = (uint32_t)a;
	}
	// the host makes room, the gather places the payloads (the stream's ES grows in place here)
	std::vector<uint32_t> pes_offset(m), es_base(n);
	std::vector<uint64_t> pes_pts(m);
	for (uint32_t r = 0; r < n; r++) {
		StreamState &s = st[streams[r]];
		es_base[r] = (uint32_t)s.es.size();
		s.es.resize(s.es.size() + out[r].total);
	}
	for (uint32_t i = 0; i < m; i++) {
		const uint32_t len = (uint32_t)(key[i] >> 32);
		if (!len) continue;
		const uint32_t r = request_at(req, pos[i]);
		const uint32_t off = (uint32_t)(scan[i] >> 32) - (uint32_t)(scan[out[r].c0] >> 32);
		if (key[i] & 1) {
			pes_offset[(uint32_t)scan[i]] = es_base[r] + off;
			pes_pts[(uint32_t)scan[i]] = pts[i];
		}
		std::copy(stage.begin() + src[i], stage.begin() + src[i] + len, st[streams[r]].es.begin() + es_base[r] + off);
	}
	for (uint32_t r = 0; r < n; r++) {
		StreamState &s = st[streams[r]];
		const PsReqOut &o = out[r];
		for (uint32_t k = 0; k < o.pes; k++) s.pes.push_back({pes_offset[o.pes_first + k], pes_pts[o.pes_first + k]});
		std::vector<uint8_t> data = s.leftover;
		data.insert(data.end(), bufs[r].begin(), bufs[r].end());
		s.leftover.assign(data.begin() + o.consumed, data.end());
		s.in_sync = o.in_sync != 0;
		rows.push_back(o.total);
		rows.push_back(o.pes);
		rows.push_back((uint32_t)s.leftover.size());
		rows.push_back(o.in_sync);
		std::vector<uint32_t> items;
		for (uint32_t i = o.c0; i < o.c0 + o.count; i++) {
			const uint32_t p = pos[i] - req[r].base;
			if (marked[i] && ps_item_at(stage.data() + req[r].base, req[r].n, p).kind == PS_ITEM) items.push_back(p);
		}
		rows.push_back((uint32_t)items.size());
		rows.insert(rows.end(), items.begin(), items.end());
	}
}

static uint32_t rd32(FILE *f) {
	uint32_t v;
	if (fread(&v, 4, 1, f) != 1) { fprintf(stderr, "short input\n"); exit(2); }
	return v;
}

int main(int argc, char **argv) {
	if (argc != 3) { fprintf(stderr, "usage: ps_many_check IN OUT\n"); return 2; }
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
		k = s.in_sync ? 1 : 0;
		fwrite(&k, 4, 1, o);
	}
	fclose(o);
	return 0;
}
