// Host build of the program stream demuxer's per-item arithmetic (jsmpeg_b200/csrc/psdemux.cuh), for
// tests/test_ps_demux.py: reads a buffer (argv[1]) and byte positions (stdin, one per line) and prints, per
// position, "kind len payload_start payload_len has_pts pts" (payload fields 0 unless a PES packet).
#include <cstdio>
#include <vector>

#include "../../jsmpeg_b200/csrc/psdemux.cuh"

int main(int argc, char **argv) {
	if (argc < 2) return 2;
	FILE *f = fopen(argv[1], "rb");
	if (!f) return 2;
	std::vector<uint8_t> buf;
	int c;
	while ((c = fgetc(f)) != EOF) buf.push_back((uint8_t)c);
	fclose(f);
	const uint32_t n = (uint32_t)buf.size();
	unsigned long p;
	while (scanf("%lu", &p) == 1) {
		const PsItem it = ps_item_at(buf.data(), n, (uint32_t)p);
		PsPayload pl{0, 0, 0, 0};
		if (it.kind == PS_ITEM && buf[p + 3] > 0xBB) pl = ps_payload(buf.data() + p, it.len);
		printf("%d %u %u %u %d %llu %d\n", it.kind, it.len, pl.start, pl.len, pl.has_pts, (unsigned long long)pl.pts,
		       ps_is_pack(buf.data(), n, (uint32_t)p) ? 1 : 0);
	}
	return 0;
}
