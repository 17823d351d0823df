// Host build of the record -> public macroblock conversion (jsmpeg_b200/csrc/macroblocks.cuh), for
// tests/test_macroblock_index.py: reads 16-byte mb_record_t records (argv[1]) and a picture_coding_type (argv[2]) and
// writes the 16-byte jsmpeg_b200_macroblock_t entries to stdout.
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../jsmpeg_b200/csrc/macroblocks.cuh"

int main(int argc, char **argv) {
	if (argc < 3) return 2;
	FILE *f = fopen(argv[1], "rb");
	if (!f) return 2;
	const int picture_type = atoi(argv[2]);
	mb_record_t r;
	while (fread(&r, sizeof r, 1, f) == 1) {
		const jsmpeg_b200_macroblock_t m = export_macroblock(r, picture_type);
		fwrite(&m, sizeof m, 1, stdout);
	}
	fclose(f);
	return 0;
}
