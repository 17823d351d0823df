// Host build of the compact record -> raster row conversion of the coefficient export (coef_record_row,
// jsmpeg_b200/csrc/coef_records.h), for tests/test_coefficient_export.py: reads 32-byte compact records (argv[1]) and
// writes each one's 64 raster values (int16, rows 0..7 through coef_record_row) to stdout.
#include <cstdio>

#include "../../jsmpeg_b200/csrc/coef_records.h"

int main(int argc, char **argv) {
	if (argc < 2) return 2;
	FILE *f = fopen(argv[1], "rb");
	if (!f) return 2;
	coef_record_t r;
	while (fread(&r, sizeof r, 1, f) == 1) {
		for (int row = 0; row < 8; row++) {
			int16_t out[8];
			coef_record_row(r, row, out);
			fwrite(out, sizeof out, 1, stdout);
		}
	}
	fclose(f);
	return 0;
}
