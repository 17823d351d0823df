// Host build of the residual export's block code, for tests/test_residual_export.py: the transform export_residuals_kernel
// and stage 2 run (idct_block, idct_dc: jsmpeg_b200/csrc/idct.cuh) and the compact record scatter the kernel stages its
// rows with (coef_record_scatter: jsmpeg_b200/csrc/coef_records.h).
//     residuals_check idct FILE     FILE = int16 blocks of 64 raster coefficients (not premultiplied); per block
//                                   writes 65 int32: idct_block of its eight 16-byte rows, then idct_dc of value 0
//     residuals_check scatter FILE  FILE = 32-byte compact records; per record writes the 64 int16 of a zeroed raster
//                                   block after coef_record_scatter
// Build: g++ -O1 -std=c++17 -I/usr/local/cuda/include.
#define JSMPEG_WALK_EMU 1
#include <cstdint>
#include <cstdio>
#include <cstring>

#include <cuda_runtime.h>  // vector types and the host definitions of __device__ / __forceinline__ only

static inline int __dp2a_lo(int a, int b, int c) {  // c + a.lo16 * b.byte0 + a.hi16 * b.byte1 (all signed)
	return c + (int)(int16_t)(a & 0xffff) * (int)(int8_t)(b & 0xff) + (int)(int16_t)((uint32_t)a >> 16) * (int)(int8_t)((b >> 8) & 0xff);
}

#include "../../jsmpeg_b200/csrc/coef_records.h"
#include "../../jsmpeg_b200/csrc/idct.cuh"

int main(int argc, char **argv) {
	if (argc < 3) return 2;
	FILE *f = fopen(argv[2], "rb");
	if (!f) return 2;
	if (!strcmp(argv[1], "idct")) {
		int16_t c[64];
		while (fread(c, sizeof c, 1, f) == 1) {
			uint4 q[8];
			memcpy(q, c, sizeof q);
			int v[65];
			idct_block(q, reinterpret_cast<int(&)[64]>(v));
			v[64] = idct_dc(c[0]);
			fwrite(v, sizeof v, 1, stdout);
		}
	} else if (!strcmp(argv[1], "scatter")) {
		coef_record_t r;
		while (fread(&r, sizeof r, 1, f) == 1) {
			int16_t raster[64] = {0};
			coef_record_scatter(r, raster);
			fwrite(raster, sizeof raster, 1, stdout);
		}
	} else {
		return 2;
	}
	fclose(f);
	return 0;
}
