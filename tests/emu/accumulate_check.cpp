// Host build of the accumulated map's block code, for tests/test_accumulated_model.py: accumulate_block
// (jsmpeg_b200/csrc/accumulate.cuh), the per-block step of accumulate_kernel, over every block of one picture.
//     accumulate_check FILE   FILE = int32 mb_width, mb_height, has_prev; mb_size records of 16 bytes (mb_record_t);
//                             the residual, int16 [coded_size * 3 / 2]; with has_prev the previous map, int16
//                             [coded_size * 3 / 2][4].  Writes the map, int16 [coded_size * 3 / 2][4].
// Every buffer is allocated at its exact size, so an AddressSanitizer build catches a read or write outside a map.
// Build: g++ -O1 -std=c++17 -I/usr/local/cuda/include.
#define JSMPEG_WALK_EMU 1
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>  // vector types and the host definitions of __device__ / __forceinline__ only

#include "../../jsmpeg_b200/csrc/accumulate.cuh"

int main(int argc, char **argv) {
	if (argc < 2) return 2;
	FILE *f = fopen(argv[1], "rb");
	if (!f) return 2;
	int32_t head[3];
	if (fread(head, sizeof head, 1, f) != 1) return 2;
	const int W = head[0], H = head[1];
	const size_t n = (size_t)W * H * 384;
	std::vector<uint8_t> rec((size_t)W * H * 16);
	std::vector<int16_t> res(n);
	uint2 *prev = head[2] ? new uint2[n] : nullptr;
	uint2 *map = new uint2[n];
	if (fread(rec.data(), 1, rec.size(), f) != rec.size() || fread(res.data(), 2, n, f) != n) return 2;
	if (prev && fread(prev, 8, n, f) != n) return 2;
	fclose(f);
	const int ysize = W * H * 256;
	for (int mb_row = 0; mb_row < H; mb_row++)
		for (int mb_col = 0; mb_col < W; mb_col++)
			for (int b = 0; b < 6; b++) {
				uint2 r;
				memcpy(&r, rec.data() + ((size_t)mb_row * W + mb_col) * 16, 8);
				// the block's residual, as the kernel's transform gives it
				int stride, origin;
				if (b < 4) {
					stride = W * 16;
					origin = (mb_row * 16 + (b >> 1) * 8) * stride + mb_col * 16 + (b & 1) * 8;
				} else {
					stride = W * 8;
					origin = (b == 4 ? ysize + ysize / 4 : ysize) + mb_row * 8 * stride + mb_col * 8;
				}
				int v[64];
				for (int i = 0; i < 64; i++) v[i] = res[origin + (i >> 3) * stride + (i & 7)];
				accumulate_block(r, b, mb_row, mb_col, W, H, v, prev, map);
			}
	fwrite(map, 8, n, stdout);
	delete[] prev;
	delete[] map;
	return 0;
}
