/*
 * jsmpeg_b200_napi.c -- N-API addon exposing libjsmpeg_b200.so to Node.js.
 *
 * NOT BUILT OR TESTED IN THIS REPOSITORY'S IMAGE: there is no `node`, no `node_api.h` and no JS
 * engine here or on the GPU boxes (see INTEGRATION.md).  It is the thin shim north_star asks for:
 * every export forwards 1:1 to one of the 15 functions of the reference's native ABI
 * (reference src/wasm/mpeg1.h:10-25) as declared in include/jsmpeg_b200.h -- the same functions
 * the reference's own glue reaches through `module.instance.exports` (src/mpeg1-wasm.js:29-116).
 * Plane memory is handed to JS as EXTERNAL ArrayBuffers over the library's pinned host planes
 * (zero copy, like the `heapU8.subarray` views of src/mpeg1-wasm.js:110-116).
 *
 * Build (where Node headers exist):
 *   gcc -shared -fPIC -I$(node -p "require('node:path').dirname(process.execPath)")/../include/node \
 *       -I../include jsmpeg_b200_napi.c -L../jsmpeg_b200 -ljsmpeg_b200 -Wl,-rpath,'$ORIGIN/../jsmpeg_b200' \
 *       -o jsmpeg_b200.node
 */
#include <node_api.h>
#include <stdint.h>
#include <string.h>

#include "jsmpeg_b200.h"

#define NAPI_OK(call) do { if ((call) != napi_ok) { napi_throw_error(env, NULL, #call " failed"); return NULL; } } while (0)

static mpeg1_decoder_t *decoder_arg(napi_env env, napi_callback_info info, size_t want, napi_value *argv) {
	size_t argc = want;
	void *ptr = NULL;
	if (napi_get_cb_info(env, info, &argc, argv, NULL, NULL) != napi_ok || argc < 1) return NULL;
	if (napi_get_value_external(env, argv[0], &ptr) != napi_ok) return NULL;
	return (mpeg1_decoder_t *)ptr;
}

static napi_value js_create(napi_env env, napi_callback_info info) {
	size_t argc = 2;
	napi_value argv[2], out;
	uint32_t size = 512 * 1024, mode = BIT_BUFFER_MODE_EXPAND;
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	if (argc > 0) napi_get_value_uint32(env, argv[0], &size);
	if (argc > 1) napi_get_value_uint32(env, argv[1], &mode);
	NAPI_OK(napi_create_external(env, mpeg1_decoder_create(size, (bit_buffer_mode_t)mode), NULL, NULL, &out));
	return out;
}

static napi_value js_destroy(napi_env env, napi_callback_info info) {
	napi_value argv[1];
	mpeg1_decoder_t *d = decoder_arg(env, info, 1, argv);
	if (d) mpeg1_decoder_destroy(d);
	return NULL;
}

/* write(decoder, Uint8Array) : get_write_ptr + memcpy + did_write (src/mpeg1-wasm.js:52-70) */
static napi_value js_write(napi_env env, napi_callback_info info) {
	napi_value argv[2], out;
	mpeg1_decoder_t *d = decoder_arg(env, info, 2, argv);
	napi_typedarray_type type;
	size_t length, offset;
	void *data;
	napi_value ab;
	if (!d) return NULL;
	NAPI_OK(napi_get_typedarray_info(env, argv[1], &type, &length, &data, &ab, &offset));
	memcpy(mpeg1_decoder_get_write_ptr(d, (unsigned)length), data, length);
	mpeg1_decoder_did_write(d, (unsigned)length);
	NAPI_OK(napi_create_uint32(env, (uint32_t)length, &out));
	return out;
}

#define INT_GETTER(name, call)                                                   \
	static napi_value name(napi_env env, napi_callback_info info) {              \
		napi_value argv[1], out;                                                 \
		mpeg1_decoder_t *d = decoder_arg(env, info, 1, argv);                    \
		if (!d) return NULL;                                                     \
		NAPI_OK(napi_create_int32(env, (int32_t)(call), &out));                  \
		return out;                                                              \
	}
INT_GETTER(js_get_index, mpeg1_decoder_get_index(d))
INT_GETTER(js_has_sequence_header, mpeg1_decoder_has_sequence_header(d))
INT_GETTER(js_get_coded_size, mpeg1_decoder_get_coded_size(d))
INT_GETTER(js_get_width, mpeg1_decoder_get_width(d))
INT_GETTER(js_get_height, mpeg1_decoder_get_height(d))

static napi_value js_set_index(napi_env env, napi_callback_info info) {
	napi_value argv[2];
	uint32_t index = 0;
	mpeg1_decoder_t *d = decoder_arg(env, info, 2, argv);
	if (!d) return NULL;
	napi_get_value_uint32(env, argv[1], &index);
	mpeg1_decoder_set_index(d, index);
	return NULL;
}

static napi_value js_get_frame_rate(napi_env env, napi_callback_info info) {
	napi_value argv[1], out;
	mpeg1_decoder_t *d = decoder_arg(env, info, 1, argv);
	if (!d) return NULL;
	NAPI_OK(napi_create_double(env, mpeg1_decoder_get_frame_rate(d), &out));
	return out;
}

static napi_value js_decode(napi_env env, napi_callback_info info) {
	napi_value argv[1], out;
	mpeg1_decoder_t *d = decoder_arg(env, info, 1, argv);
	if (!d) return NULL;
	NAPI_OK(napi_get_boolean(env, mpeg1_decoder_decode(d), &out));
	return out;
}

/* Extension (not in the reference, which skips B pictures -- src/mpeg1.js:181-184): setDecodeB(decoder, on)
 * switches the B-picture decode on; lastPictureType(decoder) = picture_coding_type of the picture the last
 * decode() consumed (1 I, 2 P, 3 B), so that a player can put pictures into display order. */
static napi_value js_set_decode_b(napi_env env, napi_callback_info info) {
	napi_value argv[2];
	uint32_t on = 0;
	mpeg1_decoder_t *d = decoder_arg(env, info, 2, argv);
	if (!d) return NULL;
	napi_get_value_uint32(env, argv[1], &on);
	jsmpeg_b200_decoder_set_option(d, "decode_b", (int)on);
	return NULL;
}
static napi_value js_last_picture_type(napi_env env, napi_callback_info info) {
	napi_value argv[1], out;
	int type = 0;
	mpeg1_decoder_t *d = decoder_arg(env, info, 1, argv);
	if (!d) return NULL;
	jsmpeg_b200_decoder_last_picture(d, &type, NULL);
	NAPI_OK(napi_create_int32(env, type, &out));
	return out;
}

/* planes(decoder) -> {y, cr, cb}: zero-copy Uint8Arrays over the pinned host planes of the most
 * recently decoded picture; valid until the next decode() (src/mpeg1-wasm.js:110-118). */
static napi_value plane_view(napi_env env, void *ptr, size_t n) {
	napi_value ab, view;
	if (napi_create_external_arraybuffer(env, ptr, n, NULL, NULL, &ab) != napi_ok) return NULL;
	if (napi_create_typedarray(env, napi_uint8_array, n, ab, 0, &view) != napi_ok) return NULL;
	return view;
}
static napi_value js_planes(napi_env env, napi_callback_info info) {
	napi_value argv[1], out;
	mpeg1_decoder_t *d = decoder_arg(env, info, 1, argv);
	size_t n;
	if (!d) return NULL;
	n = (size_t)mpeg1_decoder_get_coded_size(d);
	NAPI_OK(napi_create_object(env, &out));
	napi_set_named_property(env, out, "y", plane_view(env, mpeg1_decoder_get_y_ptr(d), n));
	napi_set_named_property(env, out, "cr", plane_view(env, mpeg1_decoder_get_cr_ptr(d), n >> 2));
	napi_set_named_property(env, out, "cb", plane_view(env, mpeg1_decoder_get_cb_ptr(d), n >> 2));
	return out;
}

/* Extension: setExportMacroblocks(decoder, on) switches the decoder's "macroblocks" option; macroblocks(decoder) is a
 * zero-copy Uint8Array over the pinned macroblock entries (16 bytes per macroblock, raster order, the layout of
 * jsmpeg_b200_macroblock_t) of the picture the last decode() rendered -- valid until the next decode(), like the
 * planes; undefined before the sequence header. */
static napi_value js_set_export_macroblocks(napi_env env, napi_callback_info info) {
	napi_value argv[2];
	uint32_t on = 0;
	mpeg1_decoder_t *d = decoder_arg(env, info, 2, argv);
	if (!d) return NULL;
	napi_get_value_uint32(env, argv[1], &on);
	jsmpeg_b200_decoder_set_option(d, "macroblocks", (int)on);
	return NULL;
}
/* Extension: setConceal(decoder, on) switches the decoder's "conceal" option: each macroblock a damaged picture lacks
 * gets the co-located samples of the picture it predicts from. */
static napi_value js_set_conceal(napi_env env, napi_callback_info info) {
	napi_value argv[2];
	uint32_t on = 0;
	mpeg1_decoder_t *d = decoder_arg(env, info, 2, argv);
	if (!d) return NULL;
	napi_get_value_uint32(env, argv[1], &on);
	jsmpeg_b200_decoder_set_option(d, "conceal", (int)on);
	return NULL;
}
static napi_value js_macroblocks(napi_env env, napi_callback_info info) {
	napi_value argv[1];
	mpeg1_decoder_t *d = decoder_arg(env, info, 1, argv);
	void *entries;
	size_t n;
	if (!d) return NULL;
	entries = jsmpeg_b200_decoder_get_macroblocks(d);
	if (!entries) return NULL;
	n = (size_t)((mpeg1_decoder_get_width(d) + 15) / 16) * (size_t)((mpeg1_decoder_get_height(d) + 15) / 16) * 16;
	return plane_view(env, entries, n);
}

static napi_value init(napi_env env, napi_value exports) {
	static const struct { const char *name; napi_callback fn; } table[] = {
		{"create", js_create}, {"destroy", js_destroy}, {"write", js_write},
		{"getIndex", js_get_index}, {"setIndex", js_set_index},
		{"hasSequenceHeader", js_has_sequence_header}, {"getFrameRate", js_get_frame_rate},
		{"getCodedSize", js_get_coded_size}, {"getWidth", js_get_width}, {"getHeight", js_get_height},
		{"decode", js_decode}, {"planes", js_planes},
		{"setDecodeB", js_set_decode_b}, {"lastPictureType", js_last_picture_type},
		{"setExportMacroblocks", js_set_export_macroblocks}, {"macroblocks", js_macroblocks},
		{"setConceal", js_set_conceal},
	};
	for (size_t i = 0; i < sizeof(table) / sizeof(table[0]); i++) {
		napi_value fn;
		if (napi_create_function(env, table[i].name, NAPI_AUTO_LENGTH, table[i].fn, NULL, &fn) != napi_ok) return NULL;
		napi_set_named_property(env, exports, table[i].name, fn);
	}
	return exports;
}

NAPI_MODULE(NODE_GYP_MODULE_NAME, init)
