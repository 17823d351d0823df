/*
 * jsmpeg_b200.h -- C ABI of libjsmpeg_b200.so: an H100 (sm_90a CUDA) implementation of jsmpeg's
 * MPEG-1 video decode path.  Plain pointers and sizes only.
 *
 * Part 1 is EXACTLY the ABI the reference's own native plugin boundary binds -- the 15 functions
 * its WASM build exports (reference src/wasm/mpeg1.h:10-25, export list build.sh:53-67) and its
 * JS glue calls (src/mpeg1-wasm.js:29, 36, 43, 50, 62-69, 75-88, 103-108).  A reference-side
 * binding that loads this library instead of the WASM module gets the same behaviour:
 * same call protocol, same return values, same bit-index semantics, bit-identical planes.
 *
 * Part 2 is our batch extension (not in the reference): N independent streams on one GPU,
 * device-resident planes, one call decodes the next pictures of every stream.
 */
#ifndef JSMPEG_B200_H
#define JSMPEG_B200_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------ */
/* Part 1: the reference ABI (src/wasm/mpeg1.h:10-25)                                          */

typedef struct mpeg1_decoder_t mpeg1_decoder_t;

/* src/wasm/buffer.h:8-11 */
typedef enum {
	BIT_BUFFER_MODE_EVICT = 1,
	BIT_BUFFER_MODE_EXPAND = 2
} bit_buffer_mode_t;

/* mpeg1.h:12 / mpeg1.c:777-782.  Never fails and never takes the process down: without a usable
 * CUDA device (or after any CUDA error later on) the decoder is DEAD -- decode() returns false like
 * "no sequence header yet", writes are swallowed, jsmpeg_b200_decoder_last_error says why (the
 * reason is also printed to stderr once).  Uses the CUDA device set with
 * jsmpeg_b200_set_default_device, else the one named by the environment variable
 * JSMPEG_B200_DEVICE, else device 0. */
mpeg1_decoder_t *mpeg1_decoder_create(unsigned int buffer_size, bit_buffer_mode_t buffer_mode);
/* mpeg1.h:13 / mpeg1.c:784-798 */
void mpeg1_decoder_destroy(mpeg1_decoder_t *self);
/* mpeg1.h:14 / mpeg1.c:800-802, buffer.c:48-65: room for byte_size more bytes (EXPAND: grows;
 * EVICT: discards consumed bytes, buffer.c:167-190); the pointer is HOST memory (pinned) and ALWAYS
 * covers byte_size bytes -- where the reference's own sizing (buffer.c:53-57) would not, the buffer
 * grows to length + byte_size (csrc/bitbuffer.h). */
void *mpeg1_decoder_get_write_ptr(mpeg1_decoder_t *self, unsigned int byte_size);
/* mpeg1.h:15-16 / mpeg1.c:804-810: read position in BITS */
int mpeg1_decoder_get_index(mpeg1_decoder_t *self);
void mpeg1_decoder_set_index(mpeg1_decoder_t *self, unsigned int index);
/* mpeg1.h:17 / mpeg1.c:812-819: commits the bytes; parses the first sequence header */
void mpeg1_decoder_did_write(mpeg1_decoder_t *self, unsigned int byte_size);

/* mpeg1.h:19-23 / mpeg1.c:821-839 */
int mpeg1_decoder_has_sequence_header(mpeg1_decoder_t *self);
float mpeg1_decoder_get_frame_rate(mpeg1_decoder_t *self);
int mpeg1_decoder_get_coded_size(mpeg1_decoder_t *self);
int mpeg1_decoder_get_width(mpeg1_decoder_t *self);
int mpeg1_decoder_get_height(mpeg1_decoder_t *self);
/* mpeg1.h:24-26 / mpeg1.c:841-851: planes of the most recently decoded picture, HOST-visible
 * (pinned), coded size (stride = coded width, coded width / 2); borrowed until the next decode. */
void *mpeg1_decoder_get_y_ptr(mpeg1_decoder_t *self);
void *mpeg1_decoder_get_cr_ptr(mpeg1_decoder_t *self);
void *mpeg1_decoder_get_cb_ptr(mpeg1_decoder_t *self);
/* mpeg1.h:27 / mpeg1.c:853-864: false = no sequence header yet or no picture start code in the
 * buffer; true otherwise (also for skipped B/D pictures).  Synchronous: the planes are complete
 * and host-visible when it returns. */
bool mpeg1_decoder_decode(mpeg1_decoder_t *self);

/* ------------------------------------------------------------------------------------------ */
/* Part 2: batch extension                                                                      */

typedef struct jsmpeg_b200_batch_t jsmpeg_b200_batch_t;

#define JSMPEG_B200_OUT_DEVICE 0 /* planes stay in HBM (jsmpeg_b200_batch_get_planes)           */
#define JSMPEG_B200_OUT_HOST   1 /* every decoded picture is also copied to pinned host memory  */
#define JSMPEG_B200_OUT_RGBA   2 /* run the fused planar->RGBA epilogue (canvas2d.js:53-122)    */
#define JSMPEG_B200_OUT_MACROBLOCKS 4 /* every reconstructed picture's macroblock entries beside its planes
                                       * (jsmpeg_b200_batch_get_macroblocks, below decode_macroblocks)  */
#define JSMPEG_B200_OUT_ACCUMULATED (1 << 3) /* = 8: every reconstructed I/P picture's accumulated map beside its planes
                                       * (jsmpeg_b200_batch_get_accumulated, below decode_accumulated) */
#define JSMPEG_B200_OUT_RESIDUALS (0x10) /* = 16 = bit 4: the residual of the picture get_planes gives
                                       * (jsmpeg_b200_batch_get_residuals, below the accumulated maps) */

typedef struct jsmpeg_b200_stats_t {
	uint64_t pictures;            /* decode() == true count                                     */
	uint64_t pictures_decoded;    /* I/P pictures reconstructed                                 */
	uint64_t coded_blocks;
	uint64_t macroblocks;         /* macroblocks written by stage 2                             */
	uint64_t algorithmic_bytes;   /* stage-2 bytes: records + planes written + planes referenced */
	uint64_t es_bytes;            /* bitstream bytes consumed by stage 1                        */
	uint64_t h2d_bytes, d2h_bytes;
	uint64_t kernel_launches;     /* scan + parse + reconstruct (+ rgba, + macroblock export, + accumulate) launches;
	                               * OUT_RESIDUALS adds none, but a step's reconstruct kernel with a residual task is
	                               * cut into launches of its RES variant's capacity (72 plain, 56 RGBA, 63 B, 51 B + RGBA
	                               * tasks, against 80, 60, 64, 48): a step with more tasks of one kernel than the
	                               * smaller of the two may take a different number of launches */
	uint64_t recon_launches;
	double parse_ms, recon_ms, scan_ms; /* CUDA-event device time on the launching stream       */
	uint64_t parse_errors;        /* pictures whose slice walk hit an invalid code              */
	double walk_ms;               /* part of parse_ms spent in the walk kernel (1a)             */
	uint64_t lane_walk_pictures;  /* pictures walked by the lane-parallel walk (JSMPEG_B200_WALK=lanes), not its serial fall-back */
} jsmpeg_b200_stats_t;

/* n_streams decoders on CUDA device `device`.  max_slots bounds the pictures parsed ahead
 * (records resident in HBM; cut to what the device can hold); 0 = choose from free memory.
 * Never NULL; a batch without a usable device is dead (see jsmpeg_b200_batch_last_error). */
jsmpeg_b200_batch_t *jsmpeg_b200_batch_create(int n_streams, int device, unsigned int max_slots);
void jsmpeg_b200_batch_destroy(jsmpeg_b200_batch_t *b);
/* NULL while the batch works; otherwise the first failure (a CUDA error text).  A dead batch returns
 * 0 / -1 / false from every call and never touches the device again. */
const char *jsmpeg_b200_batch_last_error(jsmpeg_b200_batch_t *b);
/* Tuning knobs, 0 on success, -1 for an unknown name.  "lookahead": pictures parsed ahead per stream
 * beyond the ones a decode call asks for.
 * "slice_walk" (default 0, or JSMPEG_B200_SLICE_WALK): I/P pictures with at least four slices are parsed by a
 * walk kernel that gives every slice a lane of its own instead of cutting one slice's bits into 32 (streams with a
 * slice per macroblock row); the results are the same bit for bit, only the speed differs.
 * "decode_b" (default 0, or the environment variable JSMPEG_B200_DECODE_B; also honoured by decoders made with
 * mpeg1_decoder_create): the B-PICTURE EXTENSION.  The reference skips B pictures (src/mpeg1.js:181-184:
 * decode() returns true, nothing is rendered) and so does this library by default.  With 1, a B picture is
 * decoded after ISO/IEC 11172-2 from the two most recent I/P pictures; decode() still consumes pictures in
 * CODED order, the planes of a B picture are what get_planes / get_host_planes / the reference ABI's
 * get_{y,cr,cb}_ptr return after it, and jsmpeg_b200_batch_last_picture tells type and temporal_reference so
 * that a player can put pictures into display order.  No reference implementation exists for this part.
 * "conceal" (default 0): ERROR CONCEALMENT.  When a picture's walk stops at an invalid code, or a slice is lost, the
 * macroblocks it did not reach are not decoded; by default (like the reference) they keep whatever their plane set
 * held, which is the picture two references back (for a B picture: the B picture two B pictures back).  With 1,
 * before a picture is reconstructed every macroblock whose record is not PRESENT gets the co-located samples of the
 * picture's forward reference -- 16x16 luma and 8x8 Cr and Cb, zero motion, a plain copy: for an I or P picture the
 * stream's newest I/P picture before it (for an I picture, what a P picture in its place would predict from), for a
 * B picture its forward (past) reference.  A PRESENT macroblock, even one whose walk stopped inside a block, is not
 * touched.  What follows from the planes follows the concealed content: get_planes, the host ring, RGBA, frames of
 * decode_frames*, decode_pictures and seek_pictures, and every picture predicted from it later.  A picture of
 * decode_pictures / decode_intra that is its own chain has no forward reference (a zeroed set), so its absent
 * macroblocks stay 0 either way.  The records define the exports, so these do NOT change: macroblock entries
 * (OUT_MACROBLOCKS, decode_macroblocks), coefficients, residuals (0 for an absent macroblock) and accumulated maps
 * (absent samples stay untraced).  A picture whose walk met no invalid code, counted the picture's macroblocks and
 * whose slices never go back to an earlier row adds no work; for the others one copy launch per reconstruct step runs
 * before it (counted in kernel_launches).  Records do not
 * depend on the option: it takes effect from the next reconstruct step.  jsmpeg_b200_decoder_set_option forwards it. */
int jsmpeg_b200_batch_set_option(jsmpeg_b200_batch_t *b, const char *name, int value);

/* per-stream twins of the reference ABI */
void *jsmpeg_b200_batch_get_write_ptr(jsmpeg_b200_batch_t *b, int stream, unsigned int byte_size);
void jsmpeg_b200_batch_did_write(jsmpeg_b200_batch_t *b, int stream, unsigned int byte_size);
int jsmpeg_b200_batch_get_index(jsmpeg_b200_batch_t *b, int stream);
void jsmpeg_b200_batch_set_index(jsmpeg_b200_batch_t *b, int stream, unsigned int index);
/* returns has_sequence_header */
int jsmpeg_b200_batch_stream_info(jsmpeg_b200_batch_t *b, int stream, int *width, int *height,
                                  int *coded_size, float *frame_rate);

/* MPEG-TS in, demultiplexed on the GPU (mirror of the reference's host demuxer src/ts.js for a
 * buffer of whole 188-byte packets): the payload of every PES packet with stream id `stream_id`
 * (0xE0 = first video stream, ts.js:213-224) is appended to `stream` exactly as if it had been
 * written with get_write_ptr/did_write.  The buffer need not hold whole packets nor begin on a packet
 * boundary: what a call leaves over is kept for the next one (ts.js:25-41) and a lost sync byte is
 * searched for like the reference does (ts.js:155-189); a PID that a later PES header binds to
 * another stream id stops feeding this stream (ts.js:81-83).  Returns the number of
 * elementary-stream bytes appended (-1: the decoder is dead).  pts_out / offset_out (capacity n_max,
 * may be NULL) receive, per PES packet in stream order (the first n_max of them; *n_pes counts all), its PTS in 90 kHz ticks (0 if absent) and the byte offset of its
 * payload in the stream's buffer -- the table Decoder.Base.write keeps (src/decoder.js:36-47). */
long jsmpeg_b200_batch_write_ts(jsmpeg_b200_batch_t *b, int stream, const uint8_t *ts, size_t n_bytes, int stream_id,
                                uint64_t *pts_out, uint32_t *offset_out, int n_max, int *n_pes);

/* MPEG-TS of many streams in one call (live ingest: a chunk from each of many sources per tick).  Request i does
 * exactly what jsmpeg_b200_batch_write_ts(b, streams[i], ts[i], n_bytes[i], stream_ids ? stream_ids[i] : 0xE0, ...)
 * does: the same elementary-stream bytes appended, the same PES table, the same bytes left over for the stream's
 * next TS write and the same PID bindings carried on, for any interleaving of write_ts and write_ts_many calls.
 * All requests are demultiplexed in one pass on the GPU; the call's kernel launches and host synchronisations do
 * not grow with n.  A stream may be named at most once per call.  Two requests may pass the same buffer (a
 * multiplex of several video programs, each to its own stream by its stream id).  Streams not named are not touched.
 *   appended_out[i] (may be NULL): ES bytes appended to streams[i] (write_ts's return value).
 *   n_pes_out[i]    (may be NULL): PES starts of request i (write_ts's *n_pes), counted even where dropped below.
 *   pts_out / offset_out (each may be NULL; n_max entries for the whole call): request 0's PES starts in stream
 *   order, then request 1's, ...; 90 kHz PTS (0 if absent) and payload offset in the stream's buffer, as write_ts;
 *   entries beyond n_max are dropped.
 * Synchronous.  Returns the ES bytes appended over all requests; -1 dead; -2 a request is invalid (n < 0; streams,
 * ts or n_bytes NULL with n > 0; a stream out of range or named twice; ts[i] NULL with n_bytes[i] > 0; the call's
 * input plus the named streams' left-over bytes 4 GiB - 4 KiB or more) -- checked before any work, and then
 * nothing changed. */
long jsmpeg_b200_batch_write_ts_many(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint8_t *const *ts,
                                     const size_t *n_bytes, const int *stream_ids, long *appended_out,
                                     uint64_t *pts_out, uint32_t *offset_out, long n_max, int32_t *n_pes_out);

/* MPEG program stream in (ISO 11172-1 system stream, .mpg / VCD .dat; ISO 13818-1 program stream, .vob),
 * demultiplexed on the GPU: the payload of every PES packet with stream id `stream_id` (0xE0..0xEF) is
 * appended to `stream` exactly as if it had been written with get_write_ptr/did_write.  The stream is
 * read as a chain of items without gaps -- pack headers of either form, end codes, and packets of
 * 6 + packet_length bytes (system header, PSM, PES) -- starting at the first valid pack header.  Bytes
 * that are not an item where one should start are a break: parsing resumes at the next valid pack
 * header.  The buffer may be cut anywhere: what a call leaves over is kept for the next one, and the
 * result does not depend on how the bytes are split into calls.  Returns the number of
 * elementary-stream bytes appended (-1: the decoder is dead; -2: stream_id is not 0xE0..0xEF, nothing
 * changed).  pts_out / offset_out (capacity n_max, may be NULL) receive, per PES packet of the stream
 * with a PTS and a non-empty payload, in stream order, its 33-bit PTS in 90 kHz ticks and the byte
 * offset of its payload in the stream's buffer; *n_pes = their number. */
long jsmpeg_b200_batch_write_ps(jsmpeg_b200_batch_t *b, int stream, const uint8_t *ps, size_t n_bytes, int stream_id,
                                uint64_t *pts_out, uint32_t *offset_out, int n_max, int *n_pes);

/* MPEG program streams of many streams in one call (a server or data loader reading a chunk of each of many .mpg /
 * .vob files per tick).  Request i does exactly what jsmpeg_b200_batch_write_ps(b, streams[i], ps[i], n_bytes[i],
 * stream_ids ? stream_ids[i] : 0xE0, ...) does: the same elementary-stream bytes appended, the same PES table, the
 * same bytes left over and the same in-sync state carried to the stream's next PS write, for any interleaving of
 * write_ps and write_ps_many calls.  All requests are demultiplexed in one pass on the GPU; the call's kernel
 * launches and host synchronisations grow neither with n nor with the breaks in the input.  A stream may be named at
 * most once per call.  Two requests may pass the same buffer (the 0xE0 and 0xE1 video streams of one .vob, each to
 * its own stream).  Streams not named are not touched.
 *   appended_out[i] (may be NULL): ES bytes appended to streams[i] (write_ps's return value).
 *   n_pes_out[i]    (may be NULL): PES table entries of request i (write_ps's *n_pes), counted even where dropped below.
 *   pts_out / offset_out (each may be NULL; n_max entries for the whole call): request 0's entries in stream order,
 *   then request 1's, ...; 33-bit PTS in 90 kHz ticks and payload offset in the stream's buffer, as write_ps;
 *   entries beyond n_max are dropped.
 * Synchronous.  Returns the ES bytes appended over all requests; -1 dead; -2 a request is invalid (n < 0; streams,
 * ps or n_bytes NULL with n > 0; a stream out of range or named twice; ps[i] NULL with n_bytes[i] > 0; a stream id
 * outside 0xE0..0xEF; the call's input plus the named streams' left-over bytes 4 GiB - 4 KiB or more, each request
 * rounded up to 16 bytes) -- checked before any work, and then nothing changed. */
long jsmpeg_b200_batch_write_ps_many(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint8_t *const *ps,
                                     const size_t *n_bytes, const int *stream_ids, long *appended_out,
                                     uint64_t *pts_out, uint32_t *offset_out, long n_max, int32_t *n_pes_out);

/* Make everything written so far resident in HBM and indexed (H2D copy of new bytes + start-code
 * scan).  Called implicitly by decode; exposed so that a benchmark can separate it.  Returns the
 * number of picture start codes currently indexed over all streams. */
long jsmpeg_b200_batch_upload(jsmpeg_b200_batch_t *b);
/* Forget the start-code index and all parsed-ahead records, and rewind every stream to bit 0
 * (the elementary streams stay resident in HBM). */
void jsmpeg_b200_batch_rewind(jsmpeg_b200_batch_t *b);

/* Empty every stream's bit buffer (length = index = 0, planes zeroed) but keep its sequence
 * parameters and all allocations: the state of a decoder that has seen the sequence header and
 * nothing else.  The next write + decode pays the full host->device path again. */
void jsmpeg_b200_batch_reset(jsmpeg_b200_batch_t *b);

/* Equivalent to n_pictures consecutive decode() calls on every stream (streams that run out of
 * pictures simply stop).  Returns the number of decode() calls that returned true. */
long jsmpeg_b200_batch_decode(jsmpeg_b200_batch_t *b, int n_pictures, int flags);

/* Device pointers (HBM) of the most recently decoded picture of a stream; 0 on success. */
int jsmpeg_b200_batch_get_planes(jsmpeg_b200_batch_t *b, int stream, void **y, void **cr, void **cb);
/* Host pointers (pinned) of the most recent picture copied out with JSMPEG_B200_OUT_HOST. */
int jsmpeg_b200_batch_get_host_planes(jsmpeg_b200_batch_t *b, int stream, void **y, void **cr, void **cb);
/* RGBA8888 picture (display size, device memory) of the most recent JSMPEG_B200_OUT_RGBA decode */
int jsmpeg_b200_batch_get_rgba(jsmpeg_b200_batch_t *b, int stream, void **rgba);
/* Synchronous copy of that RGBA picture into caller memory (width * height * 4 bytes). */
int jsmpeg_b200_batch_read_rgba(jsmpeg_b200_batch_t *b, int stream, void *rgba);
/* Synchronous copy of the most recent picture's planes into caller memory (coded size). */
int jsmpeg_b200_batch_read_planes(jsmpeg_b200_batch_t *b, int stream, void *y, void *cr, void *cb);

/* picture_coding_type (1 I, 2 P, 3 B, 4 D) and temporal_reference (ISO 11172-2 2.4.2.5) of the picture the
 * stream's last decode() consumed, decoded or skipped; -1 before the first one.  Either pointer may be NULL. */
int jsmpeg_b200_batch_last_picture(jsmpeg_b200_batch_t *b, int stream, int *picture_type, int *temporal_reference);

/* KEY PICTURES (thumbnails, seek previews, frame sampling): I pictures decoded independently of decode(), any number
 * of them from any streams in one parallel wave.  Picture k of a stream is the k-th picture start code (00 00 01 00)
 * in its current buffer (for a buffer that never evicted: the picture the (k+1)-th decode() consumes).  The index
 * lists picture k when it starts after the stream's first sequence header, its picture_coding_type is 1, and it is
 * closed: a later start code is in the buffer that is no slice (01..AF), user data (B2) or extension (B5).  A
 * listed picture decodes to exactly what a fresh decoder gives for the first sequence header + the picture's bytes
 * up to and including that closing code: where the picture codes every macroblock, what decode() gives at that
 * point of the stream; a macroblock the picture does not reach is 0 (RGBA: the conversion of those planes, the
 * odd edge opaque white).  Neither call changes anything decode() observes (bit index, planes, last_picture,
 * stats -- both make written bytes resident first, and count that upload as decode() would have); decode_intra may
 * drop parsed-ahead pictures when it needs their record slots (decode() then parses them again). */

/* I pictures of `stream` that decode_intra can decode now; returns how many there are (-1 dead, -2 stream out of
 * range); the first min(count, n_max) go to the arrays, any of which may be NULL. */
long jsmpeg_b200_batch_intra_index(jsmpeg_b200_batch_t *b, int stream, uint32_t *picture_out,
                                   uint32_t *byte_pos_out, int32_t *temporal_reference_out, long n_max);
/* Decode n listed I pictures, of any streams, in as few waves as the record slots allow.  Request i =
 * picture pictures[i] of stream streams[i] into planes_dst[i]: DEVICE memory of coded_size * 3 / 2 bytes
 * (Y | Cr | Cb, coded size, like get_planes), 16-byte aligned.  With JSMPEG_B200_OUT_RGBA in flags, rgba_dst[i]
 * (device, 16-byte aligned, width * height * 4) gets the picture too.  Synchronous: everything is written when it
 * returns.  n_present_out / error_out (may be NULL) get picture_info_t.n_present / .error per request.  Returns n;
 * -1 dead; -2 a request is invalid (stream out of range or without sequence header, picture not in the
 * intra index, NULL or misaligned destination) -- checked before any work, and then nothing changed. */
long jsmpeg_b200_batch_decode_intra(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                    void *const *planes_dst, void *const *rgba_dst, int flags,
                                    int32_t *n_present_out, int32_t *error_out);

/* RANDOM ACCESS (seek, frame sampling): any picture decode() would reconstruct, decoded from its chain start,
 * independently of decode(), many short chains side by side.  The index lists picture k (numbered as above) when it
 * starts after the first sequence header, is closed (as above), is one decode() reconstructs -- an I picture, a P
 * picture with forward_f_code != 0, and while the "decode_b" option is on a B picture with both f_codes != 0 -- and
 * has a chain start: the greatest picture j <= k of the intra index such that at least r pictures of [j, k) are
 * references (I, or P with forward_f_code != 0), r = 0 for I, 1 for P, 2 for B.  (So j = k for an I picture, the
 * last I picture before it for a P picture, one GOP further back for a B picture of an open GOP.)  A listed picture
 * decodes to exactly what get_planes gives after the decode() that consumes it, in a fresh decoder (every plane set
 * zeroed, the batch's current decode_b) fed the first sequence header + the bytes from picture j up to and including
 * picture k's closing code.  Where every picture from j through k codes every macroblock, that is what decode()
 * gives at that point of the stream.  (Damaged input: a walk that runs across a closing code reads the stream's
 * bytes behind it, as decode() does -- DESIGN 3.7.)  Neither call changes anything decode() observes, as above. */

/* Pictures of `stream` that decode_pictures can decode now; returns how many there are (-1 dead, -2 stream out of
 * range); the first min(count, n_max) go to the arrays (picture_coding_type to type_out), any of which may be NULL. */
long jsmpeg_b200_batch_picture_index(jsmpeg_b200_batch_t *b, int stream, uint32_t *picture_out,
                                     uint32_t *byte_pos_out, int32_t *type_out, int32_t *temporal_reference_out,
                                     uint32_t *chain_start_out, long n_max);
/* Decode n listed pictures, of any streams; destinations, flags, synchronism and the -2 rule as decode_intra, the
 * requests checked against the picture index.  status_out[i] (may be NULL) is PIC_DECODED, or 0 when the fresh
 * decoder never consumes picture k (a damaged earlier picture's walk ran across its start code): its planes are
 * then 0, its RGBA opaque white, its n_present / error 0.  Duplicate requests each get the picture. */
long jsmpeg_b200_batch_decode_pictures(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                       void *const *planes_dst, void *const *rgba_dst, int flags,
                                       int32_t *status_out, int32_t *n_present_out, int32_t *error_out);

/* MACROBLOCK DATA (motion detection, shot-cut cues, compressed-domain analytics): each macroblock's coding mode and
 * motion vectors of chosen pictures of any streams, read by the picture walks alone -- no coefficients, no pixels, no
 * reference pictures, so every request of a call is one wave.  One entry per macroblock, raster order (= macroblock
 * address), mb_height * mb_width entries per picture. */
typedef struct jsmpeg_b200_macroblock_t {
	int16_t fwd_x, fwd_y;  /* forward vector, luma half-pel units as used for prediction (full_pel already doubled) */
	int16_t bwd_x, bwd_y;  /* backward vector (B pictures), same units */
	uint8_t flags;         /* JSMPEG_B200_MB_* */
	uint8_t cbp;           /* bit (5 - block) set <=> block coded; blocks 0-3 luma, 4 Cb, 5 Cr */
	uint8_t qscale;        /* quantiser_scale in force */
	uint8_t reserved[5];   /* 0 */
} jsmpeg_b200_macroblock_t;   /* 16 bytes */
#define JSMPEG_B200_MB_PRESENT  0x01  /* decoded (coded or skipped); all other fields are 0 when clear */
#define JSMPEG_B200_MB_INTRA    0x02
#define JSMPEG_B200_MB_SKIPPED  0x04  /* made by a macroblock-address increment > 1 */
#define JSMPEG_B200_MB_BACKWARD 0x08  /* predicted from the backward reference (bwd_*) */
#define JSMPEG_B200_MB_FORWARD  0x10  /* predicted from the forward reference (fwd_*) */
/* FORWARD is set on every present non-intra macroblock of an I or P picture (skipped ones and P macroblocks without
 * motion predict from the forward picture with the zero vector); in a B picture the two direction flags say which
 * references a non-intra macroblock is predicted from (both: their average).  A vector whose flag is clear is 0.
 * Chroma vectors follow from the luma vector and are not exported. */

/* Pictures of `stream` that decode_macroblocks can describe now; returns how many there are (-1 dead, -2 stream out
 * of range); the first min(count, n_max) go to the arrays, any of which may be NULL.  Picture k (numbered as above) is
 * listed when it starts after the first sequence header, is closed (as above), and is one the walks decode: an I
 * picture, a P picture with forward_f_code != 0, or a B picture with both f_codes != 0 -- B pictures whatever the
 * "decode_b" option says, and with no chain start needed (a B picture's macroblock layer depends on its own bits). */
long jsmpeg_b200_batch_macroblock_index(jsmpeg_b200_batch_t *b, int stream, uint32_t *picture_out,
                                        uint32_t *byte_pos_out, int32_t *type_out, int32_t *temporal_reference_out,
                                        long n_max);
/* Describe n listed pictures, of any streams.  Request i = picture pictures[i] of stream streams[i] into mb_dst[i]:
 * DEVICE memory of mb_height * mb_width jsmpeg_b200_macroblock_t, 16-byte aligned.  Each picture is what the walk
 * gives when it starts at the picture's own start code: for a clean stream, what a fresh decoder (B pictures on) gives
 * for the first sequence header + the picture + its closing code, and the macroblocks decode() uses for picture k
 * whenever it consumes it.  Synchronous; duplicates each get the entries.  n_present_out / error_out (may be NULL) get
 * picture_info_t.n_present / .error per request.  Returns n; -1 dead; -2 a request is invalid (stream out of range or
 * without sequence header, picture not in the macroblock index, NULL or misaligned destination) -- checked before any
 * work, and then nothing changed.  Changes nothing decode() observes, as decode_intra. */
long jsmpeg_b200_batch_decode_macroblocks(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                          void *const *mb_dst, int32_t *n_present_out, int32_t *error_out);

/* MACROBLOCK DATA OF THE PLAYBACK PATH (live analytics on the pictures decode() plays: motion detection, intra share as
 * a shot-cut cue, motion overlays): with JSMPEG_B200_OUT_MACROBLOCKS in the flags of jsmpeg_b200_batch_decode or
 * jsmpeg_b200_batch_seek_pictures (combined freely with OUT_HOST / OUT_RGBA), every picture the call reconstructs gets
 * its macroblock entries beside its planes, from the walk decode() reconstructs it from: no second walk.
 *
 * A stream's ENTRIES are mb_height * mb_width jsmpeg_b200_macroblock_t in raster order, in the layout and conversion of
 * decode_macroblocks.  After a call with the flag they are the entries of the picture get_planes gives, whenever a call
 * with the flag reconstructed that picture; for a picture decode() reconstructs (PIC_DECODED: I and P pictures, B
 * pictures under decode_b) they equal byte for byte what decode_macroblocks writes for the same picture k -- on damaged
 * streams too, both reading the records of the walk that starts at k's start code.  A call that reconstructs nothing
 * for a stream leaves its entries as they were, like its planes.  A call WITHOUT the flag writes no entries: after it
 * the entries may describe an older picture than the planes.  Entries not yet written by a call with the flag are 0,
 * and again after jsmpeg_b200_batch_reset.  seek_pictures with the flag: the entries of the picture the stream's state
 * ends on (picture k, or under status 0 the picture the fresh decoder ended on; 0 where that decoder reconstructed
 * nothing).
 *
 * Each returns 0, or non-zero for a dead batch, a stream out of range or one without a sequence header. */
/* Device pointer to the entries; valid until the next decode / seek, like get_planes. */
int jsmpeg_b200_batch_get_macroblocks(jsmpeg_b200_batch_t *b, int stream, void **entries);
/* Synchronous copy of the entries into caller memory (mb_height * mb_width * 16 bytes), like read_planes. */
int jsmpeg_b200_batch_read_macroblocks(jsmpeg_b200_batch_t *b, int stream, void *dst);
/* Host pointer (pinned) to the entries of the picture get_host_planes gives: under OUT_HOST | OUT_MACROBLOCKS every
 * reconstructed picture's entries go to the slot of the host ring that receives its planes, so the planes and entries of
 * one slot always belong together. */
int jsmpeg_b200_batch_get_host_macroblocks(jsmpeg_b200_batch_t *b, int stream, void **entries);

/* COEFFICIENTS (DC images for shot-boundary detection and thumbnails, residual-energy and texture features,
 * DCT-domain learning): each block's 64 dequantised DCT coefficients of chosen pictures of any streams, as the
 * inverse transform consumes them -- no pixels and no reference pictures, so every request of a call is one wave of
 * the walks and the coefficient expansion.  The pictures are those of the macroblock index above, for the same reason
 * (a picture's coefficients depend on its own bits only: the intra DC predictors reset at every slice).
 *
 * Request i = picture pictures[i] of stream streams[i] into coef_dst[i]: DEVICE memory, 16-byte aligned, of
 * mb_height * mb_width * 6 * 64 int16 (768 bytes per macroblock): macroblocks in raster order; per macroblock the
 * blocks 0-3 luma (top-left, top-right, bottom-left, bottom-right), 4 Cb, 5 Cr (the cbp bits' order); per block the
 * 64 values in RASTER (de-zig-zagged) order, row-major 8 x 8.  Each value is dequantised, made odd toward zero and
 * clipped to [-2048, 2047], the intra DC as sat16(8 * dc) (8 * dc saturated to int16: exact while |dc| <= 4095, which
 * a conforming stream never leaves; the planes use the exact DC): ISO 11172-2's dct_recon, with ONE deviation, kept because these
 * are the values the pictures' samples are made from: the product level * quantiser_scale * Q is shifted right
 * arithmetically by 4, so a negative product is rounded toward minus infinity where ISO truncates toward zero.
 * Every value of a block whose cbp bit is clear, and of a macroblock without PRESENT, is 0: every byte of
 * coef_dst[i] is written.  mb_dst may be NULL; otherwise mb_dst[i] (16-byte aligned) gets exactly what
 * decode_macroblocks writes for the request, from the same walk.
 *
 * Each picture is what the walk and the expansion give when they start at the picture's own start code: for a clean
 * stream, what a fresh decoder (B pictures on) gives for the first sequence header + the picture + its closing code,
 * and the coefficients decode() uses for picture k.  A damaged picture: the walk reads the resident stream past the
 * closing code (as decode_intra).  Where it stops inside a macroblock header the macroblock is absent (all 0); where
 * it stops inside a block the macroblock is PRESENT with the cbp bits of the blocks it finished -- the block whose
 * codes it could not read, and those after it, have their bit clear and are 0 (not the values read before the bad
 * code) -- and every finished block holds the values of its codes.
 *
 * Synchronous; duplicates each get the data.  n_present_out / error_out (may be NULL) as decode_macroblocks.  Returns
 * n; -1 dead; -2 a request is invalid (stream out of range or without sequence header, picture not in the macroblock
 * index, NULL or misaligned coef_dst[i], misaligned or NULL mb_dst[i] when mb_dst is given) -- checked before any
 * work, and then nothing changed.  Changes nothing decode() observes, as decode_intra. */
long jsmpeg_b200_batch_decode_coefficients(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                           void *const *coef_dst, void *const *mb_dst,
                                           int32_t *n_present_out, int32_t *error_out);

/* RESIDUALS (compressed-domain video models -- I frames, motion vectors and residuals -- residual-energy motion and
 * saliency cues): the pixel-domain residual of chosen pictures of any streams, the inverse transform of every coded
 * block -- what stage 2 adds to the motion-compensated prediction (or, for an intra macroblock, clamps) -- with no
 * reference pictures, so every request of a call is one wave of the walks, the coefficient expansion and one
 * transform-and-store kernel.  The pictures are those of the macroblock index, as for decode_coefficients.
 *
 * Request i = picture pictures[i] of stream streams[i] into res_dst[i]: DEVICE memory, 16-byte aligned, of
 * coded_size * 3 / 2 int16 (coded_size * 3 bytes) in the planes' layout, in samples: Y at 0 (coded_height x
 * coded_width), Cr at coded_size, Cb at coded_size * 5 / 4 (each coded_height / 2 x coded_width / 2) -- the order and
 * offsets of get_planes and of decode_pictures' planes_dst, so residual and picture line up sample for sample.
 * Every 8 x 8 block is the reference's integer IDCT (src/mpeg1.js:916-983, with PREMULTIPLIER_MATRIX) of the block
 * decode_coefficients writes for the same request, before any add or clamp: 0 where the cbp bit is clear or the
 * macroblock is not PRESENT (every byte of res_dst[i] is written), (c0 * 32 + 128) >> 8 everywhere for a DC-only
 * block (the reference's shortcut, which the transform equals), and a damaged picture follows decode_coefficients'
 * rule (the block with the bad code, and those after it, are 0).  For a clean stream, the residual of an intra
 * macroblock is its samples before the clamp (its prediction is 0), that of any other PRESENT macroblock what stage 2
 * adds to its prediction when decode() reconstructs the picture.  An intra block's DC enters the transform as dc * 256
 * (the reference's dc << 8) with dc clamped to [-16000, 16255], a clamp that changes no sample (the transform of the
 * rest of the block stays within +-14,315); while |dc| <= 4095 that is decode_coefficients' 8 * dc times 32.
 * Coefficients are clipped to [-2048, 2047], so every value of a non-intra block satisfies |r| <= 14,314 and every
 * value of an intra one lies in [-32,000, 32,255] (255 + 2 * 16000): inside int16 (tests/test_residual_export.py).  mb_dst may be NULL; otherwise
 * mb_dst[i] (16-byte aligned) gets exactly what decode_macroblocks writes for the request, from the same walk: its
 * INTRA / FORWARD / BACKWARD flags say how to read the residual.
 *
 * Synchronous; duplicates each get the data.  n_present_out / error_out (may be NULL) as decode_macroblocks.  Returns
 * n; -1 dead; -2 a request is invalid (stream out of range or without sequence header, picture not in the macroblock
 * index, NULL or misaligned res_dst[i], misaligned or NULL mb_dst[i] when mb_dst is given) -- checked before any
 * work, and then nothing changed.  Changes nothing decode() observes, as decode_intra. */
long jsmpeg_b200_batch_decode_residuals(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                        void *const *res_dst, void *const *mb_dst,
                                        int32_t *n_present_out, int32_t *error_out);

/* ACCUMULATED MOTION AND RESIDUALS (compressed-domain video models in the CoViAR style): chosen I and P pictures of any
 * streams traced back through their reference chain to the key picture.  Every sample of a P picture follows its
 * block's forward vector into the previous reference picture, and that sample's trace on, to the I picture or to
 * where the trace ends; its motion is the sum of the vectors along the way and its residual the sum of the
 * residuals.  So P picture k ~ the picture `back` references earlier, warped by the accumulated motion, plus the
 * accumulated residual, and a model can take any picture of a GOP without its neighbours.
 *
 * The pictures are the I and P entries of the picture index (type 1 or 2), with the same chain start.  The chain is
 * consumed by decode()'s rule with decode_b OFF: B pictures between references are skipped after their header, so
 * neither the listing nor the result depends on decode_b.  B pictures are not accepted.
 *
 * Request i = picture pictures[i] of stream streams[i] into acc_dst[i]: DEVICE memory, 16-byte aligned, of
 * coded_size * 3 / 2 records of jsmpeg_b200_accumulated_t (coded_size * 12 bytes), in the planes' layout counted in
 * samples: Y at 0, Cr at coded_size, Cb at coded_size * 5 / 4 -- the map lines up sample for sample with
 * decode_pictures' planes and decode_residuals' residual.  Every byte is written.
 *
 * The rule.  Let p0 (the I picture), p1, ..., pn = k be the chain's reference pictures as the fresh decoder of
 * decode_pictures reconstructs them.  The map M_m of p_m, per sample i (its flat index in its plane), with the
 * sample's macroblock in p_m's records and its 8 x 8 block:
 *   1. macroblock not PRESENT: untraced, back = -1, dx = dy = residual = 0;
 *   2. macroblock INTRA, or the block's prediction not inside the plane (stage 2's flat-index rule, half-sample taps
 *      included; stage 2 predicts 0 for such a block): back = 0, dx = dy = residual = 0 (every macroblock of p0 is
 *      under rule 1 or 2);
 *   3. otherwise (forward-predicted, skipped and zero-vector macroblocks included), v = the forward vector, luma as
 *      decode_macroblocks exports it, chroma each component halved with truncation toward zero (as stage 2), and
 *      i' = i + (v_y >> 1) * stride + (v_x >> 1), the sample's first prediction tap in p_{m-1}: if M_{m-1}(i') is
 *      untraced, so is the sample; else back = M_{m-1}(i').back + 1, (dx, dy) = sat16(M_{m-1}(i').d + v) and
 *      residual = sat16(M_{m-1}(i').residual + r_m(i)), r_m being decode_residuals' residual of p_m.  sat16 saturates
 *      to [-32768, 32767] at every depth.
 * For a clean stream, k(x) ~ clamp(p_{n-back}(x + d / 2) + residual), exact with full-sample vectors and no clamping
 * along the trace.
 *
 * status_out[i] (may be NULL) is PIC_DECODED, or 0 when the fresh decoder never consumes picture k: every record is
 * then untraced.  n_present_out / error_out (may be NULL) are those of picture k.  Synchronous; duplicates each get
 * the map.  Returns n; -1 dead; -2 a request is invalid (stream out of range or without sequence header, picture not
 * an I or P entry of the picture index, NULL or misaligned acc_dst[i], a chain of more than 32,767 reference pictures)
 * -- checked before any work, and then nothing changed.  Changes nothing decode() observes, as decode_intra. */
typedef struct jsmpeg_b200_accumulated_t {
	int16_t dx, dy;   /* accumulated motion, half-sample units of the sample's own plane */
	int16_t residual; /* accumulated residual */
	int16_t back;     /* reference pictures back to where the trace ends; -1: untraced */
} jsmpeg_b200_accumulated_t; /* 8 bytes */
long jsmpeg_b200_batch_decode_accumulated(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                          void *const *acc_dst, int32_t *status_out, int32_t *n_present_out,
                                          int32_t *error_out);

/* ACCUMULATED MAPS OF THE PLAYBACK PATH (live compressed-domain models on the pictures decode() plays: camera walls,
 * stream moderation, action recognition on ingest): with JSMPEG_B200_OUT_ACCUMULATED in the flags of
 * jsmpeg_b200_batch_decode or jsmpeg_b200_batch_seek_pictures (combined freely with OUT_HOST, OUT_RGBA and
 * OUT_MACROBLOCKS), every I or P picture the call reconstructs (PIC_DECODED, type 1 or 2) gets the map of
 * decode_accumulated beside its planes, from the records decode() reconstructs it from: no second walk, and one depth
 * step per picture instead of the whole chain.
 *
 * A stream has one MAP per I/P plane set: coded_size * 3 / 2 jsmpeg_b200_accumulated_t in decode_accumulated's layout.
 * The map of a reconstructed I/P picture is one step of decode_accumulated's rule from its own records, its own
 * residual and `prev`, the map beside the forward set it was predicted from.  `prev` counts as absent (predicted samples
 * untraced, intra samples back 0) unless a call with the flag wrote it for the picture that set holds: a reconstruct
 * without the flag, jsmpeg_b200_batch_reset, a seek without the flag and a stream that starts on a P picture break the
 * trace, which then stays untraced up to the next I picture.  B pictures (decode_b) get no map and leave both maps as
 * they are.
 *
 * So for a picture k that decode() reconstructs under the flag, after every reference picture from the last I picture
 * through k was also reconstructed under the flag, the map is decode_accumulated's fold over exactly the I/P pictures
 * decode() reconstructed from that I picture, with the records and residuals decode_macroblocks / decode_residuals
 * give for them -- on every clean stream byte for byte decode_accumulated of k.  After seek_pictures with the flag it is
 * decode_accumulated of k for an I/P picture k, or of the newer reference for a B picture k, wherever the seek's fresh
 * decoder and decode_accumulated's chain consume the same I/P pictures: every clean stream, and with decode_b off
 * always.  More than 32,767 reference pictures without an I picture (decode_accumulated refuses such a chain) are not
 * covered: `back` is int16 and wraps.
 *
 * Nothing else decode() observes changes: planes, RGBA, host ring, entries, bit index, last_picture and the stats, but
 * kernel_launches, which counts one accumulate launch per reconstruct step with an I/P picture.  The maps are not
 * copied to the host ring.  They are made on first use (2 x coded_size * 12 bytes per stream).
 *
 * Both calls give the map of the stream's NEWEST I/P picture -- the picture get_planes gives unless the last picture
 * was a B picture (last_picture tells).  A map no call with the flag wrote for that picture reads as all untraced
 * {0, 0, 0, -1}, so does every map before the first call with the flag.  Each returns 0, or non-zero for a dead batch,
 * a stream out of range or one without a sequence header. */
/* Device pointer to the map; valid until the next decode / seek, like get_planes. */
int jsmpeg_b200_batch_get_accumulated(jsmpeg_b200_batch_t *b, int stream, void **map);
/* Synchronous copy of the map into caller memory (coded_size * 12 bytes), like read_planes. */
int jsmpeg_b200_batch_read_accumulated(jsmpeg_b200_batch_t *b, int stream, void *dst);

/* RESIDUAL OF THE PLAYBACK PATH (live compressed-domain models -- I frames, motion vectors and residuals -- on the
 * pictures decode() plays): with JSMPEG_B200_OUT_RESIDUALS in the flags of jsmpeg_b200_batch_decode or
 * jsmpeg_b200_batch_seek_pictures (combined freely with OUT_HOST, OUT_RGBA, OUT_MACROBLOCKS and OUT_ACCUMULATED), the
 * reconstruct kernel also stores the pixel-domain residual it adds to the prediction: no second walk and no second
 * transform.
 *
 * A stream has one RESIDUAL: coded_size * 3 / 2 int16 in decode_residuals' layout (Y at 0, Cr at coded_size, Cb at
 * coded_size * 5 / 4, in samples), in device memory made zeroed on first use (coded_size * 3 bytes).  After a call
 * with the flag it is the residual of the picture get_planes gives, whenever a call with the flag reconstructed that
 * picture; for a picture decode() reconstructs (PIC_DECODED: I and P pictures, B pictures under decode_b) it equals byte
 * for byte what decode_residuals writes for the same picture k -- on damaged streams too, both reading the records of
 * the walk that starts at k's start code.  The rules are those of the entries (OUT_MACROBLOCKS): a call that
 * reconstructs nothing for a stream leaves its residual as it was; a call WITHOUT the flag writes none, so afterwards
 * the residual may describe an older picture than the planes; a residual no call with the flag wrote is 0, and again
 * after jsmpeg_b200_batch_reset (rewind leaves it, like the planes); seek_pictures with the flag: the residual of the
 * picture the stream's state ends on (picture k, or under status 0 the picture the fresh decoder ended on; 0 where
 * that decoder reconstructed nothing).
 *
 * Only the stream's newest picture's residual can be observed, so decode(n) with the flag stores it only for the last
 * picture each stream reconstructs in each of its rounds; a consumer that wants every picture's residual gives
 * jsmpeg_b200_batch_decode_frames residual destinations (below).  The residual is not copied to the host ring: at coded_size * 3 bytes per picture its
 * consumer is a model on the same GPU.  Nothing else decode() observes changes: planes, RGBA, host ring, entries, maps,
 * bit index, last_picture and the stats, but kernel_launches as described there.
 *
 * Each returns 0, or non-zero for a dead batch, a stream out of range or one without a sequence header. */
/* Device pointer to the residual; valid until the next decode / seek, like get_planes. */
int jsmpeg_b200_batch_get_residuals(jsmpeg_b200_batch_t *b, int stream, void **res);
/* Synchronous copy of the residual into caller memory (coded_size * 3 bytes), like read_planes. */
int jsmpeg_b200_batch_read_residuals(jsmpeg_b200_batch_t *b, int stream, void *dst);

/* EVERY PICTURE OF decode(n) (clip loaders for training, video walls, compressed-domain models): decode(n) reconstructs
 * up to n pictures of every stream, but afterwards only the last one of each can be seen.  decode_frames does exactly
 * what jsmpeg_b200_batch_decode(b, n_pictures, flags) does and returns the same value, and also gives each picture it
 * reconstructs a destination of its own in caller device memory, written by stage 2 beside the planes: no copy-out per
 * picture and no decode(1) loop.
 *
 * FRAME j of stream s is the j-th picture the call reconstructs for s (PIC_DECODED: I and P pictures, B pictures under
 * decode_b), in consumption (coded) order; a skipped picture has none, although decode() returns true for it.
 * n_frames_out[s] (<= n_pictures) counts them.  Each destination array has one pointer per stream to device memory,
 * 16-byte aligned; frame j is at
 *   planes_dst[s] + j * coded_size * 3 / 2 bytes: what read_planes gives right after the decode() that consumed the
 *       picture (Y | Cr | Cb) -- on damaged streams too, where absent macroblocks keep the plane set's older content;
 *   rgba_dst[s] + j * width * height * 4 bytes: what read_rgba gives after that decode() had it run with OUT_RGBA (the
 *       odd edge opaque white);
 *   res_dst[s] + j * coded_size * 3 / 2 int16: byte for byte what decode_residuals writes for the picture (the residual
 *       OUT_RESIDUALS stores);
 *   mb_dst[s] + j * mb_size jsmpeg_b200_macroblock_t: byte for byte what decode_macroblocks writes for it.
 * Any of the four arrays may be NULL, and so may any entry of them: the stream then gets no frames of that kind.  Memory
 * past frame n_frames_out[s] - 1 is left untouched.  info_out (NULL: none) has n_streams * n_pictures entries, stream
 * s's frame j at s * n_pictures + j; n_frames_out (NULL: none) has n_streams.
 *
 * Per 1080p frame (1920 x 1088 coded, 120 x 68 macroblocks): planes 3,133,440 bytes, RGBA 8,294,400, residual 6,266,880,
 * macroblock entries 130,560 -- so 64 streams x 60 planar frames take about 12 GB.
 *
 * Everything decode() observes afterwards is what decode() leaves: planes, RGBA, host ring, entries, maps, residual,
 * bit index, last_picture and the stats, but kernel_launches (a step's reconstruct kernel with a frame is cut into
 * launches of its FRAME variant's capacity: 63 plain, 51 RGBA, 56 B, 46 B + RGBA tasks).  The flags keep their meaning
 * for decode()'s own buffers: with OUT_RGBA and an RGBA frame the stream's RGBA ends as its last frame, with
 * OUT_RESIDUALS and a residual frame the stream's residual ends as its last frame's; an RGBA frame without OUT_RGBA
 * leaves get_rgba as it was.
 *
 * Synchronous.  Returns what decode() returns; -1 for a dead batch; -2, before any work and with nothing changed, when
 * n_pictures < 0 or a destination is not 16-byte aligned. */
typedef struct jsmpeg_b200_frame_t {
	uint32_t byte_pos;          /* the picture's start code in the stream's buffer (the index calls' byte_pos) */
	int16_t picture_type;       /* 1 I, 2 P, 3 B (decode_b) */
	int16_t temporal_reference; /* as jsmpeg_b200_batch_last_picture */
	int32_t n_present, error;   /* picture_info_t.n_present / .error, as decode_pictures reports them */
} jsmpeg_b200_frame_t;          /* 16 bytes */

long jsmpeg_b200_batch_decode_frames(jsmpeg_b200_batch_t *b, int n_pictures, int flags, void *const *planes_dst,
                                     void *const *rgba_dst, void *const *res_dst, void *const *mb_dst,
                                     jsmpeg_b200_frame_t *info_out, int32_t *n_frames_out);

/* EVERY COMPRESSED-DOMAIN INPUT OF decode(n) (CoViAR-style clip loaders, DCT-domain models): decode_frames_into is
 * jsmpeg_b200_batch_decode_frames with two more kinds of frame, from the walk and expand decode() does anyway.  `dst`
 * (not NULL) holds the four arrays of decode_frames, with their meaning, and per stream (any array or entry NULL: none)
 *   coef[s] + j * mb_size * 768 bytes: byte for byte what decode_coefficients writes for frame j's picture (per
 *       macroblock 6 blocks of 64 int16) -- I, P and B frames, damaged streams too, both reading the records of the walk
 *       that starts at the picture's start code.  No flag is needed.
 *   acc[s] + j * coded_size * 12 bytes: for an I/P frame, byte for byte what read_accumulated gives right after the
 *       decode(1, flags) that reconstructs the picture, with OUT_ACCUMULATED's `prev` rules unchanged (a trace broken by
 *       a call without the flag, reset, a seek without the flag or a start on a P picture stays untraced up to the next I
 *       picture; maps of this call chain on into the next one); for a B frame all untraced {0, 0, 0, -1}.  A map
 *       destination requires JSMPEG_B200_OUT_ACCUMULATED in `flags`, so that the batch state stays decode(n, flags)'s.
 * Every frame below n_frames_out[s] is fully written; memory past it is left untouched.  Destinations of different
 * streams or kinds must not overlap.  Per 1080p frame: coefficients 6,266,880 bytes, map 25,067,520 bytes -- so 64
 * streams x 8 map frames take about 12.8 GB.
 *
 * Everything decode() observes afterwards is what decode(n, flags) leaves, maps included, but kernel_launches (one more
 * coefficient export launch per reconstruct step with a coefficient frame).  decode_frames(b, n, flags, p, r, e, m, i,
 * f) is decode_frames_into with {p, r, e, m, NULL, NULL}.
 *
 * Synchronous.  Returns what decode() returns; -1 for a dead batch; -2, before any work and with nothing changed, when
 * dst is NULL, n_pictures < 0, a destination is not 16-byte aligned, or an acc entry is given without OUT_ACCUMULATED. */
typedef struct jsmpeg_b200_frame_dst_t {
	void *const *planes, *const *rgba, *const *res, *const *mb; /* decode_frames' four arrays */
	void *const *coef;                                           /* per stream: frame j at + j * mb_size * 768 bytes */
	void *const *acc;                                            /* per stream: frame j at + j * coded_size * 12 bytes */
} jsmpeg_b200_frame_dst_t;

long jsmpeg_b200_batch_decode_frames_into(jsmpeg_b200_batch_t *b, int n_pictures, int flags, const jsmpeg_b200_frame_dst_t *dst,
                                          jsmpeg_b200_frame_t *info_out, int32_t *n_frames_out);

/* EVERY PICTURE OF decode(n) IN DISPLAY ORDER (clip loaders, video walls on IBBP content): decode_frames_display does to
 * the batch exactly what decode_frames_into(b, n_pictures, flags, dst, ...) does and returns the same value, but hands
 * the frames over in presentation order, each stored by stage 2 straight into its place.
 *
 * PRESENTATION, per stream, over the pictures the call reconstructs (PIC_DECODED), in consumption order -- the rule of
 * MPEG1Video's displayOrder (jsmpeg_b200/decoder.py): a B picture is presented at once; an I/P picture first presents
 * the I/P picture the stream holds, if any, and is then held itself; skipped pictures present nothing.  A held picture
 * carries over into the next call (which presents it when its successor reference arrives) or is presented by
 * jsmpeg_b200_batch_flush_frames (end of clip).  Without decode_b a stream has no B pictures, and every I/P picture is
 * presented at once: the frames are decode_frames_into's, in its order, and nothing is held.  With decode_b, a stream
 * without B pictures lags one held picture behind, as MPEG1Video does.
 *
 * FRAME j of stream s is the j-th picture the call presents, a held one of an earlier call included, so n_frames_out[s]
 * may be n_pictures + 1: size each destination for n_pictures + 1 frames (at the offsets of decode_frames_into), and
 * info_out (NULL: none) for n_streams * (n_pictures + 1) entries, stream s's frame j at s * (n_pictures + 1) + j.  Each
 * frame of each kind is byte for byte what decode_frames_into writes for that picture (the map rule of I/P frames,
 * untraced B maps included); memory past frame n_frames_out[s] - 1 is left untouched.
 *
 * HELD PICTURES live in a per-stream store of one frame of each kind the holding call asked for, made on first use.  A
 * held picture is dropped, never presented, by reset, rewind, set_index, seek_pictures, and by decode(), decode_frames,
 * decode_frames_into or any other call that reconstructs a picture into the stream's plane sets; emptying the stream's
 * buffer (EVICT) keeps it.
 *
 * Everything decode() observes afterwards is what decode(n, flags) leaves, as for decode_frames_into; with OUT_RGBA /
 * OUT_RESIDUALS the stream's RGBA and residual end as those of the last RECONSTRUCTED picture (held or presented).
 *
 * Synchronous.  Returns what decode() returns; -1 for a dead batch; -2, before any work and with nothing changed, for
 * decode_frames_into's reasons, or when a stream holds a picture and the call asks for a kind (a non-NULL entry) the
 * holding call did not. */
long jsmpeg_b200_batch_decode_frames_display(jsmpeg_b200_batch_t *b, int n_pictures, int flags,
                                             const jsmpeg_b200_frame_dst_t *dst, jsmpeg_b200_frame_t *info_out,
                                             int32_t *n_frames_out);

/* End of clip: presents every stream's held picture (decode_frames_display) as its frame 0 -- each kind `dst` asks for,
 * at frame 0's place -- with n_frames_out[s] 0 or 1 and info_out (NULL: none) of n_streams entries, and releases the
 * holds.  It reconstructs nothing and changes nothing else decode() observes.  Synchronous.  Returns the number of
 * pictures presented; -1 for a dead batch; -2, before any work and with nothing changed, when dst is NULL, a destination
 * is not 16-byte aligned, or a stream holds a picture without a kind the call asks for. */
long jsmpeg_b200_batch_flush_frames(jsmpeg_b200_batch_t *b, const jsmpeg_b200_frame_dst_t *dst, jsmpeg_b200_frame_t *info_out,
                                    int32_t *n_frames_out);

/* SEEK (players, video walls, clip loaders): move decode() of chosen streams to a chosen picture each, and play on from
 * there with decode() -- OUT_HOST, OUT_RGBA and the host ring as usual -- without stepping the other streams.  The
 * reference chains of all requests run side by side, as for decode_pictures, but into the streams' own plane sets.
 *
 * Request i moves stream streams[i] to picture pictures[i], an entry of the stream's picture index under the batch's
 * current decode_b (the listing and numbering of decode_pictures).  A stream may be named at most once per call.
 *
 * The seek chain start j is the index's chain start, except that under decode_b an I picture k needs ONE reference in
 * [j, k), not zero: the greatest I picture before k (k itself where there is none), so that the B pictures after k
 * of an open GOP are decoded from both their references.
 *
 * For each named stream, everything decode() observes afterwards is exactly what a FRESH decoder shows right after its
 * decode() that consumes picture k, the fresh decoder having every plane set zeroed (the B sets too), the batch's
 * decode_b, and being fed the first sequence header and then the stream's resident bytes from picture j to the end of
 * the buffer.  Translated to the stream's buffer: the bit index is picture k's end; get_planes / read_planes give
 * picture k, under OUT_HOST in `flags` also copied to the next slot of the host ring (get_host_planes), under
 * OUT_RGBA also converted to the stream's RGBA picture (get_rgba / read_rgba) -- `flags` as for decode(); the two I/P
 * sets and the two B sets hold what the fresh decoder's hold, and the next picture overwrites the same ones (every B
 * picture the fresh decoder reconstructs in (j, k] is reconstructed: a later picture's absent macroblocks keep a set's
 * content); last_picture gives k's type and temporal_reference.  So for a stream that begins with an I picture and
 * whose pictures from j on code every macroblock, every later decode() gives what sequential decode() from the start
 * gives at that point.
 *
 * Damaged input: the fresh decoder may never consume k, an earlier picture's walk having run across k's start code;
 * status_out[i] is then 0 and the stream is left as the fresh decoder is after that decode() (its picture written to
 * RGBA / the host ring as above).  Otherwise status_out[i] is PIC_DECODED.  n_present_out / error_out are those of the
 * picture the state ends on.  All three may be NULL.
 *
 * Unchanged: streams not named (their parsed-ahead pictures may be dropped for record slots, as in decode_intra);
 * resident bytes, sequence parameters and the decode_b option; stats, except that written bytes become resident and
 * that upload is counted.  A named stream's parsed-ahead pictures are dropped.  Synchronous.  Returns n; -1 dead; -2 a
 * request is invalid (stream out of range, without sequence header or named twice, picture not in the picture index,
 * NULL arrays with n > 0) -- checked before any work, and then nothing changed. */
long jsmpeg_b200_batch_seek_pictures(jsmpeg_b200_batch_t *b, int n, const int *streams, const uint32_t *pictures,
                                     int flags, int32_t *status_out, int32_t *n_present_out, int32_t *error_out);

void jsmpeg_b200_batch_get_stats(jsmpeg_b200_batch_t *b, jsmpeg_b200_stats_t *out);
void jsmpeg_b200_batch_reset_stats(jsmpeg_b200_batch_t *b);

/* ------------------------------------------------------------------------------------------ */
/* Test hooks (used by tests/ only): run a single stage on caller-provided device-agnostic data */

/* Stage 1 alone: parse the picture whose start code ends at start_byte of `es` (host memory) and
 * copy the records back to host arrays sized mb_size * 16 B and mb_size * 768 B. */
int jsmpeg_b200_debug_parse_picture(const uint8_t *es, uint32_t es_len, uint32_t start_byte,
                                    int mb_width, int mb_height, const uint8_t *intra_q,
                                    const uint8_t *non_intra_q, void *info_out, void *hdr_out,
                                    void *coef_out);
/* Stage 2 alone: reconstruct one picture from host record arrays and host forward planes. */
int jsmpeg_b200_debug_reconstruct(int mb_width, int mb_height, const void *hdr, const void *coef,
                                  const uint8_t *fwd_y, const uint8_t *fwd_cr, const uint8_t *fwd_cb,
                                  uint8_t *cur_y, uint8_t *cur_cr, uint8_t *cur_cb);

/* Copy the first min(cap, resident) bytes of the stream's elementary stream as it is resident in HBM into
 * `dst`; returns the resident byte count (-1: the batch is dead). */
long jsmpeg_b200_debug_read_es(jsmpeg_b200_batch_t *b, int stream, void *dst, size_t cap);

/* NULL while the decoder works, else why it is dead (see mpeg1_decoder_create). */
const char *jsmpeg_b200_decoder_last_error(mpeg1_decoder_t *self);

/* jsmpeg_b200_batch_set_option / jsmpeg_b200_batch_last_picture for a decoder of the reference ABI (which has no
 * option call): "decode_b" switches the B-picture extension on, "conceal" error concealment, "lookahead" sets the
 * pictures parsed ahead.  The
 * decoder's own option "macroblocks" (default 0): with 1, mpeg1_decoder_decode decodes with JSMPEG_B200_OUT_MACROBLOCKS
 * and jsmpeg_b200_decoder_get_macroblocks returns the entries of the picture it rendered (what get_y_ptr shows). */
int jsmpeg_b200_decoder_set_option(mpeg1_decoder_t *self, const char *name, int value);
int jsmpeg_b200_decoder_last_picture(mpeg1_decoder_t *self, int *picture_type, int *temporal_reference);
/* HOST-visible (pinned) mb_height * mb_width jsmpeg_b200_macroblock_t (jsmpeg_b200_batch_get_host_macroblocks);
 * borrowed until the next decode; NULL before the sequence header or when the decoder is dead. */
void *jsmpeg_b200_decoder_get_macroblocks(mpeg1_decoder_t *self);

/* CUDA device for decoders created through the reference ABI from now on (the reference ABI has no
 * device argument; the JS/Python class passes its `device` option here). */
void jsmpeg_b200_set_default_device(int device);

/* Bind the calling thread (and the threads it creates, and the pages it first touches, from now on) to
 * the CPUs of the NUMA node CUDA device `device` hangs off, intersected with its current affinity: a
 * decoder's pinned bit buffer and plane ring should live next to its GPU.  Returns the number of CPUs
 * bound to, 0 when the node is unknown (nothing changed), -1 on error; *node_out (may be NULL) = the node. */
int jsmpeg_b200_bind_host_to_device(int device, int *node_out);

const char *jsmpeg_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif
