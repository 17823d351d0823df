/*
 * records.h -- the stage-1 -> stage-2 record format (plain C, shared by CUDA, the host C ABI and,
 * as a format definition only, by the test oracle).
 *
 * Stage 1 (bitstream/VLC parse, one warp per picture) walks the macroblocks of a picture serially
 * and emits, per macroblock ADDRESS, one 16-byte header and up to six 64 x int16 coefficient
 * blocks.  Stage 2 (one group of threads per macroblock) reads them, runs the integer IDCT,
 * fetches the half-pel reference patch, adds + clamps and writes planar Y/Cr/Cb.
 *
 * Layout in HBM for one picture slot (mb_size = mb_width * mb_height):
 *     mb_record_t hdr [mb_size]                    16 B each, indexed by macroblock address
 *     int16_t     coef[mb_size][6][64]            128 B per block, de-zigzagged (raster) order,
 *                                                 only blocks whose cbp bit is set are written/read
 *     uint2       park[mb_size][6]                the walk's hand-over to stage 1b (common.cuh: ParseTask)
 *     staging area                                the lane-parallel walk's relative records; once the walk is done,
 *                                                 the compact coefficient plane: 32 B per block (coef_records.h)
 * Fixed slots (no allocation, no offsets): any slice / picture can be parsed independently.
 * Stage 1b hands a coded block over as its 32-byte compact record (a position mask + at most 12 values,
 * coef_records.h); only a block with more values is written here, as the 128-byte dense record below, and
 * its compact record says so.
 *
 * Coefficient values: the reference keeps `level * PREMULTIPLIER_MATRIX[i]` in int32
 * (src/mpeg1.js:810); that does not fit int16 (2047*62), so the record holds the dequantised,
 * oddified, clipped level in [-2048, 2047] (src/mpeg1.js:794-807) and stage 2 applies the
 * premultiplier in int32.  Intra DC is stored as dc itself, and stage 2 multiplies an intra block's coefficient 0
 * by 256 instead of PREMULTIPLIER[0] (= 32): the reference's `dc << 8` (src/mpeg1.js:747).  The predictor is an
 * unbounded sum of differentials (up to +-255 per block), so the record clamps it to
 * [-INTRA_DC_BOUND, 255 + INTRA_DC_BOUND], and that is exact: in the reference's transform the DC term is only ever
 * added (src/mpeg1.js:916-983), so every intra sample is clamp255(dc + ac(x)), ac being the transform of the block with
 * its DC set to 0, and |ac(x)| <= 14,315 (DESIGN 3.10's bound for any block of coefficients in [-2048, 2047]) <
 * INTRA_DC_BOUND.  A DC past either end therefore gives 0 or 255 in every sample, clamped or not.  The range fits
 * int16, and so does every residual of an intra block: |dc + ac(x)| <= 255 + 2 * INTRA_DC_BOUND = 32,255.
 * (decode_coefficients still reports an intra DC as sat16(8 * dc): the export converts it.)
 */
#ifndef JSMPEG_B200_RECORDS_H
#define JSMPEG_B200_RECORDS_H

#include <stdint.h>

#define MBF_PRESENT 0x01 /* macroblock was decoded (coded or skipped-predicted): stage 2 writes it   */
#define MBF_INTRA   0x02 /* intra macroblock: blocks overwrite; otherwise predict from forward + add */
#define MBF_SKIPPED 0x04 /* produced by an address increment > 1 (informational)                     */
/* B pictures only (the opt-in extension; the reference skips B pictures, mpeg1.js:181-184): which of the two
 * references a non-intra macroblock is predicted from -- both set = the rounded average of the two predictions
 * (ISO 11172-2 2.4.4.3).  In I and P records both bits are 0 and a non-intra macroblock predicts from forward. */
#define MBF_MOTION_BWD 0x08 /* from the backward (future) reference, vector mv_bwd */
#define MBF_MOTION_FWD 0x10 /* from the forward (past) reference, vector mv_h / mv_v */

typedef struct mb_record_t {
	int16_t mv_h;       /* forward motion vector, luma half-pel units, after full_pel doubling  */
	int16_t mv_v;
	uint8_t flags;      /* MBF_*                                                                 */
	uint8_t cbp;        /* bit (5 - block) set <=> block coded   (mask 0x20 >> block, mpeg1.js:386-391) */
	uint8_t dc_only;    /* same bit order: block takes the n==1 scalar shortcut (mpeg1.js:838-841,850-853) */
	uint8_t qscale;     /* quantiser_scale in force (informational)                              */
	uint32_t bit_pos;   /* bit offset of the macroblock inside the picture's ES span (diagnostic) */
	uint32_t mv_bwd;    /* B pictures: backward vector, (uint16)h | (uint16)v << 16, same units; else 0 */
} mb_record_t;

#define MB_COEF_INT16 (6 * 64)
#define INTRA_DC_BOUND 16000   /* intra DC in the records: clamped to [-INTRA_DC_BOUND, 255 + INTRA_DC_BOUND] */ /* int16 per macroblock in the coefficient plane */

/* Picture-level result of stage 1 (one per picture start code that decode() consumes). */
#define PIC_DECODED 1 /* I or P picture: reconstruct + swap (mpeg1.js:216-246)                  */
#define PIC_IGNORED 2 /* B / D / unknown type, or P with forward_f_code == 0 (mpeg1.js:181-193) */
/* With the B-picture extension switched on, a B picture (type 3) is PIC_DECODED too: it is reconstructed from
 * the two most recent I/P pictures into a set of its own and does NOT become a reference (no plane swap);
 * reserved[1] then holds full_pel_backward << 4 | backward_f_code. */

typedef struct picture_info_t {
	uint32_t start_byte;    /* first byte after the 00 00 01 00 start code                      */
	uint32_t end_bit;       /* bit index at which the reference's decode_picture returns         */
	int32_t  status;        /* PIC_*                                                             */
	int32_t  picture_type;  /* 1 = I, 2 = P (3 = B with the extension)                           */
	int32_t  full_pel;
	int32_t  f_code;
	int32_t  n_present;     /* macroblocks with MBF_PRESENT                                      */
	int32_t  n_coded_blocks;
	int32_t  error;         /* 0, or a PARSE_ERR_* code when the slice walk hit an invalid code   */
	int32_t  reserved[3];
} picture_info_t;

#define PARSE_ERR_INVALID_VLC 1
#define PARSE_ERR_COEF_INDEX  2 /* run pushed the zig-zag index past 63 */

#endif
