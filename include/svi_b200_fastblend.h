/*
 * svi_b200_fastblend.h — FastBlend video deflickering (PatchMatch + blending tables) on libsvi_b200.so (the same library
 * as svi_b200.h).
 *
 * diffsynth/extensions/FastBlend matches every frame of a window against its neighbours with a coarse-to-fine
 * PatchMatch and blends the remapped frames.  Its arithmetic is fp32 SIMT work (no tensor cores) in these entry points:
 *
 *   svi_fastblend_stage_frames   uint8 RGB frames -> f32 [n][4] operands (the frames cross the bus once, as bytes)
 *   svi_fastblend_downsample     integer-ratio pyramid level: cv2.resize(INTER_AREA)'s summation order, bit for bit
 *   svi_fastblend_nnf_identity   the identity nearest-neighbour field of the coarsest level
 *   svi_fastblend_nnf_upscale    the field of a level from the one below it (exactly doubled sizes)
 *   svi_fastblend_remap          the style frame remapped through a field (mean over the valid patch taps)
 *   svi_fastblend_step           one PatchMatch step: a candidate field, its guide and style patch errors, the select
 *   svi_fastblend_table          the blending tables' weighted sums, in the dtype numpy gives each of them
 *
 * Layouts are channels-last with the channel padded to 4 (channel 3 is zero and never read into a sum).  A field
 * (nnf) is int32 [B][H][W][2]: (row, column) of the source pixel matched to each target pixel.
 * Rounding: every sum and product is rounded on its own (no fused multiply-add, no reassociation); every output element
 * is computed by one thread in a fixed order, without atomics, so the same input gives the same bytes.
 * Conventions as in svi_b200.h: 0 on success, a negative status (and svi_last_error) on a rejected argument, in which
 * case nothing is launched; every launch is on `stream`.
 * A separate header so that svi_b200.h and its ABI version stay as they are.
 */
#ifndef SVI_B200_FASTBLEND_H_
#define SVI_B200_FASTBLEND_H_

#include <stdint.h>

#include "svi_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* largest patch the step kernel takes (its target windows live in shared memory) */
#define SVI_FASTBLEND_MAX_PATCH 61

/* candidate of one svi_fastblend_step */
#define SVI_FASTBLEND_CURRENT 0   /* the input field itself; the error is written unconditionally (no select) */
#define SVI_FASTBLEND_NEIGHBOUR 1 /* the neighbour step `dir` (0: from the row above, +1 row; 1: from the column to the
                                     left, +1 column; 2: from the row below, -1 row; 3: from the column to the right,
                                     -1 column; an edge row / column takes its own entry), then clamped */
#define SVI_FASTBLEND_RANDOM 2    /* field + randint(-radius, radius + 1) of draw `draw` (the stream below), clamped */

/* The random stream (uint32, wrap-around):
 *   lowbias32(x): x ^= x >> 16; x *= 0x7feb352d; x ^= x >> 15; x *= 0x846ca68b; x ^= x >> 16
 *   u(k, i)     = lowbias32(lowbias32(k ^ 0x9e3779b9) ^ i)
 * Draw k of randint(lo, hi) gives element i (flat C-order index into [B][H][W][2]) the value lo + u(k, i) % (hi - lo). */

/* One PatchMatch step over a batch of B target frames of H x W pixels, patch of (patch_size | 1) x (patch_size | 1)
 * taps (r = (patch_size - 1) / 2).  For each pixel: the candidate field entry (y', x') (see the modes above), then
 *   e_guide = sum over px in [-r, r], py in [-r, r], c in 0..2 of (tgt_guide[y+px][x+py][c] - src_guide[y'+px][x'+py][c])^2
 *   e_style = the same of tgt_style and src_style
 * with a tap outside the frame reading 0 on either side, the sum in px, py, c order, each square and each addition
 * rounded on its own; e = e_guide * guide_weight + e_style (two roundings).  Mode CURRENT writes (field, e); the others
 * write the candidate and e where e < err_in, and the input entry and err_in elsewhere.  nnf_out / err_out must not
 * alias nnf_in / err_in (a neighbour step reads entries other threads replace). */
typedef struct svi_fastblend_step_desc {
  const float* src_guide;   /* f32 [B][H][W][4] */
  const float* src_style;   /* f32 [B][H][W][4] */
  const float* tgt_guide;   /* f32 [B][H][W][4] */
  const float* tgt_style;   /* f32 [B][H][W][4]: src_style remapped through the field (svi_fastblend_remap) */
  const int32_t* nnf_in;    /* int32 [B][H][W][2], every entry inside the frame */
  const float* err_in;      /* f32 [B][H][W]; unused with mode CURRENT */
  int32_t* nnf_out;         /* int32 [B][H][W][2] */
  float* err_out;           /* f32 [B][H][W] */
  int32_t B, H, W;
  int32_t patch_size;       /* 1 .. SVI_FASTBLEND_MAX_PATCH */
  int32_t mode;             /* SVI_FASTBLEND_CURRENT / _NEIGHBOUR / _RANDOM */
  int32_t dir;              /* neighbour step, 0..3 */
  uint32_t draw;            /* random step: the stream's draw counter k */
  int32_t radius;           /* random step: offsets in [-radius, radius] */
  float guide_weight;
} svi_fastblend_step_desc;

/* dtype of a blending-table frame (f32 storage [n][4] unless said otherwise) */
#define SVI_FASTBLEND_U8 0        /* a uint8 frame held as its f32 values 0..255 (promoted as numpy promotes uint8) */
#define SVI_FASTBLEND_F32 1
#define SVI_FASTBLEND_F64 2       /* f64 storage [n][4] */

/* table operations, per pixel and channel 0..2 (channel 3 of an f32 / f64 output is written 0) */
#define SVI_FASTBLEND_MEAN 0      /* out f32 = a * f32(sa) + b / f32(sb)                      (a, b f32) */
#define SVI_FASTBLEND_HALF 1      /* out f32 = (a + b) / 2                                    (a uint8 or f32, b f32) */
#define SVI_FASTBLEND_WSUM 2      /* out = t(a, sa) + t(b, sb) [+ t(c, sc)], numpy's promotion: t(x, s) is
                                     f64(x) * s for a uint8 or f64 x, and x * f32(s) in f32 for an f32 x; a sum is
                                     f32 when both sides are, f64 otherwise.  out_type is F32, F64 or U8; a U8 output
                                     is uint8 [n][3] of the clip(0, 255) value truncated toward zero. */
typedef struct svi_fastblend_table_desc {
  int32_t op;
  int64_t n_pix;
  const void* a; int32_t a_type; double sa;
  const void* b; int32_t b_type; double sb;
  const void* c; int32_t c_type; double sc;   /* WSUM only, or null */
  void* out; int32_t out_type;
} svi_fastblend_table_desc;

/* out f32 [n][4] = R, G, B, 0 of uint8 rgb [n][3] (exact) */
int svi_fastblend_stage_frames(const uint8_t* rgb, int64_t n_pix, float* out, void* stream);
/* dst f32 [n][H/k][W/k][4] of src f32 [n][H][W][4], H and W multiples of k: per output element the k x k cell in row-major
 * order, sum += ((v0 + v1) + v2) + v3 over each group of four, then the remaining taps one by one, then sum * (1 / k^2) */
int svi_fastblend_downsample(const float* src, int32_t n, int32_t H, int32_t W, int32_t k, float* dst, void* stream);
/* nnf int32 [B][H][W][2] = (y, x) */
int svi_fastblend_nnf_identity(int32_t* nnf, int32_t B, int32_t H, int32_t W, void* stream);
/* dst int32 [B][2h][2w][2] of src int32 [B][h][w][2]: entry (y, x) = 2 src(y / 2, x / 2), plus 1 on the row of an odd y
 * below B and on the column of an odd x below B, clamped to the frame */
int svi_fastblend_nnf_upscale(const int32_t* src, int32_t B, int32_t h, int32_t w, int32_t* dst, void* stream);
/* out f32 [B][H][W][4]: per pixel the mean over the taps (px, py) in [-r, r]^2 with (y + px, x + py) and
 * (y', x') = nnf(y + px, x + py) - (px, py) inside the frame of style(y', x'), summed in px, py order, then divided */
int svi_fastblend_remap(const float* style, const int32_t* nnf, int32_t B, int32_t H, int32_t W, int32_t patch_size,
                        float* out, void* stream);
int svi_fastblend_step(const svi_fastblend_step_desc* d, void* stream);
int svi_fastblend_table(const svi_fastblend_table_desc* d, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SVI_B200_FASTBLEND_H_ */
