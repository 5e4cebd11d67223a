/*
 * svi_b200_fastblend_modes.h — FastBlend's balanced and accurate deflicker modes and keyframe interpolation on
 * libsvi_b200.so (the same library as svi_b200.h and svi_b200_fastblend.h).
 *
 * These modes run the PatchMatch of svi_b200_fastblend.h with three more options of the reference's PatchMatcher:
 *   - tracking: after the random search of each iteration, the fields of the neighbouring batch entries as candidates
 *     (entry clamp(b + d, 0, B - 1)'s field for d = 1, -1, 2, -2, ..., T, -T);
 *   - mean target style (the accurate mode): every error evaluation measures the style against the batch mean of the
 *     source style remapped through the field being evaluated;
 *   - pairwise patch error (keyframe interpolation): entries 2k and 2k + 1 share one style error, the patch distance
 *     between their two source styles at their two candidates.
 * A candidate therefore has to exist as a field before its error can be taken, so a step of these modes is
 *   svi_fastblend_candidate  -> [svi_fastblend_remap -> svi_fastblend_batch_mean] -> svi_fastblend_select,
 * where the bracketed part is the mean target style's.  svi_fastblend_running_mean and svi_fastblend_to_u8 are the
 * balanced and accurate modes' blends (the interpolation blend is svi_fastblend_table's WSUM).
 *
 * Layouts, rounding and conventions as in svi_b200_fastblend.h: channels-last frames padded to 4, int32 [B][H][W][2]
 * fields, every sum and product rounded on its own, one output element per thread in a fixed order, no atomics.
 */
#ifndef SVI_B200_FASTBLEND_MODES_H_
#define SVI_B200_FASTBLEND_MODES_H_

#include <stdint.h>

#include "svi_b200_fastblend.h"

#ifdef __cplusplus
extern "C" {
#endif

/* candidate modes of svi_fastblend_candidate: SVI_FASTBLEND_NEIGHBOUR and SVI_FASTBLEND_RANDOM (as svi_fastblend_step
 * builds them), and: */
#define SVI_FASTBLEND_TRACK 3     /* entry b takes the field of entry clamp(b + shift, 0, B - 1); with `pairwise`, of
                                     entry 2 clamp(b / 2 + shift, 0, P - 1) + b % 2, P the entries of b's parity */

typedef struct svi_fastblend_candidate_desc {
  const int32_t* nnf_in;    /* int32 [B][H][W][2], every entry inside the frame */
  int32_t* nnf_out;         /* int32 [B][H][W][2], not aliasing nnf_in */
  int32_t B, H, W;
  int32_t mode;             /* SVI_FASTBLEND_NEIGHBOUR / _RANDOM / _TRACK */
  int32_t dir;              /* neighbour: 0..3 as in svi_fastblend_step */
  uint32_t draw;            /* random: the stream's draw counter k */
  int32_t radius;           /* random: offsets in [-radius, radius] */
  int32_t shift;            /* track: d, nonzero */
  int32_t pairwise;         /* track: shift within the even and the odd entries */
} svi_fastblend_candidate_desc;

/* The error of a given candidate field and the select, per pixel of B target frames:
 *   e_guide = the patch distance of svi_fastblend_step between tgt_guide and src_guide at the candidate
 *   e_style = the same between the target style and src_style, where the target style is tgt_style[b], or the one frame
 *             tgt_style for every b when style_shared; with `pairwise` (B even), for both entries of the pair
 *             k = b / 2 instead: sum over px, py, c of (src_style[2k][cand(2k) + (px, py)] -
 *             src_style[2k + 1][cand(2k + 1) + (px, py)])^2, a tap outside the frame reading 0 on either side
 *   e       = e_guide * guide_weight + e_style
 * With select 0, writes (cand, e); with select 1, (cand, e) where e < err_in and (nnf_in, err_in) elsewhere. */
typedef struct svi_fastblend_select_desc {
  const float* src_guide;   /* f32 [B][H][W][4] */
  const float* src_style;   /* f32 [B][H][W][4] */
  const float* tgt_guide;   /* f32 [B][H][W][4] */
  const float* tgt_style;   /* f32 [B][H][W][4], or [H][W][4] with style_shared; unused (may be null) with pairwise */
  const int32_t* cand;      /* int32 [B][H][W][2], every entry inside the frame */
  const int32_t* nnf_in;    /* int32 [B][H][W][2]; unused with select 0 */
  const float* err_in;      /* f32 [B][H][W]; unused with select 0 */
  int32_t* nnf_out;         /* int32 [B][H][W][2], not aliasing cand or nnf_in */
  float* err_out;           /* f32 [B][H][W], not aliasing err_in */
  int32_t B, H, W;
  int32_t patch_size;       /* 1 .. SVI_FASTBLEND_MAX_PATCH */
  int32_t select;           /* 0 or 1 */
  int32_t style_shared;     /* 0 or 1 */
  int32_t pairwise;         /* 0 or 1 */
  float guide_weight;
} svi_fastblend_select_desc;

int svi_fastblend_candidate(const svi_fastblend_candidate_desc* d, void* stream);
int svi_fastblend_select(const svi_fastblend_select_desc* d, void* stream);
/* out f32 [n][4] = the mean of src f32 [B][n][4] over B: an f32 sum in b order, then / f32(B) (numpy's mean(axis=0)) */
int svi_fastblend_batch_mean(const float* src, int32_t B, int64_t n_pix, float* out, void* stream);
/* out f64 [n][4] = f64(frame) * s + f64(result / f32(divisor)), frame SVI_FASTBLEND_U8 (a uint8 frame held as f32) or
 * SVI_FASTBLEND_F64, result f32 [n][4]: the balanced mode's running mean (numpy's promotion: the frame's product is f64,
 * the quotient f32) */
int svi_fastblend_running_mean(const void* frame, int32_t frame_type, double s, const float* result, float divisor,
                               int64_t n_pix, double* out, void* stream);
/* out uint8 [n][3] = a clipped to [0, 255] and truncated toward zero, a SVI_FASTBLEND_U8 / _F32 (f32 [n][4]) or
 * SVI_FASTBLEND_F64 (f64 [n][4]) */
int svi_fastblend_to_u8(const void* a, int32_t a_type, int64_t n_pix, uint8_t* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SVI_B200_FASTBLEND_MODES_H_ */
