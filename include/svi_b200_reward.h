/*
 * svi_b200_reward.h — the cross-attention quality scorers (diffsynth/extensions/ImageQualityMetric: ImageReward, MPS) on
 * libsvi_b200.so (the same library as svi_b200.h).
 *
 * ImageReward runs a BLIP ViT-L/16 over a batch of images and a BERT whose every layer cross-attends from the prompt's
 * tokens to one image's 197 ViT rows; MPS runs a CLIP ViT-H/14 and text tower and a 4-layer cross model whose 257 image
 * rows per image attend to the prompt's 77 rows (one shared K/V head, keys masked by their similarity to a condition
 * prompt), then to themselves (multi-query, rotary positions).  Every matrix product is svi_gemm_bf16 and the pre-LN
 * LayerNorms are svi_layernorm_modulate; these entry points are the rest:
 *
 *   svi_reward_attn        softmax(Q K^T * scale, masked keys excluded) V: Lq query rows against Lk key rows per
 *                          sequence (each <= SVI_QUALITY_MAX_L), head width 64, K/V per head or one shared head, K/V and
 *                          mask per sequence or shared by all; the wgmma kernel and numerics of svi_quality_attn
 *   svi_reward_layernorm   LayerNorm rows f32 -> f32 (in place allowed) and the same values rounded to bf16 (BERT's
 *                          post-LN: the residual stream and the next GEMM's operand)
 *   svi_reward_embed       CLS row + patch-GEMM rows + position embedding -> f32 residual stream (no LayerNorm)
 *   svi_reward_swiglu      bf16(silu(g) * a) of f32 [a | g]
 *   svi_reward_rope        rotate-half rotary embedding of bf16 64-wide heads, in place, from cos / sin tables
 *   svi_reward_cond_mask   MPS's condition mask: per text row, max over condition rows of the dot product, over the
 *                          largest such value, compared with a threshold
 *   svi_reward_head        w . x + b of row 0 of each sequence (the folded ImageReward head)
 *
 * Layouts are row-major; leading dimensions are in elements.  No kernel uses atomics, sums run in a fixed order, and
 * each output row depends only on its own sequence or image: a frame gives the same bytes whatever batch it is scored in.
 * Conventions as in svi_b200.h: 0 on success, a negative status (and svi_last_error) on a rejected argument, in which
 * case nothing is launched; every launch is on `stream`.
 * A separate header so that svi_b200.h, its ABI version and svi_b200_quality.h stay as they are.
 */
#ifndef SVI_B200_REWARD_H_
#define SVI_B200_REWARD_H_

#include <stdint.h>

#include "svi_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Sequence b (0 <= b < batch): query rows [b*Lq, (b+1)*Lq) of Q and O, key rows [b*kv_batch_stride,
 * b*kv_batch_stride + Lk) of K and V (kv_batch_stride 0: every sequence reads the same keys).  Query head h is at columns
 * [64h, 64h + 64) of Q and O and reads K/V head h (kv_heads == num_heads) or K/V head 0 (kv_heads == 1).  key_mask (may
 * be NULL) uint8 [..][Lk]: key j of sequence b takes part iff key_mask[b*mask_batch_stride + j] != 0; every query row
 * needs at least one such key.  1 <= Lq, Lk <= SVI_QUALITY_MAX_L; the strides are 0 or >= Lk; ld* are even and cover
 * the heads; pointers 4-byte aligned; O may not overlap Q, K, V.
 * Per row as svi_quality_attn: s = q.k in fp32 (bf16 products), p = exp2((s - max) * scale * log2(e)) in fp32, P rounded
 * to bf16 for P V, the row sum of the unrounded p, O = (P V) / sum. */
int svi_reward_attn(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* O,
                    int64_t ldo, int32_t batch, int32_t Lq, int32_t Lk, int32_t num_heads, int32_t kv_heads,
                    int64_t kv_batch_stride, const uint8_t* key_mask, int64_t mask_batch_stride, float scale,
                    void* stream);

/* y f32 [M][D] = LN(x) * gamma + beta (biased variance, eps, fp32 statistics in a fixed order), yb bf16 [M][D] =
 * bf16_rn(y).  x, y, yb contiguous; y may be x (in place); D % 4 == 0, D <= 2048. */
int svi_reward_layernorm(const float* x, int32_t M, int32_t D, float eps, const float* gamma, const float* beta, float* y,
                         void* yb, void* stream);

/* out f32 [B*(1+np)][D]: row b*(1+np) = cls + pos[0], row b*(1+np) + 1 + p = patch[b*np + p] + pos[1 + p].
 * patch f32 [B*np][D], cls f32 [D], pos f32 [1+np][D]; out may not overlap patch. */
int svi_reward_embed(const float* patch, const float* cls, const float* pos, int32_t B, int32_t np, int32_t D, float* out,
                     void* stream);

/* y[m][n] = bf16_rn(a * g / (1 + exp(-g))) for a = x[m][n], g = x[m][F + n], n < F; x f32 [M][>= 2F], y bf16 [M][>= F]. */
int svi_reward_swiglu(const float* x, int64_t ldx, int32_t M, int32_t F, void* y, int64_t ldy, void* stream);

/* In place on x bf16 [M][ldx]: for every row m (position p = m % L) and head h < heads (columns [64h, 64h + 64)),
 * t' = t * cos + rotate_half(t) * sin with rotate_half(t) = [-t[32:64], t[0:32]] and cos, sin f32 [L][32] indexed by
 * (p, d % 32); computed in fp32 from the bf16 t, rounded to bf16. */
int svi_reward_rope(void* x, int64_t ldx, int32_t M, int32_t L, int32_t heads, const float* cos, const float* sin,
                    void* stream);

/* text f32 [Lt][E], cond f32 [Lc][E]: sim[i] = max_j text[i] . cond[j]; ratio f32 [Lt] = sim[i] / max_i sim[i];
 * keep uint8 [Lt] = ratio[i] > threshold.  Dot products and maxima in a fixed order. */
int svi_reward_cond_mask(const float* text, int32_t Lt, const float* cond, int32_t Lc, int32_t E, float threshold,
                         float* ratio, uint8_t* keep, void* stream);

/* out f32 [B] = sum_c w[c] * x[b*L*ldx + c] + bias (row 0 of each sequence of L rows), c < E, fixed-order sums. */
int svi_reward_head(const float* x, int64_t ldx, int32_t B, int32_t L, int32_t E, const float* w, float bias, float* out,
                    void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SVI_B200_REWARD_H_ */
