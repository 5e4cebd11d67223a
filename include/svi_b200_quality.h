/*
 * svi_b200_quality.h — image-text quality scoring (diffsynth/extensions/ImageQualityMetric: CLIP score, HPSv2 / v2.1,
 * PickScore, aesthetic score) on libsvi_b200.so (the same library as svi_b200.h).
 *
 * The scorers run a CLIP vision tower (ViT-H/14 or ViT-L/14) over a whole batch of images and a CLIP text tower over the
 * prompt.  Every matrix product is svi_gemm_bf16 and the LayerNorms are svi_layernorm_modulate; these entry points are
 * the rest:
 *
 *   svi_quality_attn          softmax(Q K^T * scale [+ causal mask]) V for `batch` independent sequences of L <= 320
 *                             tokens, head width 64 or 80, bf16 operands on wgmma tensor cores, fp32 softmax
 *                             statistics; one launch covers every sequence and head of a layer
 *   svi_quality_stage_pixels  preprocessed images f32 [B][3][S][S] -> per-channel (x - mean) / std -> the patch GEMM's
 *                             bf16 rows [B * (S/P)^2][kpad] in the Conv2d weight's (c, py, px) order, zero K padding
 *   svi_quality_embed_ln      CLS row + patch-GEMM rows + position embedding -> pre-LayerNorm -> f32 residual stream
 *   svi_quality_quick_gelu    y = x * sigmoid(1.702 x), f32 -> bf16 (the MLP activation of quick-GELU towers)
 *   svi_quality_pool          one row per sequence: the CLS row, the row of argmax(ids), or the first row whose id is
 *                             eos_id
 *   svi_quality_score         L2-normalised image features . L2-normalised text features -> [B][T] cosines, and the
 *                             folded aesthetic head w . x_hat + b -> [B]
 *
 * Layouts are row-major; leading dimensions are in elements.  No kernel uses atomics, and each output row depends only
 * on its own sequence or image: a frame gives the same bytes whatever batch it is scored in.
 * Conventions as in svi_b200.h: 0 on success, a negative status (and svi_last_error) on a rejected argument, in which
 * case nothing is launched; every launch is on `stream`.
 * A separate header so that svi_b200.h and its ABI version stay as they are.
 */
#ifndef SVI_B200_QUALITY_H_
#define SVI_B200_QUALITY_H_

#include <stdint.h>

#include "svi_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define SVI_QUALITY_MAX_L 320   /* longest sequence svi_quality_attn takes (257 image tokens, 77 text tokens) */

/* Rows [b*L, (b+1)*L) of Q, K, V (bf16, head h at columns [h*head_dim, (h+1)*head_dim)) form sequence b; O (bf16) is
 * written in the same layout.  head_dim is 64 or 80; 1 <= L <= SVI_QUALITY_MAX_L; causal != 0 masks key j > query i.
 * ldq, ldk, ldv, ldo are even and >= num_heads * head_dim; the pointers are 4-byte aligned; O may not overlap Q, K, V.
 * Per row: s = q.k in fp32 (bf16 products), p = exp2((s - max) * scale * log2(e)) in fp32, P rounded to bf16 for
 * P V, the row sum of the unrounded p, O = (P V) / sum. */
int svi_quality_attn(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* O,
                     int64_t ldo, int32_t batch, int32_t L, int32_t num_heads, int32_t head_dim, float scale,
                     int32_t causal, void* stream);

/* px f32 [B][3][S][S] (contiguous), mean_std f32 [6] device memory (mean of R, G, B, then std of R, G, B) ->
 * out bf16 [B * (S/P)^2][kpad]: row b*(S/P)^2 + gy*(S/P) + gx, column c*P*P + py*P + px =
 * bf16_rn((px[b][c][gy*P + py][gx*P + px] - mean[c]) / std[c]) (IEEE subtraction and division), columns >= 3*P*P zero.
 * S % P == 0, kpad % 8 == 0, kpad >= 3*P*P. */
int svi_quality_stage_pixels(const float* px, int32_t B, int32_t S, int32_t P, const float* mean_std, void* out,
                             int32_t kpad, void* stream);

/* out f32 [B*(1+np)][D]: row b*(1+np) = LN(cls + pos[0]), row b*(1+np) + 1 + p = LN(patch[b*np + p] + pos[1 + p]),
 * LN = LayerNorm over D (biased variance, eps) * gamma + beta.  patch f32 [B*np][D], cls f32 [D], pos f32 [1+np][D].
 * D % 4 == 0, D <= 2048; out may not overlap patch. */
int svi_quality_embed_ln(const float* patch, const float* cls, const float* pos, int32_t B, int32_t np, int32_t D,
                         float eps, const float* gamma, const float* beta, float* out, void* stream);

/* y[m][n] = bf16_rn(x * (1 / (1 + exp(-1.702 x)))) for x = x[m][n] f32, n < N; ldx, ldy >= N. */
int svi_quality_quick_gelu(const float* x, int64_t ldx, int32_t M, int32_t N, void* y, int64_t ldy, void* stream);

#define SVI_POOL_FIRST 0   /* row 0 of each sequence (the CLS token) */
#define SVI_POOL_ARGMAX 1  /* the first row holding the largest id (open_clip's EOT; transformers' eos_token_id == 2 rule) */
#define SVI_POOL_EOS 2     /* the first row whose id == eos_id, row 0 if none (transformers' rule otherwise) */
/* out f32 [n_seq][D] = row r_s of sequence s of x f32 [n_seq*L][ldx]; ids int64 [n_seq][L] (NULL for SVI_POOL_FIRST). */
int svi_quality_pool(const float* x, int64_t ldx, int32_t n_seq, int32_t L, int32_t D, const int64_t* ids, int32_t mode,
                     int64_t eos_id, float* out, void* stream);

/* img f32 [B][E], txt f32 [T][E] (T may be 0, txt then NULL).  x_hat = x / max(||x||_2, 1e-12), sums in a fixed order.
 * cos f32 [B][T] = x_hat_img[b] . x_hat_txt[t] (NULL when T == 0); aes f32 [B] = w . x_hat_img[b] + bias when w != NULL
 * (w f32 [E]).  1 <= E <= 4096. */
int svi_quality_score(const float* img, int32_t B, const float* txt, int32_t T, int32_t E, const float* w, float bias,
                      float* cos, float* aes, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SVI_B200_QUALITY_H_ */
