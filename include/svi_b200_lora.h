/*
 * svi_b200_lora.h — unmerged LoRA adapters on the DiT GEMM of libsvi_b200.so (the same library as svi_b200.h).
 *
 * The reference applies a LoRA by merging it into the weight (diffsynth/models/lora.py, W += alpha B A): switching adapters
 * then means reloading the model, and on an FP8 (e4m3) model the merged weight is rounded back to 3 mantissa bits.  This
 * entry point keeps W as it is and adds the adapter as a second K segment of the same GEMM, ahead of the epilogue:
 *
 *     out = epilogue( A[M,K] W[N,K]^T  +  U[:, g(n) R : g(n) R + R] B[N,R]^T ),   g(n) = n / group_cols (0 if group_cols == 0)
 *
 * U = alpha x A_lora^T is the adapter's down-projection, already scaled (one svi_gemm_bf16 with the alphas as `gate`);
 * several adapters are stacked along R.  With group_cols > 0 one launch covers a fused projection whose column groups have
 * their own adapters (q|k|v: 3 groups of d columns, U holding the three groups' down-projections side by side).
 * Conventions as in svi_b200.h.  A separate header so that svi_gemm_epilogue keeps its size and layout.
 */
#ifndef SVI_B200_LORA_H_
#define SVI_B200_LORA_H_

#include <stdint.h>

#include "svi_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct svi_gemm_lora {
  const void* U;      /* [M, ldu] bf16, 16-byte aligned; ldu >= groups * R, ldu % 8 == 0 */
  int64_t ldu;
  const void* B;      /* [N, ldb] bf16, 16-byte aligned (the up-projection, rank columns zero-padded to R); ldb >= R, % 8 == 0 */
  int64_t ldb;
  int32_t R;          /* rank columns per group, a positive multiple of 64 */
  int32_t group_cols; /* 0: one group; else a multiple of 128 that divides N */
} svi_gemm_lora;

/*
 * svi_gemm_bf16 with the LoRA segment above: the same arguments and checks, W bf16 or e4m3 (ep->w_e4m3), U and B always
 * bf16.  The epilogue is that of svi_gemm_bf16 (bias, activation, sums of squares, gate, residual all see the LoRA term);
 * act must be SVI_ACT_NONE or SVI_ACT_GELU_TANH, and the LayerNorm fold (ln_* / a_next) must be off.  With K % 64 == 0 and
 * one group the result is bit-identical to svi_gemm_bf16 on [A | U] and [W | B] (the same k-blocks in the same order).
 * Replaces the merged LoRA weights of lora.py:200-267 on the q, k, v, o, ffn.0 and ffn.2 projections of every block
 * (wan_video_dit.py:227-229,242,272-303,334-335,372-373).
 */
int svi_gemm_lora_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, int32_t M, int32_t N, int32_t K,
                       const svi_gemm_epilogue* ep, const svi_gemm_lora* lora, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SVI_B200_LORA_H_ */
