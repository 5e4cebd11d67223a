// The cross-attention quality scorers' row kernels (include/svi_b200_reward.h): BERT's post-LN LayerNorm with both
// outputs, the BLIP ViT's embedding sum, SwiGLU, rotate-half RoPE, MPS's condition mask and the folded ImageReward head.
// Their attention (svi_reward_attn) shares the wgmma kernel of quality_kernels.cu.
#include "common.cuh"
#include "../../include/svi_b200_reward.h"

namespace svi {
namespace reward {

constexpr int kRowThreads = 256;
constexpr int kRowValues = 8;       // values per thread: D <= 2048

// deterministic block sum: per-thread partials, a shuffle tree per warp, then the warp sums in warp order
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
  return s;
}

__global__ void __launch_bounds__(kRowThreads)
layernorm_kernel(const float* x, int D, float eps, const float* __restrict__ gamma, const float* __restrict__ beta, float* y,
                 __nv_bfloat16* __restrict__ yb) {
  __shared__ float red[kRowThreads / 32];
  const long long row = blockIdx.x;
  float v[kRowValues];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < kRowValues; ++j) {
    const int c = threadIdx.x + j * kRowThreads;
    v[j] = c < D ? x[row * D + c] : 0.f;
    s += v[j];
  }
  const float mean = block_sum(s, red) / D;       // every read of x is before this barrier, so y may be x
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < kRowValues; ++j) {
    const int c = threadIdx.x + j * kRowThreads;
    const float d = c < D ? v[j] - mean : 0.f;
    q += d * d;
  }
  const float rstd = rsqrtf(block_sum(q, red) / D + eps);
#pragma unroll
  for (int j = 0; j < kRowValues; ++j) {
    const int c = threadIdx.x + j * kRowThreads;
    if (c < D) {
      const float o = (v[j] - mean) * rstd * gamma[c] + beta[c];
      y[row * D + c] = o;
      yb[row * D + c] = __float2bfloat16_rn(o);
    }
  }
}

__global__ void embed_kernel(const float* __restrict__ patch, const float* __restrict__ cls, const float* __restrict__ pos,
                             int np, int D, float* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long row = i / D;
  const int c = (int)(i % D);
  const long long b = row / (np + 1);
  const int tok = (int)(row % (np + 1));
  const float v = tok == 0 ? cls[c] : patch[(b * np + tok - 1) * D + c];
  out[i] = v + pos[(long long)tok * D + c];
}

__global__ void swiglu_kernel(const float* __restrict__ x, long long ldx, int F, __nv_bfloat16* __restrict__ y, long long ldy,
                              long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long m = i / F;
  const int c = (int)(i % F);
  const float a = x[m * ldx + c], g = x[m * ldx + F + c];
  y[m * ldy + c] = __float2bfloat16_rn(__fmul_rn(__fdiv_rn(g, __fadd_rn(1.f, expf(-g))), a));
}

__global__ void rope_kernel(__nv_bfloat16* __restrict__ x, long long ldx, int L, int heads, const float* __restrict__ cs,
                            const float* __restrict__ sn, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int d = (int)(i % 32);
  const long long hm = i / 32;
  const int h = (int)(hm % heads);
  const long long m = hm / heads;
  const int p = (int)(m % L);
  __nv_bfloat16* t = x + m * ldx + h * 64;
  const float t1 = __bfloat162float(t[d]), t2 = __bfloat162float(t[d + 32]);
  const float c = cs[p * 32 + d], s = sn[p * 32 + d];
  t[d] = __float2bfloat16_rn(__fadd_rn(__fmul_rn(t1, c), __fmul_rn(-t2, s)));
  t[d + 32] = __float2bfloat16_rn(__fadd_rn(__fmul_rn(t2, c), __fmul_rn(t1, s)));
}

__global__ void __launch_bounds__(kRowThreads)
cond_sim_kernel(const float* __restrict__ text, const float* __restrict__ cond, int Lc, int E, float* __restrict__ sim) {
  __shared__ float red[kRowThreads / 32];
  const float* t = text + (long long)blockIdx.x * E;
  float best = -INFINITY;
  for (int j = 0; j < Lc; ++j) {
    const float* cj = cond + (long long)j * E;
    float d = 0.f;
    for (int c = threadIdx.x; c < E; c += kRowThreads) d += t[c] * cj[c];
    best = fmaxf(best, block_sum(d, red));
  }
  if (threadIdx.x == 0) sim[blockIdx.x] = best;
}

__global__ void __launch_bounds__(kRowThreads)
cond_mask_kernel(float* ratio, int Lt, float threshold, uint8_t* __restrict__ keep) {
  __shared__ float mx;
  if (threadIdx.x == 0) {
    float m = ratio[0];
    for (int i = 1; i < Lt; ++i) m = fmaxf(m, ratio[i]);
    mx = m;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < Lt; i += kRowThreads) {
    const float r = __fdiv_rn(ratio[i], mx);
    ratio[i] = r;
    keep[i] = r > threshold;
  }
}

__global__ void __launch_bounds__(kRowThreads)
head_kernel(const float* __restrict__ x, long long ld_seq, int E, const float* __restrict__ w, float bias, float* __restrict__ out) {
  __shared__ float red[kRowThreads / 32];
  const float* r = x + blockIdx.x * ld_seq;
  float d = 0.f;
  for (int c = threadIdx.x; c < E; c += kRowThreads) d += r[c] * w[c];
  d = block_sum(d, red);
  if (threadIdx.x == 0) out[blockIdx.x] = d + bias;
}

inline bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }
inline bool overlap(const void* a, size_t na, const void* b, size_t nb) {
  const char *pa = static_cast<const char*>(a), *pb = static_cast<const char*>(b);
  return pa < pb + nb && pb < pa + na;
}
inline unsigned blocks_for(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

}  // namespace reward
}  // namespace svi

using namespace svi;
using namespace svi::reward;

extern "C" int svi_reward_layernorm(const float* x, int32_t M, int32_t D, float eps, const float* gamma, const float* beta,
                                    float* y, void* yb, void* stream) {
  SVI_REQUIRE(x && gamma && beta && y && yb, "svi_reward_layernorm: null pointer");
  SVI_REQUIRE(M >= 1 && D >= 4 && D % 4 == 0 && D <= kRowValues * kRowThreads,
              "svi_reward_layernorm: need M >= 1 and D a multiple of 4 in [4, %d]", kRowValues * kRowThreads);
  SVI_REQUIRE(eps > 0.f, "svi_reward_layernorm: eps must be positive");
  SVI_REQUIRE(!overlap(yb, (size_t)M * D * 2, x, (size_t)M * D * 4) && !overlap(yb, (size_t)M * D * 2, y, (size_t)M * D * 4),
              "svi_reward_layernorm: yb overlaps x or y");
  SVI_REQUIRE(y == x || !overlap(y, (size_t)M * D * 4, x, (size_t)M * D * 4), "svi_reward_layernorm: y partly overlaps x");
  layernorm_kernel<<<(unsigned)M, kRowThreads, 0, static_cast<cudaStream_t>(stream)>>>(x, D, eps, gamma, beta, y,
                                                                                       static_cast<__nv_bfloat16*>(yb));
  SVI_CUDA_LAUNCH_CHECK("svi_reward_layernorm");
  return SVI_OK;
}

extern "C" int svi_reward_embed(const float* patch, const float* cls, const float* pos, int32_t B, int32_t np, int32_t D,
                                float* out, void* stream) {
  SVI_REQUIRE(patch && cls && pos && out, "svi_reward_embed: null pointer");
  SVI_REQUIRE(B >= 1 && np >= 1 && D >= 1, "svi_reward_embed: need B, np, D >= 1");
  const long long n = (long long)B * (np + 1) * D;
  SVI_REQUIRE(!overlap(out, (size_t)n * 4, patch, (size_t)B * np * D * 4), "svi_reward_embed: out overlaps patch");
  embed_kernel<<<blocks_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(patch, cls, pos, np, D, out, n);
  SVI_CUDA_LAUNCH_CHECK("svi_reward_embed");
  return SVI_OK;
}

extern "C" int svi_reward_swiglu(const float* x, int64_t ldx, int32_t M, int32_t F, void* y, int64_t ldy, void* stream) {
  SVI_REQUIRE(x && y, "svi_reward_swiglu: null pointer");
  SVI_REQUIRE(M >= 1 && F >= 1 && ldx >= 2LL * F && ldy >= F, "svi_reward_swiglu: need M, F >= 1, ldx >= 2F and ldy >= F");
  const long long n = (long long)M * F;
  swiglu_kernel<<<blocks_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, ldx, F, static_cast<__nv_bfloat16*>(y),
                                                                                   ldy, n);
  SVI_CUDA_LAUNCH_CHECK("svi_reward_swiglu");
  return SVI_OK;
}

extern "C" int svi_reward_rope(void* x, int64_t ldx, int32_t M, int32_t L, int32_t heads, const float* cos, const float* sin,
                               void* stream) {
  SVI_REQUIRE(x && cos && sin, "svi_reward_rope: null pointer");
  SVI_REQUIRE(M >= 1 && L >= 1 && heads >= 1 && ldx >= 64LL * heads, "svi_reward_rope: need M, L, heads >= 1 and ldx >= 64 heads");
  const long long n = (long long)M * heads * 32;
  rope_kernel<<<blocks_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<__nv_bfloat16*>(x), ldx, L, heads,
                                                                                 cos, sin, n);
  SVI_CUDA_LAUNCH_CHECK("svi_reward_rope");
  return SVI_OK;
}

extern "C" int svi_reward_cond_mask(const float* text, int32_t Lt, const float* cond, int32_t Lc, int32_t E, float threshold,
                                    float* ratio, uint8_t* keep, void* stream) {
  SVI_REQUIRE(text && cond && ratio && keep, "svi_reward_cond_mask: null pointer");
  SVI_REQUIRE(Lt >= 1 && Lt <= 65535 && Lc >= 1 && E >= 1, "svi_reward_cond_mask: need 1 <= Lt <= 65535, Lc, E >= 1");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cond_sim_kernel<<<(unsigned)Lt, kRowThreads, 0, st>>>(text, cond, Lc, E, ratio);
  SVI_CUDA_LAUNCH_CHECK("svi_reward_cond_mask");
  cond_mask_kernel<<<1, kRowThreads, 0, st>>>(ratio, Lt, threshold, keep);
  SVI_CUDA_LAUNCH_CHECK("svi_reward_cond_mask");
  return SVI_OK;
}

extern "C" int svi_reward_head(const float* x, int64_t ldx, int32_t B, int32_t L, int32_t E, const float* w, float bias,
                               float* out, void* stream) {
  SVI_REQUIRE(x && w && out, "svi_reward_head: null pointer");
  SVI_REQUIRE(B >= 1 && L >= 1 && E >= 1 && ldx >= E, "svi_reward_head: need B, L, E >= 1 and ldx >= E");
  head_kernel<<<(unsigned)B, kRowThreads, 0, static_cast<cudaStream_t>(stream)>>>(x, (long long)L * ldx, E, w, bias, out);
  SVI_CUDA_LAUNCH_CHECK("svi_reward_head");
  return SVI_OK;
}
