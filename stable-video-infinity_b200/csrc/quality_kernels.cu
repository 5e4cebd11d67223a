// Image-text quality scoring: the CLIP towers' batched short-sequence attention and their staging, pooling and scoring
// kernels (include/svi_b200_quality.h), and the same attention with separate query / key lengths, a shared K/V head and a
// key mask for the cross-attention scorers (svi_reward_attn, include/svi_b200_reward.h).  The projections and MLPs are
// svi_gemm_bf16 calls, the block LayerNorms svi_layernorm_modulate.
//
// Attention.  One CTA of four warps takes 64 query rows of one head of one sequence; the grid covers every sequence and
// head of a layer in one launch.  K and V^T of the sequence's first `kv_len` keys are staged in shared memory once, both
// as K-major wgmma B operands in core-matrix order (no swizzle); the warpgroup keeps its 64 query rows as register A
// fragments (wgmma RS form) and walks the keys in chunks of 64 with an online softmax (fp32 max and sum, bf16 P, which
// goes back into wgmma as the register A operand of P V).  Causal CTAs stage and visit only the keys up to their last
// query row.  With a key mask, masked keys get a score of -inf like keys past Lk; a query row whose keys seen so far are
// all masked keeps a running max of -inf, and its rescale factors and probabilities are taken against 0 instead (they
// are all 0), so a fully masked chunk ahead of the first kept key contributes nothing.
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/svi_b200_quality.h"
#include "../../include/svi_b200_reward.h"

namespace svi {
namespace quality {

constexpr int kAttnThreads = 128;   // 4 warps x 16 query rows
constexpr int kBQ = 64;
constexpr int kBK = 64;

// D[64 x N] (+)= A[64 x 16] (registers, the m64k16 fragment of wgmma.cuh) * B[16 x N] (K-major, no swizzle)
template <int N> struct WgmmaRS;

template <> struct WgmmaRS<64> {
  static __device__ __forceinline__ void run(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
  }
};

template <> struct WgmmaRS<80> {
  static __device__ __forceinline__ void run(float (&d)[40], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %45, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, {%40, %41, %42, %43}, %44, p, 1, 1, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
  }
};

// no-swizzle K-major descriptor: 8-row x 16-byte core matrices, LBO = next core matrix along K, SBO = next along N
__device__ __forceinline__ uint64_t desc_interleave(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}

// byte offset of element (n, k) of a K-major operand of `kdim` columns in core-matrix order
__device__ __forceinline__ uint32_t cm_offset(int n, int k, int kdim) {
  return (uint32_t)((n >> 3) * (kdim * 16) + (k >> 3) * 128 + (n & 7) * 16 + (k & 7) * 2);
}

__host__ __device__ constexpr int round_up(int x, int m) { return (x + m - 1) / m * m; }

template <int HD>
__host__ __device__ constexpr size_t attn_smem_bytes(int kv_pad) {
  return (size_t)kv_pad * HD * 2 * 2 + kv_pad;   // K [kv_pad][HD] and V^T [HD][kv_pad], bf16; the key mask, one byte a key
}

// Sequence b: query rows [b*Lq, (b+1)*Lq) of Q and O, key rows [b*kv_stride, b*kv_stride + Lk) of K and V, query head h
// reading K/V head h (kv_shared == 0) or 0 (kv_shared != 0), mask bytes mask[b*mask_stride + key] (mask may be null).
template <int HD>
__global__ void __launch_bounds__(kAttnThreads)
attn_kernel(const __nv_bfloat16* __restrict__ Q, long long ldq, const __nv_bfloat16* __restrict__ K, long long ldk,
            const __nv_bfloat16* __restrict__ V, long long ldv, __nv_bfloat16* __restrict__ O, long long ldo, int Lq,
            int Lk, long long kv_stride, int kv_shared, const uint8_t* __restrict__ mask, long long mask_stride,
            float scale_log2, int causal) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int q0 = blockIdx.x * kBQ, h = blockIdx.y, b = blockIdx.z;
  const int kv_len = causal ? min(Lk, q0 + kBQ) : Lk;
  const int kv_pad = round_up(kv_len, kBK);
  unsigned char* Ks = smem;                                  // (n = key, k = d), K-major
  unsigned char* Vt = smem + (size_t)kv_pad * HD * 2;        // (n = d, k = key), K-major
  unsigned char* Ms = smem + (size_t)kv_pad * HD * 4;        // 1 = key kept
  const long long row0 = (long long)b * Lq, krow0 = (long long)b * kv_stride;
  const int hk = kv_shared ? 0 : h;

  if (mask != nullptr)
    for (int j = threadIdx.x; j < kv_len; j += kAttnThreads) Ms[j] = mask[b * mask_stride + j] != 0;
  // stage K and V^T in core-matrix order; keys [kv_len, kv_pad) are zero (their P is zero, and 0 * garbage could be NaN)
  for (int i = threadIdx.x; i < kv_pad * (HD / 2); i += kAttnThreads) {
    const int j = i / (HD / 2), c = (i % (HD / 2)) * 2;
    uint32_t kw = 0u, vw = 0u;
    if (j < kv_len) {
      kw = *reinterpret_cast<const uint32_t*>(K + (krow0 + j) * ldk + hk * HD + c);
      vw = *reinterpret_cast<const uint32_t*>(V + (krow0 + j) * ldv + hk * HD + c);
    }
    *reinterpret_cast<uint32_t*>(Ks + cm_offset(j, c, HD)) = kw;
    const __nv_bfloat162 v2 = *reinterpret_cast<const __nv_bfloat162*>(&vw);
    *reinterpret_cast<__nv_bfloat16*>(Vt + cm_offset(c, j, kv_pad)) = v2.x;
    *reinterpret_cast<__nv_bfloat16*>(Vt + cm_offset(c + 1, j, kv_pad)) = v2.y;
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> wgmma operand reads
  __syncthreads();

  // every warp runs every chunk (wgmma is warpgroup-wide); rows past Lq compute on zero Q and store nothing
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32, g = lane / 4, t = lane % 4;
  const int r_lo = q0 + warp * 16 + g, r_hi = r_lo + 8;

  uint32_t qf[HD / 16][4];
#pragma unroll
  for (int kk = 0; kk < HD / 16; ++kk) {
    const int c = h * HD + kk * 16 + t * 2;
    qf[kk][0] = r_lo < Lq ? *reinterpret_cast<const uint32_t*>(Q + (row0 + r_lo) * ldq + c) : 0u;
    qf[kk][1] = r_hi < Lq ? *reinterpret_cast<const uint32_t*>(Q + (row0 + r_hi) * ldq + c) : 0u;
    qf[kk][2] = r_lo < Lq ? *reinterpret_cast<const uint32_t*>(Q + (row0 + r_lo) * ldq + c + 8) : 0u;
    qf[kk][3] = r_hi < Lq ? *reinterpret_cast<const uint32_t*>(Q + (row0 + r_hi) * ldq + c + 8) : 0u;
  }

  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
  const uint32_t ks_addr = smem_u32(Ks), vt_addr = smem_u32(Vt);

  for (int kc = 0; kc < kv_pad / kBK; ++kc) {
    float s[kBK / 2];
#pragma unroll
    for (int i = 0; i < kBK / 2; ++i) s[i] = 0.f;
    wgmma_fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
      WgmmaRS<kBK>::run(s, qf[kk], desc_interleave(ks_addr + cm_offset(kc * kBK, kk * 16, HD), 128, HD * 16), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);

    float cm_lo = -INFINITY, cm_hi = -INFINITY;
#pragma unroll
    for (int n = 0; n < kBK / 8; ++n) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int key = kc * kBK + n * 8 + t * 2 + e;
        const bool dropped = key >= Lk || (mask != nullptr && !Ms[key]);
        if (dropped || (causal && key > r_lo)) s[4 * n + e] = -INFINITY;
        if (dropped || (causal && key > r_hi)) s[4 * n + 2 + e] = -INFINITY;
        cm_lo = fmaxf(cm_lo, s[4 * n + e]);
        cm_hi = fmaxf(cm_hi, s[4 * n + 2 + e]);
      }
    }
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) {
      cm_lo = fmaxf(cm_lo, __shfl_xor_sync(0xffffffffu, cm_lo, off));
      cm_hi = fmaxf(cm_hi, __shfl_xor_sync(0xffffffffu, cm_hi, off));
    }
    // without a key mask, key 0 is in chunk 0 and never masked, so the running max is finite from the first chunk on and
    // the reference point below is the running max itself
    const float mn_lo = fmaxf(m_lo, cm_lo), mn_hi = fmaxf(m_hi, cm_hi);
    const float ref_lo = mn_lo == -INFINITY ? 0.f : mn_lo, ref_hi = mn_hi == -INFINITY ? 0.f : mn_hi;
    const float a_lo = exp2f((m_lo - ref_lo) * scale_log2), a_hi = exp2f((m_hi - ref_hi) * scale_log2);
    m_lo = mn_lo;
    m_hi = mn_hi;
    l_lo *= a_lo;
    l_hi *= a_hi;
#pragma unroll
    for (int n = 0; n < HD / 8; ++n) {
      o[4 * n] *= a_lo; o[4 * n + 1] *= a_lo; o[4 * n + 2] *= a_hi; o[4 * n + 3] *= a_hi;
    }
    uint32_t pa[kBK / 16][4];
#pragma unroll
    for (int n = 0; n < kBK / 8; ++n) {
      const float p0 = exp2f((s[4 * n] - ref_lo) * scale_log2), p1 = exp2f((s[4 * n + 1] - ref_lo) * scale_log2);
      const float p2 = exp2f((s[4 * n + 2] - ref_hi) * scale_log2), p3 = exp2f((s[4 * n + 3] - ref_hi) * scale_log2);
      l_lo += p0 + p1;
      l_hi += p2 + p3;
      pa[n / 2][(n & 1) * 2] = pack_bf16x2(p0, p1);
      pa[n / 2][(n & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kBK / 16; ++kk)
      WgmmaRS<HD>::run(o, pa[kk], desc_interleave(vt_addr + cm_offset(0, kc * kBK + kk * 16, kv_pad), 128, kv_pad * 16), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
  }
#pragma unroll
  for (int off = 1; off < 4; off <<= 1) {
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, off);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, off);
  }
  const float inv_lo = 1.f / l_lo, inv_hi = 1.f / l_hi;
#pragma unroll
  for (int n = 0; n < HD / 8; ++n) {
    const int c = h * HD + n * 8 + t * 2;
    if (r_lo < Lq) *reinterpret_cast<uint32_t*>(O + (row0 + r_lo) * ldo + c) = pack_bf16x2(o[4 * n] * inv_lo, o[4 * n + 1] * inv_lo);
    if (r_hi < Lq) *reinterpret_cast<uint32_t*>(O + (row0 + r_hi) * ldo + c) = pack_bf16x2(o[4 * n + 2] * inv_hi, o[4 * n + 3] * inv_hi);
  }
}

template <int HD>
int launch_attn(const char* name, const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv,
                void* O, int64_t ldo, int batch, int Lq, int Lk, int heads, int64_t kv_stride, int kv_shared,
                const uint8_t* mask, int64_t mask_stride, float scale, int causal, cudaStream_t stream) {
  static bool attr_set = false;       // the largest plan's shared memory, allowed once per process
  if (!attr_set) {
    const cudaError_t e = cudaFuncSetAttribute(attn_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)attn_smem_bytes<HD>(round_up(SVI_QUALITY_MAX_L, kBK)));
    if (e != cudaSuccess) {
      set_last_error("%s: cudaFuncSetAttribute failed: %s", name, cudaGetErrorString(e));
      return SVI_ERR_DRIVER;
    }
    attr_set = true;
  }
  const dim3 grid((unsigned)((Lq + kBQ - 1) / kBQ), (unsigned)heads, (unsigned)batch);
  attn_kernel<HD><<<grid, kAttnThreads, attn_smem_bytes<HD>(round_up(Lk, kBK)), stream>>>(
      static_cast<const __nv_bfloat16*>(Q), ldq, static_cast<const __nv_bfloat16*>(K), ldk,
      static_cast<const __nv_bfloat16*>(V), ldv, static_cast<__nv_bfloat16*>(O), ldo, Lq, Lk, (long long)kv_stride,
      kv_shared, mask, (long long)mask_stride, scale * 1.4426950408889634f, causal);
  SVI_CUDA_LAUNCH_CHECK(name);
  return SVI_OK;
}

// ------------------------------------------------------------------------------------------------ staging and pooling
__global__ void stage_pixels_kernel(const float* __restrict__ px, int S, int P, int G, const float* __restrict__ ms,
                                    uint32_t* __restrict__ out, int kpad, long long n_pairs) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pairs) return;
  const int half = kpad / 2;
  const long long row = i / half;
  const int col = (int)(i % half) * 2;
  const long long b = row / (G * G);
  const int p = (int)(row % (G * G)), gy = p / G, gx = p % G;
  float v[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int k = col + e;
    v[e] = 0.f;
    if (k < 3 * P * P) {
      const int c = k / (P * P), r = k % (P * P), py = r / P, pxx = r % P;
      const float x = px[((b * 3 + c) * S + gy * P + py) * (long long)S + gx * P + pxx];
      v[e] = __fdiv_rn(__fsub_rn(x, ms[c]), ms[3 + c]);
    }
  }
  out[i] = pack_bf16x2(v[0], v[1]);
}

constexpr int kRowThreads = 256;

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
embed_ln_kernel(const float* __restrict__ patch, const float* __restrict__ cls, const float* __restrict__ pos, int np,
                int D, float eps, const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ out) {
  __shared__ float red[kRowThreads / 32];
  const long long row = blockIdx.x;
  const int b = (int)(row / (np + 1)), tok = (int)(row % (np + 1));
  const float* src = tok == 0 ? cls : patch + ((long long)b * np + tok - 1) * D;
  const float* pe = pos + (long long)tok * D;
  float v[8];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = threadIdx.x + j * kRowThreads;
    v[j] = c < D ? src[c] + pe[c] : 0.f;
    s += v[j];
  }
  const float mean = block_sum(s, red) / D;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = threadIdx.x + j * kRowThreads;
    const float d = c < D ? v[j] - mean : 0.f;
    q += d * d;
  }
  const float rstd = rsqrtf(block_sum(q, red) / D + eps);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = threadIdx.x + j * kRowThreads;
    if (c < D) out[row * D + c] = (v[j] - mean) * rstd * gamma[c] + beta[c];
  }
}

__global__ void quick_gelu_kernel(const float* __restrict__ x, long long ldx, int N, __nv_bfloat16* __restrict__ y,
                                  long long ldy, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long m = i / N;
  const int c = (int)(i % N);
  const float v = x[m * ldx + c];
  y[m * ldy + c] = __float2bfloat16_rn(v * (1.f / (1.f + expf(-1.702f * v))));
}

__global__ void pool_kernel(const float* __restrict__ x, long long ldx, int L, int D, const long long* __restrict__ ids,
                            int mode, long long eos_id, float* __restrict__ out) {
  const int s = blockIdx.x;
  int r = 0;
  if (mode == SVI_POOL_ARGMAX) {
    long long best = ids[(long long)s * L];
    for (int j = 1; j < L; ++j) {
      const long long v = ids[(long long)s * L + j];
      if (v > best) best = v, r = j;
    }
  } else if (mode == SVI_POOL_EOS) {
    for (int j = 0; j < L; ++j)
      if (ids[(long long)s * L + j] == eos_id) { r = j; break; }
  }
  const float* src = x + ((long long)s * L + r) * ldx;
  for (int c = threadIdx.x; c < D; c += blockDim.x) out[(long long)s * D + c] = src[c];
}

__device__ __forceinline__ float row_inv_norm(const float* x, int E, float* red) {
  float q = 0.f;
  for (int c = threadIdx.x; c < E; c += blockDim.x) q += x[c] * x[c];
  return 1.f / fmaxf(sqrtf(block_sum(q, red)), 1e-12f);
}

__global__ void __launch_bounds__(kRowThreads)
score_kernel(const float* __restrict__ img, const float* __restrict__ txt, int T, int E, const float* __restrict__ w,
             float bias, float* __restrict__ cos, float* __restrict__ aes) {
  __shared__ float red[kRowThreads / 32];
  const int b = blockIdx.x;
  const float* xi = img + (long long)b * E;
  const float ni = row_inv_norm(xi, E, red);   // 1 / max(||x||, 1e-12)
  for (int t = 0; t < T; ++t) {
    const float* xt = txt + (long long)t * E;
    const float nt = row_inv_norm(xt, E, red);
    float d = 0.f;
    for (int c = threadIdx.x; c < E; c += blockDim.x) d += (xi[c] * ni) * (xt[c] * nt);
    d = block_sum(d, red);
    if (threadIdx.x == 0) cos[(long long)b * T + t] = d;
  }
  if (w != nullptr) {
    float d = 0.f;
    for (int c = threadIdx.x; c < E; c += blockDim.x) d += (xi[c] * ni) * w[c];
    d = block_sum(d, red);
    if (threadIdx.x == 0) aes[b] = d + bias;
  }
}

inline bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }
inline bool overlap(const void* a, size_t na, const void* b, size_t nb) {
  const char *pa = static_cast<const char*>(a), *pb = static_cast<const char*>(b);
  return pa < pb + nb && pb < pa + na;
}

}  // namespace quality
}  // namespace svi

using namespace svi;
using namespace svi::quality;

extern "C" int svi_quality_attn(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv,
                                void* O, int64_t ldo, int32_t batch, int32_t L, int32_t num_heads, int32_t head_dim,
                                float scale, int32_t causal, void* stream) {
  SVI_REQUIRE(Q && K && V && O, "svi_quality_attn: null pointer");
  SVI_REQUIRE(head_dim == 64 || head_dim == 80, "svi_quality_attn: head_dim %d is not implemented (64 or 80)", head_dim);
  SVI_REQUIRE(L >= 1 && L <= SVI_QUALITY_MAX_L, "svi_quality_attn: L = %d outside [1, %d]", L, SVI_QUALITY_MAX_L);
  SVI_REQUIRE(batch >= 1 && batch <= 65535 && num_heads >= 1 && num_heads <= 65535,
              "svi_quality_attn: batch %d / num_heads %d outside [1, 65535]", batch, num_heads);
  const int64_t w = (int64_t)num_heads * head_dim;
  SVI_REQUIRE(ldq >= w && ldk >= w && ldv >= w && ldo >= w, "svi_quality_attn: a leading dimension is below num_heads * head_dim = %lld",
              (long long)w);
  SVI_REQUIRE(ldq % 2 == 0 && ldk % 2 == 0 && ldv % 2 == 0 && ldo % 2 == 0, "svi_quality_attn: leading dimensions must be even");
  SVI_REQUIRE(aligned(Q, 4) && aligned(K, 4) && aligned(V, 4) && aligned(O, 4), "svi_quality_attn: pointers must be 4-byte aligned");
  SVI_REQUIRE(scale > 0.f && scale < 1e30f, "svi_quality_attn: scale must be positive and finite");
  const size_t rows = (size_t)batch * L;
  const size_t bo = ((rows - 1) * ldo + w) * 2;
  SVI_REQUIRE(!overlap(O, bo, Q, ((rows - 1) * ldq + w) * 2) && !overlap(O, bo, K, ((rows - 1) * ldk + w) * 2) &&
              !overlap(O, bo, V, ((rows - 1) * ldv + w) * 2), "svi_quality_attn: O overlaps Q, K or V");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const char* name = "svi_quality_attn";
  return head_dim == 64 ? launch_attn<64>(name, Q, ldq, K, ldk, V, ldv, O, ldo, batch, L, L, num_heads, L, 0, nullptr, 0,
                                          scale, causal != 0, st)
                        : launch_attn<80>(name, Q, ldq, K, ldk, V, ldv, O, ldo, batch, L, L, num_heads, L, 0, nullptr, 0,
                                          scale, causal != 0, st);
}

extern "C" int svi_reward_attn(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* O,
                               int64_t ldo, int32_t batch, int32_t Lq, int32_t Lk, int32_t num_heads, int32_t kv_heads,
                               int64_t kv_batch_stride, const uint8_t* key_mask, int64_t mask_batch_stride, float scale,
                               void* stream) {
  SVI_REQUIRE(Q && K && V && O, "svi_reward_attn: null pointer");
  SVI_REQUIRE(Lq >= 1 && Lq <= SVI_QUALITY_MAX_L && Lk >= 1 && Lk <= SVI_QUALITY_MAX_L,
              "svi_reward_attn: Lq = %d / Lk = %d outside [1, %d]", Lq, Lk, SVI_QUALITY_MAX_L);
  SVI_REQUIRE(batch >= 1 && batch <= 65535 && num_heads >= 1 && num_heads <= 65535,
              "svi_reward_attn: batch %d / num_heads %d outside [1, 65535]", batch, num_heads);
  SVI_REQUIRE(kv_heads == 1 || kv_heads == num_heads, "svi_reward_attn: kv_heads %d must be 1 or num_heads", kv_heads);
  SVI_REQUIRE(kv_batch_stride == 0 || kv_batch_stride >= Lk, "svi_reward_attn: kv_batch_stride must be 0 or >= Lk");
  SVI_REQUIRE(mask_batch_stride == 0 || mask_batch_stride >= Lk, "svi_reward_attn: mask_batch_stride must be 0 or >= Lk");
  const int64_t wq = (int64_t)num_heads * 64, wk = (int64_t)kv_heads * 64;
  SVI_REQUIRE(ldq >= wq && ldo >= wq && ldk >= wk && ldv >= wk,
              "svi_reward_attn: a leading dimension is below the heads' width (q, o: %lld; k, v: %lld)", (long long)wq,
              (long long)wk);
  SVI_REQUIRE(ldq % 2 == 0 && ldk % 2 == 0 && ldv % 2 == 0 && ldo % 2 == 0, "svi_reward_attn: leading dimensions must be even");
  SVI_REQUIRE(aligned(Q, 4) && aligned(K, 4) && aligned(V, 4) && aligned(O, 4), "svi_reward_attn: pointers must be 4-byte aligned");
  SVI_REQUIRE(scale > 0.f && scale < 1e30f, "svi_reward_attn: scale must be positive and finite");
  const size_t q_rows = (size_t)batch * Lq, k_rows = (size_t)(kv_batch_stride * (batch - 1) + Lk);
  const size_t bo = ((q_rows - 1) * ldo + wq) * 2;
  SVI_REQUIRE(!overlap(O, bo, Q, ((q_rows - 1) * ldq + wq) * 2) && !overlap(O, bo, K, ((k_rows - 1) * ldk + wk) * 2) &&
              !overlap(O, bo, V, ((k_rows - 1) * ldv + wk) * 2), "svi_reward_attn: O overlaps Q, K or V");
  return launch_attn<64>("svi_reward_attn", Q, ldq, K, ldk, V, ldv, O, ldo, batch, Lq, Lk, num_heads, kv_batch_stride,
                         kv_heads == 1, key_mask, mask_batch_stride, scale, 0, static_cast<cudaStream_t>(stream));
}

extern "C" int svi_quality_stage_pixels(const float* px, int32_t B, int32_t S, int32_t P, const float* mean_std, void* out,
                                        int32_t kpad, void* stream) {
  SVI_REQUIRE(px && mean_std && out, "svi_quality_stage_pixels: null pointer");
  SVI_REQUIRE(B >= 1 && P >= 1 && S >= P && S % P == 0 && S <= 4096, "svi_quality_stage_pixels: S must be a positive multiple of P");
  SVI_REQUIRE(kpad % 8 == 0 && kpad >= 3 * P * P, "svi_quality_stage_pixels: kpad must be a multiple of 8 and >= 3*P*P");
  SVI_REQUIRE(aligned(out, 4), "svi_quality_stage_pixels: out must be 4-byte aligned");
  const int G = S / P;
  const long long n_pairs = (long long)B * G * G * (kpad / 2);
  const int threads = 256;
  stage_pixels_kernel<<<(unsigned)((n_pairs + threads - 1) / threads), threads, 0, static_cast<cudaStream_t>(stream)>>>(
      px, S, P, G, mean_std, static_cast<uint32_t*>(out), kpad, n_pairs);
  SVI_CUDA_LAUNCH_CHECK("svi_quality_stage_pixels");
  return SVI_OK;
}

extern "C" int svi_quality_embed_ln(const float* patch, const float* cls, const float* pos, int32_t B, int32_t np,
                                    int32_t D, float eps, const float* gamma, const float* beta, float* out, void* stream) {
  SVI_REQUIRE(patch && cls && pos && gamma && beta && out, "svi_quality_embed_ln: null pointer");
  SVI_REQUIRE(B >= 1 && np >= 1 && D >= 4 && D % 4 == 0 && D <= 8 * kRowThreads,
              "svi_quality_embed_ln: need B, np >= 1 and D a multiple of 4 in [4, %d]", 8 * kRowThreads);
  SVI_REQUIRE(!overlap(out, (size_t)B * (np + 1) * D * 4, patch, (size_t)B * np * D * 4), "svi_quality_embed_ln: out overlaps patch");
  const long long rows = (long long)B * (np + 1);
  SVI_REQUIRE(rows < (1LL << 31), "svi_quality_embed_ln: too many rows");
  embed_ln_kernel<<<(unsigned)rows, kRowThreads, 0, static_cast<cudaStream_t>(stream)>>>(patch, cls, pos, np, D, eps, gamma,
                                                                                           beta, out);
  SVI_CUDA_LAUNCH_CHECK("svi_quality_embed_ln");
  return SVI_OK;
}

extern "C" int svi_quality_quick_gelu(const float* x, int64_t ldx, int32_t M, int32_t N, void* y, int64_t ldy, void* stream) {
  SVI_REQUIRE(x && y, "svi_quality_quick_gelu: null pointer");
  SVI_REQUIRE(M >= 1 && N >= 1 && ldx >= N && ldy >= N, "svi_quality_quick_gelu: need M, N >= 1 and ldx, ldy >= N");
  const long long n = (long long)M * N;
  const int threads = 256;
  quick_gelu_kernel<<<(unsigned)((n + threads - 1) / threads), threads, 0, static_cast<cudaStream_t>(stream)>>>(
      x, ldx, N, static_cast<__nv_bfloat16*>(y), ldy, n);
  SVI_CUDA_LAUNCH_CHECK("svi_quality_quick_gelu");
  return SVI_OK;
}

extern "C" int svi_quality_pool(const float* x, int64_t ldx, int32_t n_seq, int32_t L, int32_t D, const int64_t* ids,
                                int32_t mode, int64_t eos_id, float* out, void* stream) {
  SVI_REQUIRE(x && out, "svi_quality_pool: null pointer");
  SVI_REQUIRE(mode == SVI_POOL_FIRST || mode == SVI_POOL_ARGMAX || mode == SVI_POOL_EOS, "svi_quality_pool: bad mode %d", mode);
  SVI_REQUIRE(mode == SVI_POOL_FIRST || ids, "svi_quality_pool: mode %d needs ids", mode);
  SVI_REQUIRE(n_seq >= 1 && n_seq <= (1 << 30) && L >= 1 && D >= 1 && ldx >= D, "svi_quality_pool: need n_seq, L, D >= 1, ldx >= D");
  pool_kernel<<<(unsigned)n_seq, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, ldx, L, D, reinterpret_cast<const long long*>(ids), mode, (long long)eos_id, out);
  SVI_CUDA_LAUNCH_CHECK("svi_quality_pool");
  return SVI_OK;
}

extern "C" int svi_quality_score(const float* img, int32_t B, const float* txt, int32_t T, int32_t E, const float* w,
                                 float bias, float* cos, float* aes, void* stream) {
  SVI_REQUIRE(img, "svi_quality_score: null image features");
  SVI_REQUIRE(B >= 1 && B <= (1 << 30) && T >= 0 && E >= 1 && E <= 4096, "svi_quality_score: need B >= 1, T >= 0, 1 <= E <= 4096");
  SVI_REQUIRE(T == 0 || (txt && cos), "svi_quality_score: T > 0 needs txt and cos");
  SVI_REQUIRE(!w || aes, "svi_quality_score: w needs aes");
  SVI_REQUIRE(T > 0 || w, "svi_quality_score: nothing to compute (T == 0 and no head)");
  score_kernel<<<(unsigned)B, kRowThreads, 0, static_cast<cudaStream_t>(stream)>>>(img, txt, T, E, w, bias, cos, aes);
  SVI_CUDA_LAUNCH_CHECK("svi_quality_score");
  return SVI_OK;
}
