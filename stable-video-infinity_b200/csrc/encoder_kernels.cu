// Kernels of the two conditioning encoders that run once per clip (umT5 text encoder, CLIP ViT image encoder):
// token-embedding gather, T5 RMS norm, fp32-output LayerNorm, gated-activation product and a small-sequence attention
// with arbitrary head width, additive relative-position bias and key mask.  The projections and MLPs of both encoders
// run on svi_gemm_bf16 (wgmma); what is here is HBM/latency-bound glue and the 512- / 257-token attention
// (0.2 % of the encoders' FLOPs), written as plain fp32 SIMT code.
//
// Replaces: reference diffsynth/models/wan_video_text_encoder.py (T5LayerNorm :22-35, T5Attention :55-89 incl. the
// T5RelativeEmbedding bias :159-190 and the key mask, T5FeedForward :105-110, token_embedding :246) and
// diffsynth/models/wan_video_image_encoder.py (SelfAttention :255-268, pre_norm :471).
#include "common.cuh"
#include "../../include/svi_b200.h"

namespace svi {
namespace enc {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float block_sum(float v, float* red) {   // 256 threads
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) {
    t = warp_sum(t);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}

// out[i, :] = float(table[ids[i], :])
__global__ void __launch_bounds__(256)
embedding_gather_kernel(const long long* __restrict__ ids, const __nv_bfloat16* __restrict__ table, int dim, long long vocab,
                        float* __restrict__ out) {
  long long id = ids[blockIdx.x];
  if (id < 0 || id >= vocab) id = 0;     // validated on the host; never read out of bounds on the device
  const __nv_bfloat162* src = reinterpret_cast<const __nv_bfloat162*>(table + id * dim);
  float2* dst = reinterpret_cast<float2*>(out + (long long)blockIdx.x * dim);
  for (int i = threadIdx.x; i < dim / 2; i += blockDim.x) dst[i] = __bfloat1622float2(src[i]);
}

// y = w * x * rsqrt(mean(x^2) + eps)  -> bf16   (T5LayerNorm)
__global__ void __launch_bounds__(256)
rmsnorm_affine_kernel(const float* __restrict__ x, int D, float eps, const float* __restrict__ w,
                      __nv_bfloat16* __restrict__ y) {
  __shared__ float red[8];
  const float4* xr = reinterpret_cast<const float4*>(x + (long long)blockIdx.x * D);
  float s = 0.f;
  for (int i = threadIdx.x; i < D / 4; i += 256) {
    const float4 v = xr[i];
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  const float rs = rsqrtf(block_sum(s, red) / (float)D + eps);
  uint2* yr = reinterpret_cast<uint2*>(y + (long long)blockIdx.x * D);
  for (int i = threadIdx.x; i < D / 4; i += 256) {
    const float4 v = xr[i];
    const float4 g = __ldg(reinterpret_cast<const float4*>(w) + i);
    uint2 pk;
    pk.x = pack_bf16x2(v.x * rs * g.x, v.y * rs * g.y);
    pk.y = pack_bf16x2(v.z * rs * g.z, v.w * rs * g.w);
    yr[i] = pk;
  }
}

// y = LayerNorm(x) * gamma + beta  -> f32 (the ViT pre-norm output IS the residual stream, so it stays fp32)
__global__ void __launch_bounds__(256)
layernorm_f32_kernel(const float* __restrict__ x, int D, float eps, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float* __restrict__ y) {
  __shared__ float red[8];
  const float* xr = x + (long long)blockIdx.x * D;
  float s = 0.f;
  for (int i = threadIdx.x; i < D; i += 256) s += xr[i];
  const float mean = block_sum(s, red) / (float)D;
  float q = 0.f;
  for (int i = threadIdx.x; i < D; i += 256) {
    const float c = xr[i] - mean;
    q += c * c;
  }
  const float rstd = rsqrtf(block_sum(q, red) / (float)D + eps);
  float* yr = y + (long long)blockIdx.x * D;
  for (int i = threadIdx.x; i < D; i += 256) yr[i] = (xr[i] - mean) * rstd * gamma[i] + beta[i];
}

__global__ void mul_bf16_kernel(const __nv_bfloat162* __restrict__ a, const __nv_bfloat162* __restrict__ b,
                                __nv_bfloat162* __restrict__ out, long long n2) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n2; i += (long long)gridDim.x * blockDim.x) {
    const float2 x = __bfloat1622float2(a[i]), y = __bfloat1622float2(b[i]);
    out[i] = __floats2bfloat162_rn(x.x * y.x, x.y * y.y);
  }
}

// ---------------------------------------------------------------------------------------------
// Small-sequence attention: one block = 32 query rows of one head (8 warps x 4 rows), K/V streamed through shared
// memory in tiles of 32 keys, online softmax in fp32.  Lane j scores key j of the tile; lane c owns output columns
// c, c+32, c+64, c+96 (< head_dim).
// ---------------------------------------------------------------------------------------------
constexpr int AS_QB = 32;
constexpr int AS_KT = 32;
constexpr int AS_MAX_HD = 128;
constexpr int AS_ROWS_PER_WARP = 4;

struct SmallAttnParams {
  const __nv_bfloat16 *Q, *K, *V;
  __nv_bfloat16* O;
  long long ldq, ldk, ldv, ldo;
  int Lq, Lk, hd;
  float scale;
  const float* bias_table;   // [n_buckets, H] or null
  const int* bucket;         // [Lq, Lk] bucket index of (query, key) or null
  const int* key_mask;       // [Lk], 0 = masked, or null
  int H;
};

__global__ void __launch_bounds__(256)
attn_small_kernel(SmallAttnParams p) {
  extern __shared__ float sm[];
  const int hd = p.hd, kst = hd + 1;
  float* q_s = sm;                       // [32][hd]
  float* k_s = q_s + AS_QB * hd;         // [32][hd + 1]
  float* v_s = k_s + AS_KT * kst;        // [32][hd]
  float* p_s = v_s + AS_KT * hd;         // [8][32]
  const int head = blockIdx.y, q0 = blockIdx.x * AS_QB;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col0 = head * hd;

  for (int i = threadIdx.x; i < AS_QB * hd; i += 256) {
    const int r = i / hd, d = i - r * hd;
    q_s[i] = (q0 + r < p.Lq) ? __bfloat162float(p.Q[(long long)(q0 + r) * p.ldq + col0 + d]) : 0.f;
  }
  float m[AS_ROWS_PER_WARP], l[AS_ROWS_PER_WARP], acc[AS_ROWS_PER_WARP][4];
#pragma unroll
  for (int r = 0; r < AS_ROWS_PER_WARP; ++r) {
    m[r] = -INFINITY;
    l[r] = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
  }

  for (int j0 = 0; j0 < p.Lk; j0 += AS_KT) {
    __syncthreads();   // previous tile fully consumed (and q_s written, first time round)
    for (int i = threadIdx.x; i < AS_KT * hd; i += 256) {
      const int j = i / hd, d = i - j * hd;
      const bool ok = j0 + j < p.Lk;
      k_s[j * kst + d] = ok ? __bfloat162float(p.K[(long long)(j0 + j) * p.ldk + col0 + d]) : 0.f;
      v_s[j * hd + d] = ok ? __bfloat162float(p.V[(long long)(j0 + j) * p.ldv + col0 + d]) : 0.f;
    }
    __syncthreads();
    const int key = j0 + lane;
    const bool key_ok = key < p.Lk && (!p.key_mask || p.key_mask[key] != 0);
#pragma unroll
    for (int r = 0; r < AS_ROWS_PER_WARP; ++r) {
      const int row = warp * AS_ROWS_PER_WARP + r;
      const int qi = q0 + row;
      float s = 0.f;
      const float* qr = q_s + row * hd;
      const float* kr = k_s + lane * kst;
      for (int d = 0; d < hd; ++d) s += qr[d] * kr[d];
      s *= p.scale;
      if (p.bias_table && key < p.Lk && qi < p.Lq) s += p.bias_table[p.bucket[(long long)qi * p.Lk + key] * p.H + head];
      if (!key_ok) s = -INFINITY;
      const float m_new = fmaxf(m[r], warp_max(s));
      float pj = 0.f, corr = 1.f;
      if (m_new > -INFINITY) {
        pj = __expf(s - m_new);                 // masked: exp(-inf) = 0
        corr = __expf(m[r] - m_new);            // m[r] = -inf on the first live tile: 0
      }
      l[r] = l[r] * corr + warp_sum(pj);
      m[r] = m_new;
      __syncwarp();
      p_s[warp * 32 + lane] = pj;
      __syncwarp();
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int d = lane + 32 * c;
        if (d < hd) {
          float a = acc[r][c] * corr;
          for (int j = 0; j < AS_KT; ++j) a += p_s[warp * 32 + j] * v_s[j * hd + d];
          acc[r][c] = a;
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < AS_ROWS_PER_WARP; ++r) {
    const int qi = q0 + warp * AS_ROWS_PER_WARP + r;
    if (qi >= p.Lq) continue;
    const float inv = l[r] > 0.f ? 1.f / l[r] : 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int d = lane + 32 * c;
      if (d < hd) p.O[(long long)qi * p.ldo + col0 + d] = __float2bfloat16_rn(acc[r][c] * inv);
    }
  }
}

}  // namespace enc
}  // namespace svi

extern "C" int svi_embedding_gather(const int64_t* ids, int32_t n, const void* table_bf16, int32_t dim, int64_t vocab,
                                    float* out, void* stream) {
  using namespace svi;
  SVI_REQUIRE(ids && table_bf16 && out && n > 0 && dim > 0 && dim % 2 == 0 && vocab > 0, "svi_embedding_gather: bad arguments");
  enc::embedding_gather_kernel<<<n, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(ids), reinterpret_cast<const __nv_bfloat16*>(table_bf16), dim, vocab, out);
  SVI_CUDA_LAUNCH_CHECK("svi_embedding_gather");
  return SVI_OK;
}

extern "C" int svi_rmsnorm_affine(const float* x, int32_t M, int32_t D, float eps, const float* w, void* y_bf16,
                                  void* stream) {
  using namespace svi;
  SVI_REQUIRE(x && w && y_bf16 && M > 0 && D > 0 && D % 4 == 0, "svi_rmsnorm_affine: need M > 0, D %% 4 == 0");
  SVI_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w)) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(y_bf16) & 7) == 0, "svi_rmsnorm_affine: alignment");
  enc::rmsnorm_affine_kernel<<<M, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, D, eps, w,
                                                                               reinterpret_cast<__nv_bfloat16*>(y_bf16));
  SVI_CUDA_LAUNCH_CHECK("svi_rmsnorm_affine");
  return SVI_OK;
}

extern "C" int svi_layernorm_f32(const float* x, int32_t M, int32_t D, float eps, const float* gamma, const float* beta,
                                 float* y, void* stream) {
  using namespace svi;
  SVI_REQUIRE(x && gamma && beta && y && M > 0 && D > 0, "svi_layernorm_f32: bad arguments");
  enc::layernorm_f32_kernel<<<M, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, D, eps, gamma, beta, y);
  SVI_CUDA_LAUNCH_CHECK("svi_layernorm_f32");
  return SVI_OK;
}

extern "C" int svi_mul_bf16(const void* a, const void* b, void* out, int64_t n, void* stream) {
  using namespace svi;
  SVI_REQUIRE(a && b && out && n > 0 && n % 2 == 0, "svi_mul_bf16: n must be a positive even number");
  long long blocks = (n / 2 + 255) / 256;
  const int cap = 16 * sm_count();   // grid-stride loop: 16 blocks per SM
  if (cap > 0 && blocks > cap) blocks = cap;
  enc::mul_bf16_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat162*>(a), reinterpret_cast<const __nv_bfloat162*>(b),
      reinterpret_cast<__nv_bfloat162*>(out), n / 2);
  SVI_CUDA_LAUNCH_CHECK("svi_mul_bf16");
  return SVI_OK;
}

extern "C" int svi_attn_small(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* O,
                              int64_t ldo, int32_t Lq, int32_t Lk, int32_t num_heads, int32_t head_dim, float scale,
                              const float* bias_table, const int32_t* bucket, const int32_t* key_mask, void* stream) {
  using namespace svi;
  SVI_REQUIRE(Q && K && V && O && Lq > 0 && Lk > 0 && num_heads > 0, "svi_attn_small: bad arguments");
  SVI_REQUIRE(head_dim > 0 && head_dim <= enc::AS_MAX_HD, "svi_attn_small: head_dim must be in [1, 128] (got %d)", head_dim);
  SVI_REQUIRE((bias_table == nullptr) == (bucket == nullptr), "svi_attn_small: bias_table and bucket go together");
  const int64_t width = (int64_t)num_heads * head_dim;
  SVI_REQUIRE(ldq >= width && ldk >= width && ldv >= width && ldo >= width, "svi_attn_small: leading dimensions too small");
  // read with 4-byte scalar loads
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(bias_table) & 3) == 0, "svi_attn_small: bias_table must be 4-byte aligned");
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(bucket) & 3) == 0, "svi_attn_small: bucket must be 4-byte aligned");
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(key_mask) & 3) == 0, "svi_attn_small: key_mask must be 4-byte aligned");
  enc::SmallAttnParams p;
  p.Q = reinterpret_cast<const __nv_bfloat16*>(Q);
  p.K = reinterpret_cast<const __nv_bfloat16*>(K);
  p.V = reinterpret_cast<const __nv_bfloat16*>(V);
  p.O = reinterpret_cast<__nv_bfloat16*>(O);
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
  p.Lq = Lq; p.Lk = Lk; p.hd = head_dim; p.scale = scale;
  p.bias_table = bias_table; p.bucket = bucket; p.key_mask = key_mask; p.H = num_heads;
  const size_t smem = sizeof(float) * ((size_t)enc::AS_QB * head_dim + (size_t)enc::AS_KT * (head_dim + 1) +
                                       (size_t)enc::AS_KT * head_dim + 8 * 32);
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(enc::attn_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    attr_set = true;
  }
  dim3 grid((Lq + enc::AS_QB - 1) / enc::AS_QB, num_heads);
  enc::attn_small_kernel<<<grid, 256, smem, static_cast<cudaStream_t>(stream)>>>(p);
  SVI_CUDA_LAUNCH_CHECK("svi_attn_small");
  return SVI_OK;
}
