// Kernels of the wav2vec2 audio feature extractor (SVI-Talk's audio conditioning) that are not matrix products: the
// per-channel statistics over time of the first conv's GroupNorm (groups = channels), the norm + affine + activation that
// writes the next conv's operand, the im2col gather of a channels-last 1-D convolution (also one group of the grouped
// positional conv, read in place through a column window), and the 50 Hz -> 25 Hz linear interpolation fused with the
// feature projection's LayerNorm.  Every convolution and projection runs on svi_gemm_bf16 (wgmma); attention on
// svi_attn_small.  Replaces, in the reference: utils/src/audio_analysis/wav2vec2.py (the transformers Wav2Vec2Model
// feature encoder, feature projection and encoder it subclasses) and utils/src/audio_analysis/torch_utils.py:16-19
// (linear_interpolation).
#include "common.cuh"
#include "../../include/svi_b200.h"

namespace svi {
namespace audio {

// ---------------------------------------------------------------------------------------------
// Column statistics.  Rows are cut into fixed blocks of `rows_per_block(T)` rows (a function of T only, never of the device);
// pass 1 writes the fp64 (sum, sum of squares) of every (row block, column), pass 2 adds the blocks of a column in index
// order.  No atomics: the same input gives bit-identical statistics on any H100 and any run.
// ---------------------------------------------------------------------------------------------
constexpr int CS_COLS = 32;          // columns per CTA (one warp row)
constexpr int CS_LANES = 8;          // row lanes per CTA
constexpr long long CS_MAX_BLOCKS = 1024;

__host__ __device__ inline long long rows_per_block(long long T) {
  const long long unit = 256;
  long long r = (T + unit * CS_MAX_BLOCKS - 1) / (unit * CS_MAX_BLOCKS);
  return (r < 1 ? 1 : r) * unit;
}

__global__ void __launch_bounds__(CS_COLS * CS_LANES)
col_partials_kernel(const float* __restrict__ x, long long ldx, long long T, int C, long long rpb, double* __restrict__ part) {
  __shared__ double s_sum[CS_LANES][CS_COLS], s_sq[CS_LANES][CS_COLS];
  const int c = blockIdx.x * CS_COLS + threadIdx.x;
  const long long r0 = (long long)blockIdx.y * rpb;
  long long r1 = r0 + rpb;
  if (r1 > T) r1 = T;
  double s = 0.0, q = 0.0;
  if (c < C) {
    for (long long r = r0 + threadIdx.y; r < r1; r += CS_LANES) {
      const double v = (double)x[r * ldx + c];
      s += v;
      q += v * v;
    }
  }
  s_sum[threadIdx.y][threadIdx.x] = s;
  s_sq[threadIdx.y][threadIdx.x] = q;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double ss = 0.0, qq = 0.0;
#pragma unroll
    for (int l = 0; l < CS_LANES; ++l) {
      ss += s_sum[l][threadIdx.x];
      qq += s_sq[l][threadIdx.x];
    }
    part[((long long)blockIdx.y * 2 + 0) * C + c] = ss;
    part[((long long)blockIdx.y * 2 + 1) * C + c] = qq;
  }
}

__global__ void col_combine_kernel(const double* __restrict__ part, int nblk, long long T, int C, float* __restrict__ mean,
                                   float* __restrict__ var) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s = 0.0, q = 0.0;
  for (int b = 0; b < nblk; ++b) {
    s += part[((long long)b * 2 + 0) * C + c];
    q += part[((long long)b * 2 + 1) * C + c];
  }
  const double m = s / (double)T;
  double v = q / (double)T - m * m;     // fp64: the cancellation costs nothing at the fp32 precision that is stored
  mean[c] = (float)m;
  var[c] = (float)(v > 0.0 ? v : 0.0);
}

__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == SVI_ACT_GELU_ERF) return gelu_erf(v);
  if (act == SVI_ACT_GELU_TANH) return gelu_tanh(v);
  if (act == SVI_ACT_SILU) return silu(v);
  if (act == SVI_ACT_RELU) return fmaxf(v, 0.f);
  return v;
}

// y[t, c] = bf16(act((x[t, c] - mean[c]) * rsqrt(var[c] + eps) * gamma[c] + beta[c]))
__global__ void __launch_bounds__(256)
col_norm_act_kernel(const float* __restrict__ x, long long ldx, long long T, int C, const float* __restrict__ mean,
                    const float* __restrict__ var, float eps, const float* __restrict__ gamma, const float* __restrict__ beta,
                    int act, __nv_bfloat16* __restrict__ y, long long ldy) {
  const long long n = T * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / C;
    const int c = (int)(i - t * C);
    float v = (x[t * ldx + c] - mean[c]) * rsqrtf(var[c] + eps);
    if (gamma) v *= gamma[c];
    if (beta) v += beta[c];
    y[t * ldy + c] = __float2bfloat16_rn(apply_act(v, act));
  }
}

// ---------------------------------------------------------------------------------------------
// Conv1d im2col: out[t, j*C + c] = src[t*stride - pad_left + j, col0 + c] (zero outside [0, T_in)), columns [k*C, Kpad)
// zero; split: columns [Kpad, 2 Kpad) hold the bf16 residual v - bf16(v) of the same values.  One thread = 8 output columns.
// ---------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float load_f(const T* p);
template <>
__device__ __forceinline__ float load_f<float>(const float* p) { return *p; }
template <>
__device__ __forceinline__ float load_f<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }

template <typename T>
__global__ void __launch_bounds__(256)
conv1d_gather_kernel(const T* __restrict__ src, long long lds, long long T_in, int col0, int C, int k, int stride, int pad_left,
                     long long T_out, int split, __nv_bfloat16* __restrict__ out, long long ldo, int Kpad) {
  const int chunks = Kpad / 8;
  const long long n = T_out * chunks;
  const int kc = k * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / chunks;
    const int j0 = (int)(i - t * chunks) * 8;
    const long long base = t * stride - pad_left;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int col = j0 + e;
      float val = 0.f;
      if (col < kc) {
        const int tap = col / C;
        const int ch = col - tap * C;
        const long long r = base + tap;
        if (r >= 0 && r < T_in) val = load_f<T>(src + r * lds + col0 + ch);
      }
      v[e] = val;
    }
    uint4 hi;
    hi.x = pack_bf16x2(v[0], v[1]);
    hi.y = pack_bf16x2(v[2], v[3]);
    hi.z = pack_bf16x2(v[4], v[5]);
    hi.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(out + t * ldo + j0) = hi;
    if (split) {
      const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&hi);
      uint4 lo;
      lo.x = pack_bf16x2(v[0] - __bfloat162float(h[0]), v[1] - __bfloat162float(h[1]));
      lo.y = pack_bf16x2(v[2] - __bfloat162float(h[2]), v[3] - __bfloat162float(h[3]));
      lo.z = pack_bf16x2(v[4] - __bfloat162float(h[4]), v[5] - __bfloat162float(h[5]));
      lo.w = pack_bf16x2(v[6] - __bfloat162float(h[6]), v[7] - __bfloat162float(h[7]));
      *reinterpret_cast<uint4*>(out + t * ldo + Kpad + j0) = lo;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Linear interpolation over time (align_corners=True, source coordinate computed as torch's upsample_linear1d does) fused
// with a LayerNorm over the C channels of the blended row -> bf16.  One CTA per output row; the row is staged in shared memory.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
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

__global__ void __launch_bounds__(256)
interp_layernorm_kernel(const float* __restrict__ x, long long ldx, long long T_in, int C, float scale, float eps,
                        const float* __restrict__ gamma, const float* __restrict__ beta, __nv_bfloat16* __restrict__ y,
                        long long ldy) {
  extern __shared__ float row[];
  __shared__ float red[8];
  const long long t = blockIdx.x;
  // area_pixel_compute_source_index (align_corners) + compute_indices_weights_linear of ATen
  const float src = scale * (float)t;
  long long i0 = (long long)src;
  if (i0 > T_in - 1) i0 = T_in - 1;
  const long long i1 = i0 + (i0 < T_in - 1 ? 1 : 0);
  float l1 = src - (float)i0;
  l1 = fminf(fmaxf(l1, 0.f), 1.f);
  const float l0 = 1.f - l1;
  const float* a = x + i0 * ldx;
  const float* b = x + i1 * ldx;
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += 256) {
    const float v = l0 * a[c] + l1 * b[c];
    row[c] = v;
    s += v;
  }
  const float mean = block_sum(s, red) / (float)C;
  float q = 0.f;
  for (int c = threadIdx.x; c < C; c += 256) {
    const float d = row[c] - mean;
    q += d * d;
  }
  const float rstd = rsqrtf(block_sum(q, red) / (float)C + eps);
  __nv_bfloat16* yr = y + t * ldy;
  for (int c = threadIdx.x; c < C; c += 256) yr[c] = __float2bfloat16_rn((row[c] - mean) * rstd * gamma[c] + beta[c]);
}

inline int grid_for(long long n, int block) {
  long long g = (n + block - 1) / block;
  const long long cap = 16LL * sm_count();   // grid-stride loops: 16 blocks per SM
  if (cap > 0 && g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace audio
}  // namespace svi

extern "C" size_t svi_col_stats_workspace_bytes(int64_t T, int32_t C) {
  if (T <= 0 || C <= 0) return 0;
  const long long rpb = svi::audio::rows_per_block(T);
  return (size_t)((T + rpb - 1) / rpb) * 2 * (size_t)C * sizeof(double);
}

extern "C" int svi_col_stats(const float* x, int64_t ldx, int64_t T, int32_t C, float* mean, float* var, void* workspace,
                             size_t workspace_bytes, void* stream) {
  using namespace svi;
  SVI_REQUIRE(x && mean && var && workspace && T > 0 && C > 0 && ldx >= C, "svi_col_stats: bad arguments");
  SVI_REQUIRE(workspace_bytes >= svi_col_stats_workspace_bytes(T, C) && (reinterpret_cast<uintptr_t>(workspace) & 7) == 0,
              "svi_col_stats: workspace must be 8-byte aligned and hold svi_col_stats_workspace_bytes(T, C) = %zu bytes",
              svi_col_stats_workspace_bytes(T, C));
  const long long rpb = audio::rows_per_block(T);
  const int nblk = (int)((T + rpb - 1) / rpb);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  double* part = static_cast<double*>(workspace);
  dim3 grid((C + audio::CS_COLS - 1) / audio::CS_COLS, nblk);
  audio::col_partials_kernel<<<grid, dim3(audio::CS_COLS, audio::CS_LANES), 0, s>>>(x, ldx, T, C, rpb, part);
  SVI_CUDA_LAUNCH_CHECK("svi_col_stats");
  audio::col_combine_kernel<<<(C + 127) / 128, 128, 0, s>>>(part, nblk, T, C, mean, var);
  SVI_CUDA_LAUNCH_CHECK("svi_col_stats");
  return SVI_OK;
}

extern "C" int svi_col_norm_act(const float* x, int64_t ldx, int64_t T, int32_t C, const float* mean, const float* var, float eps,
                                const float* gamma, const float* beta, int32_t act, void* y_bf16, int64_t ldy, void* stream) {
  using namespace svi;
  SVI_REQUIRE(x && mean && var && y_bf16 && T > 0 && C > 0 && ldx >= C && ldy >= C, "svi_col_norm_act: bad arguments");
  SVI_REQUIRE(act >= 0 && act <= 4, "svi_col_norm_act: unknown activation %d", act);
  audio::col_norm_act_kernel<<<audio::grid_for(T * C, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, ldx, T, C, mean, var, eps, gamma, beta, act, reinterpret_cast<__nv_bfloat16*>(y_bf16), ldy);
  SVI_CUDA_LAUNCH_CHECK("svi_col_norm_act");
  return SVI_OK;
}

extern "C" int svi_conv1d_gather(const void* src, int32_t src_is_f32, int64_t lds, int64_t T_in, int32_t col0, int32_t C,
                                 int32_t kernel, int32_t stride, int32_t pad_left, int32_t pad_right, int64_t T_out,
                                 int32_t split, void* out_bf16, int64_t ldo, int32_t Kpad, void* stream) {
  using namespace svi;
  SVI_REQUIRE(src && out_bf16 && T_in > 0 && C > 0 && kernel > 0 && stride > 0 && pad_left >= 0 && pad_right >= 0 && col0 >= 0,
              "svi_conv1d_gather: bad arguments");
  SVI_REQUIRE(lds >= (int64_t)col0 + C, "svi_conv1d_gather: lds must be >= col0 + C");
  const int64_t span = T_in + pad_left + pad_right - kernel;
  SVI_REQUIRE(span >= 0 && T_out > 0 && T_out <= span / stride + 1,
              "svi_conv1d_gather: T_out must be in [1, (T_in + pads - kernel) / stride + 1]");
  SVI_REQUIRE(Kpad % 8 == 0 && (int64_t)Kpad >= (int64_t)kernel * C, "svi_conv1d_gather: Kpad must be a multiple of 8 and >= kernel * C");
  SVI_REQUIRE(ldo % 8 == 0 && ldo >= (int64_t)Kpad * (split ? 2 : 1) && (reinterpret_cast<uintptr_t>(out_bf16) & 15) == 0,
              "svi_conv1d_gather: out must be 16-byte aligned with ldo %% 8 == 0 and ldo >= Kpad (2 Kpad with split)");
  const int grid = audio::grid_for(T_out * (Kpad / 8), 256);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(out_bf16);
  if (src_is_f32)
    audio::conv1d_gather_kernel<float><<<grid, 256, 0, s>>>(static_cast<const float*>(src), lds, T_in, col0, C, kernel, stride,
                                                            pad_left, T_out, split, out, ldo, Kpad);
  else
    audio::conv1d_gather_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(static_cast<const __nv_bfloat16*>(src), lds, T_in, col0, C,
                                                                    kernel, stride, pad_left, T_out, split, out, ldo, Kpad);
  SVI_CUDA_LAUNCH_CHECK("svi_conv1d_gather");
  return SVI_OK;
}

extern "C" int svi_interp_layernorm(const float* x, int64_t ldx, int64_t T_in, int32_t C, int64_t T_out, float eps,
                                    const float* gamma, const float* beta, void* y_bf16, int64_t ldy, void* stream) {
  using namespace svi;
  SVI_REQUIRE(x && gamma && beta && y_bf16 && T_in > 0 && T_out > 0 && C > 0 && ldx >= C && ldy >= C,
              "svi_interp_layernorm: bad arguments");
  SVI_REQUIRE(C <= 12288, "svi_interp_layernorm: C must be <= 12288 (got %d)", C);
  SVI_REQUIRE(T_out < (1LL << 31), "svi_interp_layernorm: T_out too large");
  // ATen: scale = (input_size - 1) / (output_size - 1) in the op-math type, 0 for a single output
  const float scale = T_out > 1 ? (float)(T_in - 1) / (float)(T_out - 1) : 0.f;
  audio::interp_layernorm_kernel<<<(unsigned)T_out, 256, C * sizeof(float), static_cast<cudaStream_t>(stream)>>>(
      x, ldx, T_in, C, scale, eps, gamma, beta, reinterpret_cast<__nv_bfloat16*>(y_bf16), ldy);
  SVI_CUDA_LAUNCH_CHECK("svi_interp_layernorm");
  return SVI_OK;
}
