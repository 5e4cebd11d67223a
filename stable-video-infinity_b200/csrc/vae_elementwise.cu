// Memory-bound kernels of the Wan VAE path (channels-last activations): RMS-norm + SiLU + bf16 staging of conv
// inputs, nearest upsample, space-to-depth, planar <-> channels-last conversion, row softmax.
#include "common.cuh"
#include "../../include/svi_b200.h"

namespace svi {
namespace vae {

// one warp per pixel; C <= 1024 (each lane keeps up to 8 float4)
__global__ void __launch_bounds__(256)
norm_act_kernel(const float* __restrict__ x, long long n_pix, int C, long long ldx, const float* __restrict__ gamma,
                int do_silu, __nv_bfloat16* __restrict__ y, int Cpad) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int nvec = C >> 2;
  const float sqrt_c = sqrtf((float)C);
  for (long long p = warp_global; p < n_pix; p += nwarps) {
    const float4* xr = reinterpret_cast<const float4*>(x + p * ldx);
    float4 v[8];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = lane + i * 32;
      if (idx < nvec) {
        v[i] = xr[idx];
        ss += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
      }
    }
    float mul = 1.f;
    if (gamma) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      mul = sqrt_c / fmaxf(sqrtf(ss), 1e-12f);   // F.normalize: x / max(||x||, eps)
    }
    uint2* yr = reinterpret_cast<uint2*>(y + p * Cpad);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = lane + i * 32;
      if (idx < nvec) {
        float o[4] = {v[i].x * mul, v[i].y * mul, v[i].z * mul, v[i].w * mul};
        if (gamma) {
          const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + idx);
          o[0] *= g.x; o[1] *= g.y; o[2] *= g.z; o[3] *= g.w;
        }
        if (do_silu) {
#pragma unroll
          for (int j = 0; j < 4; ++j) o[j] = silu(o[j]);
        }
        uint2 pk;
        pk.x = pack_bf16x2(o[0], o[1]);
        pk.y = pack_bf16x2(o[2], o[3]);
        yr[idx] = pk;
      }
    }
    for (int idx = nvec + lane; idx < (Cpad >> 2); idx += 32) yr[idx] = make_uint2(0u, 0u);
  }
}

__global__ void __launch_bounds__(256)
upsample2x_kernel(const float* __restrict__ x, int H, int W, int C, __nv_bfloat16* __restrict__ y) {
  const int cv = C >> 2;
  const long long total = (long long)4 * H * W * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % cv);
    const long long pix = i / cv;
    const int ox = (int)(pix % (2 * W)), oy = (int)(pix / (2 * W));
    const float4 v = *reinterpret_cast<const float4*>(x + ((long long)(oy >> 1) * W + (ox >> 1)) * C + c4 * 4);
    uint2 pk;
    pk.x = pack_bf16x2(v.x, v.y);
    pk.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(y + pix * C + c4 * 4) = pk;
  }
}

__global__ void __launch_bounds__(256)
space_to_depth_kernel(const float* __restrict__ x, int H, int W, int C, int act, __nv_bfloat16* __restrict__ y) {
  const int cv = C >> 2, H2 = H >> 1, W2 = W >> 1;
  const long long total = (long long)H * W * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % cv);
    const long long pix = i / cv;
    const int ix = (int)(pix % W), iy = (int)(pix / W);
    float4 v = *reinterpret_cast<const float4*>(x + pix * C + c4 * 4);
    if (act == SVI_ACT_SILU) {
      v.x = silu(v.x); v.y = silu(v.y); v.z = silu(v.z); v.w = silu(v.w);
    }
    uint2 pk;
    pk.x = pack_bf16x2(v.x, v.y);
    pk.y = pack_bf16x2(v.z, v.w);
    const long long op = (long long)(iy >> 1) * W2 + (ix >> 1);
    const int blk = ((iy & 1) << 1) | (ix & 1);
    *reinterpret_cast<uint2*>(y + op * (4LL * C) + (long long)blk * C + c4 * 4) = pk;
  }
  (void)H2;
}

__global__ void __launch_bounds__(256)
from_planar_kernel(const float* __restrict__ x, int C, long long n_pix, long long ldc, const float* __restrict__ scale,
                   const float* __restrict__ shift, void* __restrict__ out, int ldo, int out_is_bf16) {
  const long long total = n_pix * ldo;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % ldo);
    const long long p = i / ldo;
    float v = 0.f;
    if (c < C) {
      v = x[(long long)c * ldc + p];
      if (scale) v *= scale[c];
      if (shift) v += shift[c];
    }
    if (out_is_bf16) reinterpret_cast<__nv_bfloat16*>(out)[i] = __float2bfloat16_rn(v);
    else reinterpret_cast<float*>(out)[i] = v;
  }
}

__global__ void __launch_bounds__(256)
to_planar_kernel(const float* __restrict__ x, long long ldx, int C, long long n_pix, const float* __restrict__ pre_shift,
                 const float* __restrict__ scale, int clamp, float* __restrict__ out, long long ldc) {
  const long long total = n_pix * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % n_pix;
    const int c = (int)(i / n_pix);
    float v = x[p * ldx + c];
    if (pre_shift) v += pre_shift[c];
    if (scale) v *= scale[c];
    if (clamp) v = fminf(fmaxf(v, -1.f), 1.f);
    out[(long long)c * ldc + p] = v;
  }
}

// planar f32 video [3][T][H][W] in [-1, 1] -> uint8 frames [T][H][W][3]: clip((v + 1) * 127.5, 0, 255) truncated, the
// arithmetic of the reference's tensor2video (svi_video.py:366-370) in the same fp32 order
__global__ void __launch_bounds__(256)
frames_to_uint8_kernel(const float* __restrict__ v, long long plane, long long n_pix, unsigned char* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_pix; i += (long long)gridDim.x * blockDim.x) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float f = fminf(fmaxf((v[c * plane + i] + 1.0f) * 127.5f, 0.0f), 255.0f);
      out[i * 3 + c] = (unsigned char)f;
    }
  }
}

// one 256-thread block per row
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ s, int N, long long lds, float scale, __nv_bfloat16* __restrict__ p,
                    long long ldp) {
  __shared__ float red[8];
  const float* row = s + (long long)blockIdx.x * lds;
  __nv_bfloat16* prow = p + (long long)blockIdx.x * ldp;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < N; i += blockDim.x) mx = fmaxf(mx, row[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x; i < N; i += blockDim.x) sum += __expf((row[i] - mx) * scale);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.f / sum;
  for (int i = threadIdx.x; i < ldp; i += blockDim.x)
    prow[i] = __float2bfloat16_rn(i < N ? __expf((row[i] - mx) * scale) * inv : 0.f);
}

inline int grid_for(long long n, int block) {
  long long g = (n + block - 1) / block;
  const long long cap = 16LL * sm_count();   // grid-stride loops: 16 blocks per SM
  if (cap > 0 && g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace vae
}  // namespace svi

using namespace svi;
using namespace svi::vae;

extern "C" int svi_vae_norm_act(const float* x, int64_t n_pix, int32_t C, int64_t ldx, const float* gamma,
                                int32_t silu, void* y, int32_t Cpad, void* stream) {
  SVI_REQUIRE(x && y && n_pix > 0, "svi_vae_norm_act: null pointer / empty");
  SVI_REQUIRE(C > 0 && C % 4 == 0 && C <= 1024 && Cpad >= C && Cpad % 4 == 0 && ldx >= C && ldx % 4 == 0,
              "svi_vae_norm_act: need C %% 4 == 0, C <= 1024, Cpad >= C, ldx >= C (C=%d Cpad=%d)", C, Cpad);
  norm_act_kernel<<<grid_for(n_pix * 32, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, n_pix, C, ldx, gamma, silu, reinterpret_cast<__nv_bfloat16*>(y), Cpad);
  SVI_CUDA_LAUNCH_CHECK("svi_vae_norm_act");
  return SVI_OK;
}
extern "C" int svi_vae_upsample2x(const float* x, int32_t H, int32_t W, int32_t C, void* y, void* stream) {
  SVI_REQUIRE(x && y && H > 0 && W > 0 && C > 0 && C % 4 == 0, "svi_vae_upsample2x: bad arguments");
  upsample2x_kernel<<<grid_for(4LL * H * W * (C / 4), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, H, W, C, reinterpret_cast<__nv_bfloat16*>(y));
  SVI_CUDA_LAUNCH_CHECK("svi_vae_upsample2x");
  return SVI_OK;
}
extern "C" int svi_vae_space_to_depth(const float* x, int32_t H, int32_t W, int32_t C, void* y, void* stream) {
  SVI_REQUIRE(x && y && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && C > 0 && C % 4 == 0,
              "svi_vae_space_to_depth: need even H, W and C %% 4 == 0");
  space_to_depth_kernel<<<grid_for((long long)H * W * (C / 4), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, H, W, C, SVI_ACT_NONE, reinterpret_cast<__nv_bfloat16*>(y));
  SVI_CUDA_LAUNCH_CHECK("svi_vae_space_to_depth");
  return SVI_OK;
}
extern "C" int svi_vae_space_to_depth_act(const float* x, int32_t H, int32_t W, int32_t C, int32_t act, void* y, void* stream) {
  SVI_REQUIRE(x && y && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && C > 0 && C % 4 == 0,
              "svi_vae_space_to_depth_act: need even H, W and C %% 4 == 0");
  SVI_REQUIRE(act == SVI_ACT_NONE || act == SVI_ACT_SILU, "svi_vae_space_to_depth_act: activation must be none or SiLU");
  space_to_depth_kernel<<<grid_for((long long)H * W * (C / 4), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, H, W, C, act, reinterpret_cast<__nv_bfloat16*>(y));
  SVI_CUDA_LAUNCH_CHECK("svi_vae_space_to_depth_act");
  return SVI_OK;
}
extern "C" int svi_vae_from_planar(const float* x, int32_t C, int64_t n_pix, int64_t ldc, const float* scale,
                                   const float* shift, void* out, int32_t ldo, int32_t out_is_bf16, void* stream) {
  SVI_REQUIRE(x && out && C > 0 && n_pix > 0 && ldo >= C && ldc >= n_pix, "svi_vae_from_planar: bad arguments");
  from_planar_kernel<<<grid_for(n_pix * ldo, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, C, n_pix, ldc, scale,
                                                                                               shift, out, ldo, out_is_bf16);
  SVI_CUDA_LAUNCH_CHECK("svi_vae_from_planar");
  return SVI_OK;
}
extern "C" int svi_vae_to_planar(const float* x, int64_t ldx, int32_t C, int64_t n_pix, const float* pre_shift,
                                 const float* scale, int32_t clamp, float* out, int64_t ldc, void* stream) {
  SVI_REQUIRE(x && out && C > 0 && n_pix > 0 && ldx >= C && ldc >= n_pix, "svi_vae_to_planar: bad arguments");
  to_planar_kernel<<<grid_for(n_pix * C, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, ldx, C, n_pix, pre_shift,
                                                                                           scale, clamp, out, ldc);
  SVI_CUDA_LAUNCH_CHECK("svi_vae_to_planar");
  return SVI_OK;
}
extern "C" int svi_frames_to_uint8(const float* video, int64_t plane_stride, int64_t n_pix, void* out_u8, void* stream) {
  SVI_REQUIRE(video && out_u8 && n_pix > 0 && plane_stride >= n_pix, "svi_frames_to_uint8: bad arguments");
  frames_to_uint8_kernel<<<grid_for(n_pix, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      video, plane_stride, n_pix, static_cast<unsigned char*>(out_u8));
  SVI_CUDA_LAUNCH_CHECK("svi_frames_to_uint8");
  return SVI_OK;
}
extern "C" int svi_softmax_rows(const float* s, int32_t rows, int32_t N, int64_t lds, float scale, void* p, int64_t ldp,
                                void* stream) {
  SVI_REQUIRE(s && p && rows > 0 && N > 0 && lds >= N && ldp >= N, "svi_softmax_rows: bad arguments");
  softmax_rows_kernel<<<rows, 256, 0, static_cast<cudaStream_t>(stream)>>>(s, N, lds, scale,
                                                                           reinterpret_cast<__nv_bfloat16*>(p), ldp);
  SVI_CUDA_LAUNCH_CHECK("svi_softmax_rows");
  return SVI_OK;
}
