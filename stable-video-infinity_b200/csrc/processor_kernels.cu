// Video processors (include/svi_b200_processors.h): Pillow-exact contrast and sharpness, and RIFE's averaging mode.
//
// The editors must give Pillow's bytes, so every float operation is rounded on its own (__fadd_rn / __fmul_rn /
// __fsub_rn: no contraction into FMAs) in the order Pillow's C code evaluates it.  Grids are (blocks per frame, frames):
// one thread per output byte, except the luma sum, which reduces each frame in integers.
#include <math.h>

#include "common.cuh"
#include "../../include/svi_b200_processors.h"

namespace svi {
namespace processors {

constexpr int kThreads = 256;
constexpr int kMaxFrames = 65535;   // gridDim.y

inline unsigned blocks(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

// ImagingBlend: d + rate (x - d) in float; inside [0, 1] the result is only truncated, outside it is clipped first.
__device__ __forceinline__ uint8_t blend(int d, int x, float rate, bool interpolate) {
  const float t = __fadd_rn((float)d, __fmul_rn(rate, (float)(x - d)));
  if (interpolate) return (uint8_t)(int)t;
  if (t <= 0.f) return 0;
  if (t >= 255.f) return 255;
  return (uint8_t)(int)t;
}

__global__ void luma_sum_kernel(const uint8_t* __restrict__ rgb, long long n_pix, unsigned long long* __restrict__ sums) {
  const uint8_t* f = rgb + (long long)blockIdx.y * n_pix * 3;
  unsigned long long s = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_pix; i += (long long)gridDim.x * blockDim.x) {
    const uint8_t* p = f + 3 * i;
    s += (19595u * p[0] + 38470u * p[1] + 7471u * p[2] + 0x8000u) >> 16;
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  __shared__ unsigned long long part[kThreads / 32];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int w = 0; w < kThreads / 32; ++w) t += part[w];
    atomicAdd(sums + blockIdx.y, t);
  }
}

// rgb and out may be the same buffer (each byte is read and written by one thread), so neither is __restrict__.
__global__ void enhance_blend_kernel(const uint8_t* rgb, long long frame_bytes,
                                     const float* __restrict__ degenerate, float rate, bool interpolate,
                                     uint8_t* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= frame_bytes) return;
  const long long o = (long long)blockIdx.y * frame_bytes + i;
  out[o] = blend((int)degenerate[blockIdx.y], rgb[o], rate, interpolate);
}

__global__ void sharpen_kernel(const uint8_t* __restrict__ rgb, int H, int W, float rate, bool interpolate,
                               uint8_t* __restrict__ out) {
  const long long row = 3LL * W, frame_bytes = row * H;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= frame_bytes) return;
  const uint8_t* f = rgb + (long long)blockIdx.y * frame_bytes;
  const int y = (int)(i / row), x = (int)((i - (long long)y * row) / 3);
  const int v = f[i];
  int d = v;
  if (y > 0 && y < H - 1 && x > 0 && x < W - 1) {
    const float edge = __fdiv_rn(1.f, 13.f), centre = __fdiv_rn(5.f, 13.f);
    float ss = 0.f;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx)
        ss = __fadd_rn(ss, __fmul_rn((float)f[i + dy * row + dx * 3], (dy == 0 && dx == 0) ? centre : edge));
    d = ss <= 0.f ? 0 : ss >= 255.f ? 255 : (int)__fadd_rn(ss, 0.5f);
  }
  out[(long long)blockIdx.y * frame_bytes + i] = blend(d, v, rate, interpolate);
}

// blockIdx.y = inner frame - 1; one thread per output byte (pixel p, RGB channel c <- BGR channel 2 - c).
__global__ void rife_average_kernel(const float* __restrict__ frame, const float* __restrict__ merged, long long n_pix,
                                    uint8_t* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * n_pix) return;
  const long long p = i / 3, c = 2 - (i - 3 * p);
  const long long f = blockIdx.y + 1;
  const float a = frame[(f * n_pix + p) * 4 + c];
  const float m = merged[((long long)blockIdx.y * n_pix + p) * 4 + c];
  const float v = __fmul_rn(__fdiv_rn(__fadd_rn(a, m), 2.f), 255.f);
  out[f * 3 * n_pix + i] = (uint8_t)(int)fminf(fmaxf(v, 0.f), 255.f);
}

}  // namespace processors
}  // namespace svi

using namespace svi;

extern "C" int svi_luma_sum_u8(const uint8_t* rgb, int32_t frames, int64_t n_pix, uint64_t* sums, void* stream) {
  SVI_REQUIRE(rgb && sums, "svi_luma_sum_u8: null pointer");
  SVI_REQUIRE(frames > 0 && frames <= processors::kMaxFrames, "svi_luma_sum_u8: frames must be in [1, 65535], got %d",
              frames);
  SVI_REQUIRE(n_pix > 0 && n_pix < (1LL << 40), "svi_luma_sum_u8: bad pixel count");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (cudaMemsetAsync(sums, 0, sizeof(uint64_t) * frames, s) != cudaSuccess) {
    set_last_error("svi_luma_sum_u8: cudaMemsetAsync failed");
    return SVI_ERR_DRIVER;
  }
  const unsigned bx = processors::blocks(n_pix) < 64u ? processors::blocks(n_pix) : 64u;
  processors::luma_sum_kernel<<<dim3(bx, frames), processors::kThreads, 0, s>>>(
      rgb, (long long)n_pix, reinterpret_cast<unsigned long long*>(sums));
  SVI_CUDA_LAUNCH_CHECK("svi_luma_sum_u8");
  return SVI_OK;
}

extern "C" int svi_enhance_blend_u8(const uint8_t* rgb, int32_t frames, int64_t n_pix, const float* degenerate,
                                    float rate, uint8_t* out, void* stream) {
  SVI_REQUIRE(rgb && degenerate && out, "svi_enhance_blend_u8: null pointer");
  SVI_REQUIRE(frames > 0 && frames <= processors::kMaxFrames, "svi_enhance_blend_u8: frames must be in [1, 65535], got %d",
              frames);
  SVI_REQUIRE(n_pix > 0 && n_pix < (1LL << 40), "svi_enhance_blend_u8: bad pixel count");
  SVI_REQUIRE(isfinite(rate), "svi_enhance_blend_u8: rate must be finite");
  const long long fb = 3LL * n_pix;
  processors::enhance_blend_kernel<<<dim3(processors::blocks(fb), frames), processors::kThreads, 0,
                                     static_cast<cudaStream_t>(stream)>>>(rgb, fb, degenerate, rate,
                                                                          rate >= 0.f && rate <= 1.f, out);
  SVI_CUDA_LAUNCH_CHECK("svi_enhance_blend_u8");
  return SVI_OK;
}

extern "C" int svi_sharpen_u8(const uint8_t* rgb, int32_t frames, int32_t H, int32_t W, float rate, uint8_t* out,
                              void* stream) {
  SVI_REQUIRE(rgb && out, "svi_sharpen_u8: null pointer");
  SVI_REQUIRE(frames > 0 && frames <= processors::kMaxFrames, "svi_sharpen_u8: frames must be in [1, 65535], got %d",
              frames);
  SVI_REQUIRE(H > 0 && W > 0 && (long long)H * W < (1LL << 40), "svi_sharpen_u8: bad frame size %d x %d", W, H);
  SVI_REQUIRE(isfinite(rate), "svi_sharpen_u8: rate must be finite");
  const long long total = 3LL * H * W * frames;
  SVI_REQUIRE(out + total <= rgb || rgb + total <= out, "svi_sharpen_u8: out must not overlap rgb");
  processors::sharpen_kernel<<<dim3(processors::blocks(3LL * H * W), frames), processors::kThreads, 0,
                               static_cast<cudaStream_t>(stream)>>>(rgb, H, W, rate, rate >= 0.f && rate <= 1.f, out);
  SVI_CUDA_LAUNCH_CHECK("svi_sharpen_u8");
  return SVI_OK;
}

extern "C" int svi_rife_average_u8(const float* frame, const float* merged, int32_t frames, int64_t n_pix, uint8_t* out,
                                   void* stream) {
  SVI_REQUIRE(frame && merged && out, "svi_rife_average_u8: null pointer");
  SVI_REQUIRE(frames >= 3 && frames - 2 <= processors::kMaxFrames, "svi_rife_average_u8: frames must be in [3, 65537], "
              "got %d", frames);
  SVI_REQUIRE(n_pix > 0 && n_pix < (1LL << 40), "svi_rife_average_u8: bad pixel count");
  processors::rife_average_kernel<<<dim3(processors::blocks(3LL * n_pix), frames - 2), processors::kThreads, 0,
                                    static_cast<cudaStream_t>(stream)>>>(frame, merged, (long long)n_pix, out);
  SVI_CUDA_LAUNCH_CHECK("svi_rife_average_u8");
  return SVI_OK;
}
