// RIFE (IFNet) frame interpolation: the element-wise kernels around the convolutions (include/svi_b200_rife.h).
//
//   stage_frames   uint8 RGB -> f32 BGR in [0, 1]                                   (RIFE/__init__.py:135, process_image)
//   block_input    F.interpolate of the block input and flow, both directions, concat, space-to-depth bf16   (:8-12 of
//                  IFBlock.forward and IFNet.forward's two block calls)
//   update_warp    F.interpolate x s of the heads' flow / mask, the averaged update, warp() of both images, and the
//                  sigmoid blend + decode_images (uint8 truncation, BGR -> RGB)
//
// The bilinear resizes follow ATen's upsample_bilinear2d for a given scale_factor (recompute_scale_factor=False): source
// index max(scale * (d + 0.5) - 0.5, 0) with scale = (float)(1 / scale_factor), lower tap (int)src, upper tap clamped to
// the last row / column.  warp() follows grid_sample(bilinear, border, align_corners=True) on linspace(-1, 1) + flow /
// ((size - 1) / 2).  One thread per output pixel, no atomics: the result does not depend on how pairs are batched.
#include "common.cuh"
#include "../../include/svi_b200_rife.h"

namespace svi {
namespace rife {

constexpr int STATE_C = 12;     // warped img0 (3), warped img1 (3), mask, 0, flow0 (2), flow1 (2)
constexpr int BLOCK_C = 11;     // channels of one block input pixel
constexpr int BLOCK_LD = 48;    // channel pitch of the space-to-depth block input: 4 * 11 + 4 zeros

struct Tap {
  int i0, i1;
  float l0, l1;
};

// ATen upsample_bilinear2d (align_corners=False, explicit scale) source taps of destination index d
__device__ __forceinline__ Tap src_tap(int d, float scale, int in_size) {
  float r = scale * ((float)d + 0.5f) - 0.5f;
  r = r < 0.f ? 0.f : r;
  Tap t;
  t.i0 = (int)r;
  t.i1 = t.i0 + (t.i0 < in_size - 1 ? 1 : 0);
  t.l1 = r - (float)t.i0;
  t.l0 = 1.f - t.l1;
  return t;
}

__device__ __forceinline__ float lerp2(const Tap& ty, const Tap& tx, float v00, float v01, float v10, float v11) {
  return ty.l0 * (tx.l0 * v00 + tx.l1 * v01) + ty.l1 * (tx.l0 * v10 + tx.l1 * v11);
}

// torch.linspace(-1, 1, n)[i] in float (ATen's two-sided formula)
__device__ __forceinline__ float linspace_pm1(int i, int n) {
  const float step = 2.f / (float)(n - 1);
  return i < n / 2 ? -1.f + step * (float)i : 1.f - step * (float)(n - 1 - i);
}

// grid_sample bilinear / border / align_corners=True of a 3-channel f32 [H][W][4] image at normalised (gx, gy)
__device__ __forceinline__ void sample_border(const float* img, int H, int W, float gx, float gy, float out[3]) {
  float ix = ((gx + 1.f) / 2.f) * (float)(W - 1);
  float iy = ((gy + 1.f) / 2.f) * (float)(H - 1);
  ix = fminf((float)(W - 1), fmaxf(ix, 0.f));
  iy = fminf((float)(H - 1), fmaxf(iy, 0.f));
  const float fx = floorf(ix), fy = floorf(iy);
  const int x0 = (int)fx, y0 = (int)fy;
  const float x1 = fx + 1.f, y1 = fy + 1.f;
  const float nw = (x1 - ix) * (y1 - iy), ne = (ix - fx) * (y1 - iy);
  const float sw = (x1 - ix) * (iy - fy), se = (ix - fx) * (iy - fy);
  const bool xr = x0 + 1 < W, yd = y0 + 1 < H;
  const float4 a = *reinterpret_cast<const float4*>(img + ((long long)y0 * W + x0) * 4);
  float4 b = make_float4(0.f, 0.f, 0.f, 0.f), c = b, d = b;
  if (xr) b = *reinterpret_cast<const float4*>(img + ((long long)y0 * W + x0 + 1) * 4);
  if (yd) c = *reinterpret_cast<const float4*>(img + ((long long)(y0 + 1) * W + x0) * 4);
  if (xr && yd) d = *reinterpret_cast<const float4*>(img + ((long long)(y0 + 1) * W + x0 + 1) * 4);
  // the same accumulation order as ATen's grid_sampler_2d: nw, ne, sw, se (out-of-range taps contribute nothing)
  out[0] = a.x * nw; out[1] = a.y * nw; out[2] = a.z * nw;
  if (xr) { out[0] += b.x * ne; out[1] += b.y * ne; out[2] += b.z * ne; }
  if (yd) { out[0] += c.x * sw; out[1] += c.y * sw; out[2] += c.z * sw; }
  if (xr && yd) { out[0] += d.x * se; out[1] += d.y * se; out[2] += d.z * se; }
}

__global__ void stage_frames_kernel(const uint8_t* __restrict__ rgb, long long n, float4* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* s = rgb + 3 * i;
  out[i] = make_float4((float)s[2] / 255.f, (float)s[1] / 255.f, (float)s[0] / 255.f, 0.f);
}

// the 12 state channels of pair p at full-resolution pixel (y, x); first block: the images, zero mask and flow
__device__ __forceinline__ void load_state(const svi_rife_block_input& d, int p, int y, int x, float v[STATE_C]) {
  const long long pix = (long long)y * d.W + x;
  if (d.state) {
    const float4* s = reinterpret_cast<const float4*>(d.state + ((long long)p * d.H * d.W + pix) * STATE_C);
    const float4 a = s[0], b = s[1], c = s[2];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y;
    v[6] = b.z; v[7] = b.w; v[8] = c.x; v[9] = c.y; v[10] = c.z; v[11] = c.w;
  } else {
    const float4 a = *reinterpret_cast<const float4*>(d.img0 + p * d.img_stride + pix * 4);
    const float4 b = *reinterpret_cast<const float4*>(d.img1 + p * d.img_stride + pix * 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = b.x; v[4] = b.y; v[5] = b.z;
#pragma unroll
    for (int k = 6; k < STATE_C; ++k) v[k] = 0.f;
  }
}

// one thread per (pair, space-to-depth pixel): 4 block-resolution pixels x 11 channels, for both directions
__global__ void block_input_kernel(const svi_rife_block_input d) {
  const int w2 = d.w / 2, h2 = d.h / 2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)d.pairs * h2 * w2) return;
  const int x2 = (int)(i % w2), y2 = (int)((i / w2) % h2), p = (int)(i / ((long long)w2 * h2));
  __align__(16) __nv_bfloat16 o0[BLOCK_LD], o1[BLOCK_LD];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const Tap ty = src_tap(2 * y2 + (q >> 1), d.src_scale, d.H);
    const Tap tx = src_tap(2 * x2 + (q & 1), d.src_scale, d.W);
    float v00[STATE_C], v01[STATE_C], v10[STATE_C], v11[STATE_C];
    load_state(d, p, ty.i0, tx.i0, v00);
    load_state(d, p, ty.i0, tx.i1, v01);
    load_state(d, p, ty.i1, tx.i0, v10);
    load_state(d, p, ty.i1, tx.i1, v11);
    float v[STATE_C];
#pragma unroll
    for (int k = 0; k < STATE_C; ++k) v[k] = lerp2(ty, tx, v00[k], v01[k], v10[k], v11[k]);
#pragma unroll
    for (int k = 8; k < STATE_C; ++k) v[k] *= d.flow_mul;
    const int b = q * BLOCK_C;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      o0[b + k] = __float2bfloat16_rn(v[k]);
      o0[b + 3 + k] = __float2bfloat16_rn(v[3 + k]);
      o1[b + k] = __float2bfloat16_rn(v[3 + k]);
      o1[b + 3 + k] = __float2bfloat16_rn(v[k]);
    }
    o0[b + 6] = __float2bfloat16_rn(v[6]);
    o1[b + 6] = __float2bfloat16_rn(-v[6]);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      o0[b + 7 + k] = __float2bfloat16_rn(v[8 + k]);
      o1[b + 7 + k] = __float2bfloat16_rn(v[8 + ((k + 2) & 3)]);
    }
  }
#pragma unroll
  for (int k = 4 * BLOCK_C; k < BLOCK_LD; ++k) o0[k] = o1[k] = __float2bfloat16_rn(0.f);
  __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(d.out);
  const long long img = (long long)h2 * w2 * BLOCK_LD;
  uint4* dst0 = reinterpret_cast<uint4*>(out + p * img + ((long long)y2 * w2 + x2) * BLOCK_LD);
  uint4* dst1 = reinterpret_cast<uint4*>(out + (p + d.pairs) * img + ((long long)y2 * w2 + x2) * BLOCK_LD);
#pragma unroll
  for (int k = 0; k < BLOCK_LD / 8; ++k) {
    dst0[k] = reinterpret_cast<const uint4*>(o0)[k];
    dst1[k] = reinterpret_cast<const uint4*>(o1)[k];
  }
}

// bilinear x s upsample of one image's heads output (flow 4, mask 1) at full-resolution pixel (y, x)
__device__ __forceinline__ void head_at(const svi_rife_update& d, int img, const Tap& ty, const Tap& tx, float f[5]) {
  const float* base = d.heads + (long long)img * d.h * d.w * d.heads_ld;
  const float* r00 = base + ((long long)ty.i0 * d.w + tx.i0) * d.heads_ld;
  const float* r01 = base + ((long long)ty.i0 * d.w + tx.i1) * d.heads_ld;
  const float* r10 = base + ((long long)ty.i1 * d.w + tx.i0) * d.heads_ld;
  const float* r11 = base + ((long long)ty.i1 * d.w + tx.i1) * d.heads_ld;
#pragma unroll
  for (int k = 0; k < 5; ++k) f[k] = lerp2(ty, tx, r00[k], r01[k], r10[k], r11[k]);
#pragma unroll
  for (int k = 0; k < 4; ++k) f[k] *= d.flow_mul;
}

__global__ void update_warp_kernel(const svi_rife_update d) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)d.pairs * d.H * d.W) return;
  const int x = (int)(i % d.W), y = (int)((i / d.W) % d.H), p = (int)(i / ((long long)d.W * d.H));
  const long long pix = (long long)y * d.W + x;
  const Tap ty = src_tap(y, d.src_scale, d.h), tx = src_tap(x, d.src_scale, d.w);
  float f0[5], f1[5];
  head_at(d, p, ty, tx, f0);
  head_at(d, p + d.pairs, ty, tx, f1);
  float4* st = reinterpret_cast<float4*>(d.state + ((long long)p * d.H * d.W + pix) * STATE_C);
  float flow[4], mask = 0.f;
  if (d.first) {
    flow[0] = flow[1] = flow[2] = flow[3] = 0.f;
  } else {
    const float4 b = st[1], c = st[2];
    mask = b.z;
    flow[0] = c.x; flow[1] = c.y; flow[2] = c.z; flow[3] = c.w;
  }
  // flow = flow + (f0 + cat(f1[2:4], f1[:2])) / 2;  mask = mask + (m0 + (-m1)) / 2
#pragma unroll
  for (int k = 0; k < 4; ++k) flow[k] = flow[k] + (f0[k] + f1[(k + 2) & 3]) / 2.f;
  mask = mask + (f0[4] + (-f1[4])) / 2.f;
  // warp(): grid = linspace(-1, 1) + flow / ((size - 1) / 2)
  const float gx = linspace_pm1(x, d.W), gy = linspace_pm1(y, d.H);
  const float sx = (float)((d.W - 1.0) / 2.0), sy = (float)((d.H - 1.0) / 2.0);
  float w0[3], w1[3];
  sample_border(d.img0 + p * d.img_stride, d.H, d.W, gx + flow[0] / sx, gy + flow[1] / sy, w0);
  sample_border(d.img1 + p * d.img_stride, d.H, d.W, gx + flow[2] / sx, gy + flow[3] / sy, w1);
  st[0] = make_float4(w0[0], w0[1], w0[2], w1[0]);
  st[1] = make_float4(w1[1], w1[2], mask, 0.f);
  st[2] = make_float4(flow[0], flow[1], flow[2], flow[3]);
  if (!d.merged && !d.rgb) return;
  const float sg = 1.f / (1.f + expf(-mask));
  float m[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) m[k] = w0[k] * sg + w1[k] * (1.f - sg);
  if (d.merged) {
    float o[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) o[k] = d.clip ? fminf(fmaxf(m[k], 0.f), 1.f) : m[k];
    *reinterpret_cast<float4*>(d.merged + p * d.merged_stride + pix * 4) = make_float4(o[0], o[1], o[2], sg);
  }
  if (d.rgb) {
    uint8_t* o = d.rgb + p * d.rgb_stride + pix * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) o[2 - k] = (uint8_t)fminf(fmaxf(m[k] * 255.f, 0.f), 255.f);
  }
}

template <class K, class... A>
int launch_1d(K kernel, long long n, cudaStream_t st, const char* name, A... args) {
  if (n == 0) return SVI_OK;
  const int threads = 256;
  kernel<<<(unsigned)((n + threads - 1) / threads), threads, 0, st>>>(args...);
  SVI_CUDA_LAUNCH_CHECK(name);
  return SVI_OK;
}

}  // namespace rife
}  // namespace svi

extern "C" int svi_rife_stage_frames(const uint8_t* rgb, int64_t n_pix, float* out, void* stream) {
  using namespace svi;
  SVI_REQUIRE(rgb && out, "svi_rife_stage_frames: null pointer");
  SVI_REQUIRE(n_pix >= 0 && n_pix < (1LL << 40), "svi_rife_stage_frames: bad pixel count");
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "svi_rife_stage_frames: out must be 16-byte aligned");
  return rife::launch_1d(rife::stage_frames_kernel, n_pix, static_cast<cudaStream_t>(stream), "svi_rife_stage_frames", rgb,
                         (long long)n_pix, reinterpret_cast<float4*>(out));
}

extern "C" int svi_rife_block_input_launch(const svi_rife_block_input* d, void* stream) {
  using namespace svi;
  SVI_REQUIRE(d && d->img0 && d->img1 && d->out, "svi_rife_block_input_launch: null pointer");
  SVI_REQUIRE(d->pairs > 0 && d->H > 0 && d->W > 0 && d->h > 0 && d->w > 0 && d->h % 2 == 0 && d->w % 2 == 0,
              "svi_rife_block_input_launch: need pairs, H, W > 0 and even h, w > 0");
  SVI_REQUIRE(d->src_scale > 0.f, "svi_rife_block_input_launch: src_scale must be > 0");
  SVI_REQUIRE(d->img_stride % 4 == 0 && d->img_stride >= 0, "svi_rife_block_input_launch: img_stride must be a multiple of 4");
  SVI_REQUIRE(((reinterpret_cast<uintptr_t>(d->img0) | reinterpret_cast<uintptr_t>(d->img1) |
                reinterpret_cast<uintptr_t>(d->state) | reinterpret_cast<uintptr_t>(d->out)) & 15) == 0,
              "svi_rife_block_input_launch: img0, img1, state and out must be 16-byte aligned");
  return rife::launch_1d(rife::block_input_kernel, (long long)d->pairs * (d->h / 2) * (d->w / 2),
                         static_cast<cudaStream_t>(stream), "svi_rife_block_input_launch", *d);
}

extern "C" int svi_rife_update_warp(const svi_rife_update* d, void* stream) {
  using namespace svi;
  SVI_REQUIRE(d && d->heads && d->img0 && d->img1 && d->state, "svi_rife_update_warp: null pointer");
  SVI_REQUIRE(d->pairs > 0 && d->H > 1 && d->W > 1 && d->h > 0 && d->w > 0, "svi_rife_update_warp: need pairs > 0, H, W > 1, h, w > 0");
  SVI_REQUIRE(d->heads_ld >= 8 && d->heads_ld % 4 == 0, "svi_rife_update_warp: heads_ld must be >= 8 and a multiple of 4");
  SVI_REQUIRE(d->src_scale > 0.f, "svi_rife_update_warp: src_scale must be > 0");
  SVI_REQUIRE(d->img_stride % 4 == 0 && d->img_stride >= 0 && d->merged_stride % 4 == 0 && d->merged_stride >= 0 &&
                  d->rgb_stride >= 0,
              "svi_rife_update_warp: img_stride and merged_stride must be multiples of 4");
  SVI_REQUIRE(((reinterpret_cast<uintptr_t>(d->img0) | reinterpret_cast<uintptr_t>(d->img1) |
                reinterpret_cast<uintptr_t>(d->state) | reinterpret_cast<uintptr_t>(d->merged) |
                reinterpret_cast<uintptr_t>(d->heads)) & 15) == 0,
              "svi_rife_update_warp: img0, img1, state, merged and heads must be 16-byte aligned");
  return rife::launch_1d(rife::update_warp_kernel, (long long)d->pairs * d->H * d->W, static_cast<cudaStream_t>(stream),
                         "svi_rife_update_warp", *d);
}
