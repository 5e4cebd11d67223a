// FastBlend: PatchMatch and blending-table arithmetic (include/svi_b200_fastblend.h).
//
// Every kernel computes one output element per thread in a fixed order, with each addition and product rounded on its
// own (__fadd_rn / __fmul_rn / __fdiv_rn: no contraction into FMAs), so tests/ can hold it to a torch restatement
// (oracle/fastblend_oracle.py) bit for bit.  Frames are channels-last, channel padded to 4.
#include "common.cuh"
#include "../../include/svi_b200_fastblend.h"
#include "../../include/svi_b200_fastblend_modes.h"

namespace svi {
namespace fastblend {

constexpr int kTile = 16;   // step kernel: 16 x 16 target pixels per block

__device__ __forceinline__ uint32_t lowbias32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}

__device__ __forceinline__ uint32_t stream_u(uint32_t k, uint32_t i) { return lowbias32(lowbias32(k ^ 0x9e3779b9u) ^ i); }

__global__ void stage_kernel(const uint8_t* __restrict__ rgb, long long n, float4* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* s = rgb + 3 * i;
  out[i] = make_float4((float)s[0], (float)s[1], (float)s[2], 0.f);
}

// cv2's resizeAreaFast_ for an integer ratio k: row-major over the cell, groups of four added left to right into one
// term, then the term into the running sum, a scalar tail, then the product with 1 / k^2.
__global__ void downsample_kernel(const float* __restrict__ src, int n, int H, int W, int k, float* __restrict__ dst) {
  const int h = H / k, w = W / k;
  const long long total = (long long)n * h * w * 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i & 3);
  if (c == 3) { dst[i] = 0.f; return; }
  const long long p = i >> 2;
  const int x = (int)(p % w), y = (int)((p / w) % h), b = (int)(p / ((long long)w * h));
  const float* base = src + (((long long)b * H + (long long)y * k) * W + (long long)x * k) * 4 + c;
  const int area = k * k;
  auto tap = [&](int t) { return __ldg(base + ((long long)(t / k) * W + (t % k)) * 4); };
  float sum = 0.f;
  int t = 0;
  for (; t <= area - 4; t += 4) sum = __fadd_rn(sum, __fadd_rn(__fadd_rn(__fadd_rn(tap(t), tap(t + 1)), tap(t + 2)), tap(t + 3)));
  for (; t < area; t++) sum = __fadd_rn(sum, tap(t));
  dst[i] = __fmul_rn(sum, __fdiv_rn(1.f, (float)area));
}

__global__ void nnf_identity_kernel(int2* __restrict__ nnf, int B, int H, int W) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * H * W) return;
  const int x = (int)(i % W), y = (int)((i / W) % H);
  nnf[i] = make_int2(y, x);
}

__global__ void nnf_upscale_kernel(const int2* __restrict__ src, int B, int h, int w, int2* __restrict__ dst) {
  const int H = 2 * h, W = 2 * w;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * H * W) return;
  const int x = (int)(i % W), y = (int)((i / W) % H), b = (int)(i / ((long long)W * H));
  const int2 s = src[((long long)b * h + y / 2) * w + x / 2];
  int r = 2 * s.x + ((y & 1) && y < B ? 1 : 0);
  int q = 2 * s.y + ((x & 1) && x < B ? 1 : 0);
  dst[i] = make_int2(min(max(r, 0), H - 1), min(max(q, 0), W - 1));
}

__global__ void remap_kernel(const float4* __restrict__ style, const int2* __restrict__ nnf, int B, int H, int W, int r,
                             float4* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * H * W) return;
  const int x = (int)(i % W), y = (int)((i / W) % H);
  const long long frame = i - ((long long)y * W + x);
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  int num = 0;
  for (int px = max(-r, -y); px <= min(r, H - 1 - y); px++) {
    for (int py = max(-r, -x); py <= min(r, W - 1 - x); py++) {
      const int2 m = nnf[frame + (long long)(y + px) * W + (x + py)];
      const int sy = m.x - px, sx = m.y - py;
      if (sy < 0 || sx < 0 || sy >= H || sx >= W) continue;
      const float4 v = __ldg(style + frame + (long long)sy * W + sx);
      num++;
      s0 = __fadd_rn(s0, v.x);
      s1 = __fadd_rn(s1, v.y);
      s2 = __fadd_rn(s2, v.z);
    }
  }
  const float fn = (float)num;
  out[i] = make_float4(__fdiv_rn(s0, fn), __fdiv_rn(s1, fn), __fdiv_rn(s2, fn), 0.f);
}

__device__ __forceinline__ float sq_acc(float e, float4 t, float4 s) {
  const float d0 = __fsub_rn(t.x, s.x), d1 = __fsub_rn(t.y, s.y), d2 = __fsub_rn(t.z, s.z);
  e = __fadd_rn(e, __fmul_rn(d0, d0));
  e = __fadd_rn(e, __fmul_rn(d1, d1));
  return __fadd_rn(e, __fmul_rn(d2, d2));
}

// One PatchMatch step.  A block owns a 16 x 16 tile of one frame: the target guide and target style windows of the tile
// (with their r-pixel halo, zero outside the frame) are staged in shared memory; the candidate stays in registers and
// the source taps are read through the read-only cache (neighbouring candidates overlap, so they mostly hit).
__global__ void __launch_bounds__(kTile * kTile) step_kernel(svi_fastblend_step_desc d) {
  extern __shared__ float4 win[];
  const int H = d.H, W = d.W, r = (d.patch_size - 1) / 2, side = kTile + 2 * r;
  float4* tg = win;
  float4* ts = win + side * side;
  const int b = blockIdx.z, y0 = blockIdx.y * kTile, x0 = blockIdx.x * kTile;
  const long long frame = (long long)b * H * W;
  const float4* tgt_guide = reinterpret_cast<const float4*>(d.tgt_guide) + frame;
  const float4* tgt_style = reinterpret_cast<const float4*>(d.tgt_style) + frame;
  for (int j = threadIdx.y * kTile + threadIdx.x; j < side * side; j += kTile * kTile) {
    const int wy = y0 - r + j / side, wx = x0 - r + j % side;
    const bool in = wy >= 0 && wy < H && wx >= 0 && wx < W;
    tg[j] = in ? __ldg(tgt_guide + (long long)wy * W + wx) : make_float4(0.f, 0.f, 0.f, 0.f);
    ts[j] = in ? __ldg(tgt_style + (long long)wy * W + wx) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();
  const int y = y0 + threadIdx.y, x = x0 + threadIdx.x;
  if (y >= H || x >= W) return;
  const int2* nnf = reinterpret_cast<const int2*>(d.nnf_in) + frame;
  const long long pix = (long long)y * W + x;
  const int2 cur = nnf[pix];
  int cy = cur.x, cx = cur.y;
  if (d.mode == SVI_FASTBLEND_NEIGHBOUR) {
    int2 m;
    switch (d.dir) {
      case 0: m = nnf[(long long)max(y - 1, 0) * W + x]; m.x += 1; break;
      case 1: m = nnf[(long long)y * W + max(x - 1, 0)]; m.y += 1; break;
      case 2: m = nnf[(long long)min(y + 1, H - 1) * W + x]; m.x -= 1; break;
      default: m = nnf[(long long)y * W + min(x + 1, W - 1)]; m.y -= 1; break;
    }
    cy = m.x;
    cx = m.y;
  } else if (d.mode == SVI_FASTBLEND_RANDOM) {
    const uint32_t span = (uint32_t)(2 * d.radius + 1);
    const uint32_t e0 = (uint32_t)((frame + pix) * 2);
    cy += -d.radius + (int)(stream_u(d.draw, e0) % span);
    cx += -d.radius + (int)(stream_u(d.draw, e0 + 1) % span);
  }
  cy = min(max(cy, 0), H - 1);
  cx = min(max(cx, 0), W - 1);

  const float4* sg = reinterpret_cast<const float4*>(d.src_guide) + frame;
  const float4* ss = reinterpret_cast<const float4*>(d.src_style) + frame;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  float eg = 0.f, es = 0.f;
  for (int px = -r; px <= r; px++) {
    const int sy = cy + px;
    const bool row_in = sy >= 0 && sy < H;
    const float4* tg_row = tg + (threadIdx.y + r + px) * side + threadIdx.x + r;
    const float4* ts_row = ts + (threadIdx.y + r + px) * side + threadIdx.x + r;
    for (int py = -r; py <= r; py++) {
      const int sx = cx + py;
      const bool in = row_in && sx >= 0 && sx < W;
      const long long s = (long long)sy * W + sx;
      const float4 g = in ? __ldg(sg + s) : zero;
      const float4 st = in ? __ldg(ss + s) : zero;
      eg = sq_acc(eg, tg_row[py], g);
      es = sq_acc(es, ts_row[py], st);
    }
  }
  const float e = __fadd_rn(__fmul_rn(eg, d.guide_weight), es);
  const long long o = frame + pix;
  int2* nnf_out = reinterpret_cast<int2*>(d.nnf_out);
  if (d.mode == SVI_FASTBLEND_CURRENT || e < d.err_in[o]) {
    nnf_out[o] = make_int2(cy, cx);
    d.err_out[o] = e;
  } else {
    nnf_out[o] = cur;
    d.err_out[o] = d.err_in[o];
  }
}

// numpy's promotion, per table operand: a uint8 or f64 frame times a Python float is f64; an f32 frame stays f32 with
// the scalar rounded to f32.
struct Term {
  double v;
  bool f64;
};

__device__ __forceinline__ Term term(const void* p, int type, double s, long long e) {
  if (type == SVI_FASTBLEND_F64) return {__dmul_rn(static_cast<const double*>(p)[e], s), true};
  const float v = static_cast<const float*>(p)[e];
  if (type == SVI_FASTBLEND_U8) return {__dmul_rn((double)v, s), true};
  return {(double)__fmul_rn(v, (float)s), false};
}

__device__ __forceinline__ Term add(Term a, Term b) {
  if (!a.f64 && !b.f64) return {(double)__fadd_rn((float)a.v, (float)b.v), false};
  return {__dadd_rn(a.v, b.v), true};
}

__device__ __forceinline__ float load_f(const void* p, int type, long long e) {
  return type == SVI_FASTBLEND_F64 ? (float)static_cast<const double*>(p)[e] : static_cast<const float*>(p)[e];
}

__global__ void table_kernel(svi_fastblend_table_desc d) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.n_pix * 4) return;
  const int ch = (int)(i & 3);
  if (d.op == SVI_FASTBLEND_MEAN || d.op == SVI_FASTBLEND_HALF) {
    float v = 0.f;
    if (ch < 3) {
      const float a = load_f(d.a, d.a_type, i), b = load_f(d.b, d.b_type, i);
      v = d.op == SVI_FASTBLEND_MEAN ? __fadd_rn(__fmul_rn(a, (float)d.sa), __fdiv_rn(b, (float)d.sb))
                                     : __fdiv_rn(__fadd_rn(a, b), 2.f);
    }
    static_cast<float*>(d.out)[i] = v;
    return;
  }
  if (ch == 3) {
    if (d.out_type == SVI_FASTBLEND_F64) static_cast<double*>(d.out)[i] = 0.0;
    else if (d.out_type == SVI_FASTBLEND_F32) static_cast<float*>(d.out)[i] = 0.f;
    return;
  }
  Term t = add(term(d.a, d.a_type, d.sa, i), term(d.b, d.b_type, d.sb, i));
  if (d.c) t = add(t, term(d.c, d.c_type, d.sc, i));
  if (d.out_type == SVI_FASTBLEND_F64) {
    static_cast<double*>(d.out)[i] = t.v;
  } else if (d.out_type == SVI_FASTBLEND_F32) {
    static_cast<float*>(d.out)[i] = (float)t.v;
  } else {
    const double v = fmin(fmax(t.v, 0.0), 255.0);
    static_cast<uint8_t*>(d.out)[(i >> 2) * 3 + ch] = (uint8_t)(int)v;
  }
}

inline unsigned blocks(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

}  // namespace fastblend
}  // namespace svi

using namespace svi;

extern "C" int svi_fastblend_stage_frames(const uint8_t* rgb, int64_t n_pix, float* out, void* stream) {
  SVI_REQUIRE(rgb && out, "svi_fastblend_stage_frames: null pointer");
  SVI_REQUIRE(n_pix >= 0 && n_pix < (1LL << 40), "svi_fastblend_stage_frames: bad pixel count");
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "svi_fastblend_stage_frames: out must be 16-byte aligned");
  if (n_pix == 0) return SVI_OK;
  fastblend::stage_kernel<<<fastblend::blocks(n_pix, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      rgb, (long long)n_pix, reinterpret_cast<float4*>(out));
  SVI_CUDA_LAUNCH_CHECK("svi_fastblend_stage_frames");
  return SVI_OK;
}

extern "C" int svi_fastblend_downsample(const float* src, int32_t n, int32_t H, int32_t W, int32_t k, float* dst,
                                        void* stream) {
  SVI_REQUIRE(src && dst, "svi_fastblend_downsample: null pointer");
  SVI_REQUIRE(n > 0 && H > 0 && W > 0 && k >= 1 && H % k == 0 && W % k == 0,
              "svi_fastblend_downsample: H and W must be positive multiples of k");
  fastblend::downsample_kernel<<<fastblend::blocks((long long)n * (H / k) * (W / k) * 4, 256), 256, 0,
                                 static_cast<cudaStream_t>(stream)>>>(src, n, H, W, k, dst);
  SVI_CUDA_LAUNCH_CHECK("svi_fastblend_downsample");
  return SVI_OK;
}

extern "C" int svi_fastblend_nnf_identity(int32_t* nnf, int32_t B, int32_t H, int32_t W, void* stream) {
  SVI_REQUIRE(nnf, "svi_fastblend_nnf_identity: null pointer");
  SVI_REQUIRE(B > 0 && H > 0 && W > 0, "svi_fastblend_nnf_identity: bad shape");
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(nnf) & 7) == 0, "svi_fastblend_nnf_identity: nnf must be 8-byte aligned");
  fastblend::nnf_identity_kernel<<<fastblend::blocks((long long)B * H * W, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<int2*>(nnf), B, H, W);
  SVI_CUDA_LAUNCH_CHECK("svi_fastblend_nnf_identity");
  return SVI_OK;
}

extern "C" int svi_fastblend_nnf_upscale(const int32_t* src, int32_t B, int32_t h, int32_t w, int32_t* dst, void* stream) {
  SVI_REQUIRE(src && dst && src != dst, "svi_fastblend_nnf_upscale: null or aliased pointer");
  SVI_REQUIRE(B > 0 && h > 0 && w > 0, "svi_fastblend_nnf_upscale: bad shape");
  SVI_REQUIRE(((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 7) == 0,
              "svi_fastblend_nnf_upscale: fields must be 8-byte aligned");
  fastblend::nnf_upscale_kernel<<<fastblend::blocks((long long)B * 4 * h * w, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const int2*>(src), B, h, w, reinterpret_cast<int2*>(dst));
  SVI_CUDA_LAUNCH_CHECK("svi_fastblend_nnf_upscale");
  return SVI_OK;
}

extern "C" int svi_fastblend_remap(const float* style, const int32_t* nnf, int32_t B, int32_t H, int32_t W,
                                   int32_t patch_size, float* out, void* stream) {
  SVI_REQUIRE(style && nnf && out, "svi_fastblend_remap: null pointer");
  SVI_REQUIRE(B > 0 && H > 0 && W > 0 && patch_size >= 1, "svi_fastblend_remap: bad shape or patch size");
  SVI_REQUIRE(((reinterpret_cast<uintptr_t>(style) | reinterpret_cast<uintptr_t>(out)) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(nnf) & 7) == 0,
              "svi_fastblend_remap: frames must be 16-byte and the field 8-byte aligned");
  fastblend::remap_kernel<<<fastblend::blocks((long long)B * H * W, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(style), reinterpret_cast<const int2*>(nnf), B, H, W, (patch_size - 1) / 2,
      reinterpret_cast<float4*>(out));
  SVI_CUDA_LAUNCH_CHECK("svi_fastblend_remap");
  return SVI_OK;
}

extern "C" int svi_fastblend_step(const svi_fastblend_step_desc* d, void* stream) {
  SVI_REQUIRE(d, "svi_fastblend_step: null descriptor");
  SVI_REQUIRE(d->src_guide && d->src_style && d->tgt_guide && d->tgt_style && d->nnf_in && d->nnf_out && d->err_out,
              "svi_fastblend_step: null pointer");
  SVI_REQUIRE(d->B > 0 && d->H > 0 && d->W > 0 && d->B <= 65535, "svi_fastblend_step: bad shape");
  SVI_REQUIRE(d->patch_size >= 1 && d->patch_size <= SVI_FASTBLEND_MAX_PATCH, "svi_fastblend_step: patch size out of range");
  SVI_REQUIRE(d->mode == SVI_FASTBLEND_CURRENT || d->mode == SVI_FASTBLEND_NEIGHBOUR || d->mode == SVI_FASTBLEND_RANDOM,
              "svi_fastblend_step: unknown mode");
  SVI_REQUIRE(d->mode == SVI_FASTBLEND_CURRENT || d->err_in, "svi_fastblend_step: err_in is null");
  SVI_REQUIRE(d->mode != SVI_FASTBLEND_NEIGHBOUR || (d->dir >= 0 && d->dir <= 3), "svi_fastblend_step: dir must be 0..3");
  SVI_REQUIRE(d->mode != SVI_FASTBLEND_RANDOM || (d->radius >= 0 && d->radius < (1 << 20)), "svi_fastblend_step: bad radius");
  SVI_REQUIRE((const void*)d->nnf_in != (const void*)d->nnf_out && (const void*)d->err_in != (const void*)d->err_out,
              "svi_fastblend_step: outputs must not alias inputs");
  SVI_REQUIRE((long long)d->B * d->H * d->W * 2 < (1LL << 32), "svi_fastblend_step: batch too large for the stream index");
  const uintptr_t f = reinterpret_cast<uintptr_t>(d->src_guide) | reinterpret_cast<uintptr_t>(d->src_style) |
                      reinterpret_cast<uintptr_t>(d->tgt_guide) | reinterpret_cast<uintptr_t>(d->tgt_style);
  const uintptr_t n = reinterpret_cast<uintptr_t>(d->nnf_in) | reinterpret_cast<uintptr_t>(d->nnf_out);
  SVI_REQUIRE((f & 15) == 0 && (n & 7) == 0, "svi_fastblend_step: frames must be 16-byte and fields 8-byte aligned");
  const int r = (d->patch_size - 1) / 2, side = fastblend::kTile + 2 * r;
  const size_t smem = (size_t)2 * side * side * sizeof(float4);
  if (smem > 48 * 1024) {   // patches above 21 taps a side: opt in to the larger window (on the current device)
    cudaError_t e = cudaFuncSetAttribute(fastblend::step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    SVI_REQUIRE(e == cudaSuccess, "svi_fastblend_step: cannot reserve %zu bytes of shared memory", smem);
  }
  const dim3 grid((d->W + fastblend::kTile - 1) / fastblend::kTile, (d->H + fastblend::kTile - 1) / fastblend::kTile, d->B);
  fastblend::step_kernel<<<grid, dim3(fastblend::kTile, fastblend::kTile), smem, static_cast<cudaStream_t>(stream)>>>(*d);
  SVI_CUDA_LAUNCH_CHECK("svi_fastblend_step");
  return SVI_OK;
}

extern "C" int svi_fastblend_table(const svi_fastblend_table_desc* d, void* stream) {
  SVI_REQUIRE(d && d->a && d->b && d->out, "svi_fastblend_table: null pointer");
  SVI_REQUIRE(d->n_pix > 0 && d->n_pix < (1LL << 40), "svi_fastblend_table: bad pixel count");
  auto ok_type = [](int t) { return t == SVI_FASTBLEND_U8 || t == SVI_FASTBLEND_F32 || t == SVI_FASTBLEND_F64; };
  SVI_REQUIRE(ok_type(d->a_type) && ok_type(d->b_type) && (!d->c || ok_type(d->c_type)), "svi_fastblend_table: bad operand type");
  if (d->op == SVI_FASTBLEND_MEAN || d->op == SVI_FASTBLEND_HALF) {
    SVI_REQUIRE(!d->c && d->out_type == SVI_FASTBLEND_F32 && d->b_type == SVI_FASTBLEND_F32 && d->a_type != SVI_FASTBLEND_F64 &&
                    (d->op == SVI_FASTBLEND_HALF || d->a_type == SVI_FASTBLEND_F32),
                "svi_fastblend_table: MEAN takes f32 a and b, HALF uint8 or f32 a and f32 b, both give f32");
  } else {
    SVI_REQUIRE(d->op == SVI_FASTBLEND_WSUM, "svi_fastblend_table: unknown op");
    SVI_REQUIRE(ok_type(d->out_type), "svi_fastblend_table: bad output type");
  }
  fastblend::table_kernel<<<fastblend::blocks(d->n_pix * 4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(*d);
  SVI_CUDA_LAUNCH_CHECK("svi_fastblend_table");
  return SVI_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// The balanced / accurate / interpolation modes (include/svi_b200_fastblend_modes.h).
namespace svi {
namespace fastblend {

__global__ void candidate_kernel(svi_fastblend_candidate_desc d) {
  const long long n = (long long)d.B * d.H * d.W;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int H = d.H, W = d.W;
  const long long hw = (long long)H * W;
  const int b = (int)(i / hw);
  const long long pix = i - b * hw;
  const int y = (int)(pix / W), x = (int)(pix % W);
  const int2* nnf = reinterpret_cast<const int2*>(d.nnf_in);
  const long long frame = b * hw;
  int2 m;
  if (d.mode == SVI_FASTBLEND_TRACK) {
    int src;
    if (d.pairwise) {
      const int parity = b & 1, count = (d.B - parity + 1) / 2;
      src = 2 * min(max(b / 2 + d.shift, 0), count - 1) + parity;
    } else {
      src = min(max(b + d.shift, 0), d.B - 1);
    }
    m = nnf[src * hw + pix];   // fields are inside the frame already: no clamp, as the reference's track_step
  } else if (d.mode == SVI_FASTBLEND_NEIGHBOUR) {
    switch (d.dir) {
      case 0: m = nnf[frame + (long long)max(y - 1, 0) * W + x]; m.x += 1; break;
      case 1: m = nnf[frame + (long long)y * W + max(x - 1, 0)]; m.y += 1; break;
      case 2: m = nnf[frame + (long long)min(y + 1, H - 1) * W + x]; m.x -= 1; break;
      default: m = nnf[frame + (long long)y * W + min(x + 1, W - 1)]; m.y -= 1; break;
    }
    m = make_int2(min(max(m.x, 0), H - 1), min(max(m.y, 0), W - 1));
  } else {
    const uint32_t span = (uint32_t)(2 * d.radius + 1);
    const uint32_t e0 = (uint32_t)(i * 2);
    m = nnf[i];
    m.x += -d.radius + (int)(stream_u(d.draw, e0) % span);
    m.y += -d.radius + (int)(stream_u(d.draw, e0 + 1) % span);
    m = make_int2(min(max(m.x, 0), H - 1), min(max(m.y, 0), W - 1));
  }
  reinterpret_cast<int2*>(d.nnf_out)[i] = m;
}

// The error of a given candidate and the select.  The block layout is the step kernel's: a 16 x 16 tile of one frame,
// its target guide window (and target style window, unless pairwise) with an r-pixel halo in shared memory.
__global__ void __launch_bounds__(kTile * kTile) select_kernel(svi_fastblend_select_desc d) {
  extern __shared__ float4 win[];
  const int H = d.H, W = d.W, r = (d.patch_size - 1) / 2, side = kTile + 2 * r;
  float4* tg = win;
  float4* ts = win + side * side;
  const int b = blockIdx.z, y0 = blockIdx.y * kTile, x0 = blockIdx.x * kTile;
  const long long hw = (long long)H * W, frame = (long long)b * hw;
  const float4* tgt_guide = reinterpret_cast<const float4*>(d.tgt_guide) + frame;
  const float4* tgt_style = d.pairwise ? nullptr : reinterpret_cast<const float4*>(d.tgt_style) + (d.style_shared ? 0 : frame);
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j = threadIdx.y * kTile + threadIdx.x; j < side * side; j += kTile * kTile) {
    const int wy = y0 - r + j / side, wx = x0 - r + j % side;
    const bool in = wy >= 0 && wy < H && wx >= 0 && wx < W;
    tg[j] = in ? __ldg(tgt_guide + (long long)wy * W + wx) : zero;
    if (tgt_style) ts[j] = in ? __ldg(tgt_style + (long long)wy * W + wx) : zero;
  }
  __syncthreads();
  const int y = y0 + threadIdx.y, x = x0 + threadIdx.x;
  if (y >= H || x >= W) return;
  const long long pix = (long long)y * W + x, o = frame + pix;
  const int2* cand = reinterpret_cast<const int2*>(d.cand);
  const int2 c = cand[o];
  const float4* sg = reinterpret_cast<const float4*>(d.src_guide) + frame;
  float eg = 0.f, es = 0.f;
  if (!d.pairwise) {
    const float4* ss = reinterpret_cast<const float4*>(d.src_style) + frame;
    for (int px = -r; px <= r; px++) {
      const int sy = c.x + px;
      const bool row_in = sy >= 0 && sy < H;
      const float4* tg_row = tg + (threadIdx.y + r + px) * side + threadIdx.x + r;
      const float4* ts_row = ts + (threadIdx.y + r + px) * side + threadIdx.x + r;
      for (int py = -r; py <= r; py++) {
        const int sx = c.y + py;
        const bool in = row_in && sx >= 0 && sx < W;
        const long long s = (long long)sy * W + sx;
        eg = sq_acc(eg, tg_row[py], in ? __ldg(sg + s) : zero);
        es = sq_acc(es, ts_row[py], in ? __ldg(ss + s) : zero);
      }
    }
  } else {
    // both members of pair k evaluate the pair's style term in the same order, so they hold the same bits
    const long long fa = (long long)(b & ~1) * hw, fb = fa + hw;
    const int2 ca = cand[fa + pix], cb = cand[fb + pix];
    const float4* sa = reinterpret_cast<const float4*>(d.src_style) + fa;
    const float4* sb = reinterpret_cast<const float4*>(d.src_style) + fb;
    for (int px = -r; px <= r; px++) {
      const int sy = c.x + px, ay = ca.x + px, by = cb.x + px;
      const float4* tg_row = tg + (threadIdx.y + r + px) * side + threadIdx.x + r;
      for (int py = -r; py <= r; py++) {
        const int sx = c.y + py, ax = ca.y + py, bx = cb.y + py;
        const bool in = sy >= 0 && sy < H && sx >= 0 && sx < W;
        const bool in_a = ay >= 0 && ay < H && ax >= 0 && ax < W;
        const bool in_b = by >= 0 && by < H && bx >= 0 && bx < W;
        eg = sq_acc(eg, tg_row[py], in ? __ldg(sg + (long long)sy * W + sx) : zero);
        es = sq_acc(es, in_a ? __ldg(sa + (long long)ay * W + ax) : zero, in_b ? __ldg(sb + (long long)by * W + bx) : zero);
      }
    }
  }
  const float e = __fadd_rn(__fmul_rn(eg, d.guide_weight), es);
  int2* nnf_out = reinterpret_cast<int2*>(d.nnf_out);
  if (!d.select || e < d.err_in[o]) {
    nnf_out[o] = c;
    d.err_out[o] = e;
  } else {
    nnf_out[o] = reinterpret_cast<const int2*>(d.nnf_in)[o];
    d.err_out[o] = d.err_in[o];
  }
}

__global__ void batch_mean_kernel(const float* __restrict__ src, int B, long long n, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 4) return;
  if ((i & 3) == 3) { out[i] = 0.f; return; }
  float s = src[i];
  for (int b = 1; b < B; b++) s = __fadd_rn(s, src[(long long)b * n * 4 + i]);
  out[i] = __fdiv_rn(s, (float)B);
}

__global__ void running_mean_kernel(const void* frame, int frame_type, double s, const float* __restrict__ result,
                                    float divisor, long long n, double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 4) return;
  if ((i & 3) == 3) { out[i] = 0.0; return; }
  const double f = frame_type == SVI_FASTBLEND_F64 ? static_cast<const double*>(frame)[i]
                                                   : (double)static_cast<const float*>(frame)[i];
  out[i] = __dadd_rn(__dmul_rn(f, s), (double)__fdiv_rn(result[i], divisor));
}

__global__ void to_u8_kernel(const void* a, int a_type, long long n, uint8_t* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 3) return;
  const long long e = (i / 3) * 4 + i % 3;
  const double v = a_type == SVI_FASTBLEND_F64 ? static_cast<const double*>(a)[e] : (double)static_cast<const float*>(a)[e];
  out[i] = (uint8_t)(int)fmin(fmax(v, 0.0), 255.0);
}

}  // namespace fastblend
}  // namespace svi

extern "C" int svi_fastblend_candidate(const svi_fastblend_candidate_desc* d, void* stream) {
  SVI_REQUIRE(d && d->nnf_in && d->nnf_out && d->nnf_in != d->nnf_out, "svi_fastblend_candidate: null or aliased field");
  SVI_REQUIRE(d->B > 0 && d->H > 0 && d->W > 0, "svi_fastblend_candidate: bad shape");
  SVI_REQUIRE((long long)d->B * d->H * d->W * 2 < (1LL << 32), "svi_fastblend_candidate: batch too large for the stream index");
  SVI_REQUIRE(d->mode == SVI_FASTBLEND_NEIGHBOUR || d->mode == SVI_FASTBLEND_RANDOM || d->mode == SVI_FASTBLEND_TRACK,
              "svi_fastblend_candidate: unknown mode");
  SVI_REQUIRE(d->mode != SVI_FASTBLEND_NEIGHBOUR || (d->dir >= 0 && d->dir <= 3), "svi_fastblend_candidate: dir must be 0..3");
  SVI_REQUIRE(d->mode != SVI_FASTBLEND_RANDOM || (d->radius >= 0 && d->radius < (1 << 20)), "svi_fastblend_candidate: bad radius");
  SVI_REQUIRE(d->mode != SVI_FASTBLEND_TRACK || (d->shift != 0 && (!d->pairwise || d->B % 2 == 0)),
              "svi_fastblend_candidate: tracking needs a nonzero shift (and an even batch when pairwise)");
  SVI_REQUIRE(((reinterpret_cast<uintptr_t>(d->nnf_in) | reinterpret_cast<uintptr_t>(d->nnf_out)) & 7) == 0,
              "svi_fastblend_candidate: fields must be 8-byte aligned");
  fastblend::candidate_kernel<<<fastblend::blocks((long long)d->B * d->H * d->W, 256), 256, 0,
                                static_cast<cudaStream_t>(stream)>>>(*d);
  SVI_CUDA_LAUNCH_CHECK("svi_fastblend_candidate");
  return SVI_OK;
}

extern "C" int svi_fastblend_select(const svi_fastblend_select_desc* d, void* stream) {
  SVI_REQUIRE(d, "svi_fastblend_select: null descriptor");
  SVI_REQUIRE(d->src_guide && d->src_style && d->tgt_guide && d->cand && d->nnf_out && d->err_out &&
                  (d->pairwise || d->tgt_style) && (!d->select || (d->nnf_in && d->err_in)),
              "svi_fastblend_select: null pointer");
  SVI_REQUIRE(d->B > 0 && d->H > 0 && d->W > 0 && d->B <= 65535, "svi_fastblend_select: bad shape");
  SVI_REQUIRE(d->patch_size >= 1 && d->patch_size <= SVI_FASTBLEND_MAX_PATCH, "svi_fastblend_select: patch size out of range");
  SVI_REQUIRE((d->select == 0 || d->select == 1) && (d->style_shared == 0 || d->style_shared == 1) &&
                  (d->pairwise == 0 || d->pairwise == 1),
              "svi_fastblend_select: select, style_shared and pairwise are 0 or 1");
  SVI_REQUIRE(!d->pairwise || d->B % 2 == 0, "svi_fastblend_select: the pairwise error needs an even batch");
  SVI_REQUIRE((const void*)d->nnf_out != (const void*)d->cand && (const void*)d->nnf_out != (const void*)d->nnf_in &&
                  (const void*)d->err_out != (const void*)d->err_in,
              "svi_fastblend_select: outputs must not alias inputs");
  const uintptr_t f = reinterpret_cast<uintptr_t>(d->src_guide) | reinterpret_cast<uintptr_t>(d->src_style) |
                      reinterpret_cast<uintptr_t>(d->tgt_guide) | reinterpret_cast<uintptr_t>(d->tgt_style);
  const uintptr_t n = reinterpret_cast<uintptr_t>(d->cand) | reinterpret_cast<uintptr_t>(d->nnf_in) |
                      reinterpret_cast<uintptr_t>(d->nnf_out);
  SVI_REQUIRE((f & 15) == 0 && (n & 7) == 0, "svi_fastblend_select: frames must be 16-byte and fields 8-byte aligned");
  const int r = (d->patch_size - 1) / 2, side = fastblend::kTile + 2 * r;
  const size_t smem = (size_t)2 * side * side * sizeof(float4);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(fastblend::select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    SVI_REQUIRE(e == cudaSuccess, "svi_fastblend_select: cannot reserve %zu bytes of shared memory", smem);
  }
  const dim3 grid((d->W + fastblend::kTile - 1) / fastblend::kTile, (d->H + fastblend::kTile - 1) / fastblend::kTile, d->B);
  fastblend::select_kernel<<<grid, dim3(fastblend::kTile, fastblend::kTile), smem, static_cast<cudaStream_t>(stream)>>>(*d);
  SVI_CUDA_LAUNCH_CHECK("svi_fastblend_select");
  return SVI_OK;
}

extern "C" int svi_fastblend_batch_mean(const float* src, int32_t B, int64_t n_pix, float* out, void* stream) {
  SVI_REQUIRE(src && out && (const void*)src != (const void*)out, "svi_fastblend_batch_mean: null or aliased pointer");
  SVI_REQUIRE(B > 0 && n_pix > 0 && n_pix < (1LL << 40), "svi_fastblend_batch_mean: bad shape");
  fastblend::batch_mean_kernel<<<fastblend::blocks(n_pix * 4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, B, (long long)n_pix, out);
  SVI_CUDA_LAUNCH_CHECK("svi_fastblend_batch_mean");
  return SVI_OK;
}

extern "C" int svi_fastblend_running_mean(const void* frame, int32_t frame_type, double s, const float* result,
                                          float divisor, int64_t n_pix, double* out, void* stream) {
  SVI_REQUIRE(frame && result && out, "svi_fastblend_running_mean: null pointer");
  SVI_REQUIRE(frame_type == SVI_FASTBLEND_U8 || frame_type == SVI_FASTBLEND_F64,
              "svi_fastblend_running_mean: the frame is uint8 (held as f32) or f64");
  SVI_REQUIRE(n_pix > 0 && n_pix < (1LL << 40), "svi_fastblend_running_mean: bad pixel count");
  fastblend::running_mean_kernel<<<fastblend::blocks(n_pix * 4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      frame, frame_type, s, result, divisor, (long long)n_pix, out);
  SVI_CUDA_LAUNCH_CHECK("svi_fastblend_running_mean");
  return SVI_OK;
}

extern "C" int svi_fastblend_to_u8(const void* a, int32_t a_type, int64_t n_pix, uint8_t* out, void* stream) {
  SVI_REQUIRE(a && out, "svi_fastblend_to_u8: null pointer");
  SVI_REQUIRE(a_type == SVI_FASTBLEND_U8 || a_type == SVI_FASTBLEND_F32 || a_type == SVI_FASTBLEND_F64,
              "svi_fastblend_to_u8: bad operand type");
  SVI_REQUIRE(n_pix > 0 && n_pix < (1LL << 40), "svi_fastblend_to_u8: bad pixel count");
  fastblend::to_u8_kernel<<<fastblend::blocks(n_pix * 3, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      a, a_type, (long long)n_pix, out);
  SVI_CUDA_LAUNCH_CHECK("svi_fastblend_to_u8");
  return SVI_OK;
}
