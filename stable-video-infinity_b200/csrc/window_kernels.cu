// UniAnimate-DiT long-video windows: per-frame f32 sum of the stepped windows and its normalisation
// (include/svi_b200_unianimate.h).
//
// Both kernels are HBM-bound streams of float4: one thread per four consecutive pixels of one (channel, frame), a grid
// that covers every element once, no atomics.  An element's value depends only on its inputs and the order in which
// the host launches the windows, never on the grid.
#include "common.cuh"
#include "../../include/svi_b200_unianimate.h"

namespace svi {
namespace window {

constexpr int kThreads = 256;

__global__ void accumulate_kernel(const float4* __restrict__ win, int cs, long long hw4, int skip, int n_frames,
                                  float4* __restrict__ sum, int F, int start, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long p = i % hw4;
  const long long r = i / hw4;
  const int j = skip + (int)(r % n_frames);
  const long long c = r / n_frames;
  const float4 w = __ldg(win + (c * cs + j) * hw4 + p);
  float4* s = sum + (c * F + start + j) * hw4 + p;
  float4 v = *s;
  v.x = __fadd_rn(v.x, w.x);
  v.y = __fadd_rn(v.y, w.y);
  v.z = __fadd_rn(v.z, w.z);
  v.w = __fadd_rn(v.w, w.w);
  *s = v;
}

__global__ void normalize_kernel(const float4* sum, const int32_t* __restrict__ count, int F, long long hw4, float4* out,
                                 long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float n = (float)__ldg(count + (int)((i / hw4) % F));
  const float4 v = sum[i];
  out[i] = make_float4(__fdiv_rn(v.x, n), __fdiv_rn(v.y, n), __fdiv_rn(v.z, n), __fdiv_rn(v.w, n));
}

inline unsigned blocks(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

inline bool overlap(const void* a, long long a_bytes, const void* b, long long b_bytes) {
  const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), b0 = reinterpret_cast<uintptr_t>(b);
  return a0 < b0 + (uintptr_t)b_bytes && b0 < a0 + (uintptr_t)a_bytes;
}

}  // namespace window
}  // namespace svi

using namespace svi;

extern "C" int svi_window_accumulate(const float* win, int32_t C, int32_t cs, int64_t hw, int32_t skip, float* sum,
                                     int32_t F, int32_t start, void* stream) {
  SVI_REQUIRE(win && sum, "svi_window_accumulate: null pointer");
  SVI_REQUIRE(C > 0 && cs > 0 && F > 0 && hw > 0, "svi_window_accumulate: bad shape");
  SVI_REQUIRE(hw % 4 == 0, "svi_window_accumulate: hw must be a multiple of 4 (got %lld)", (long long)hw);
  SVI_REQUIRE(skip >= 0 && skip < cs, "svi_window_accumulate: need 0 <= skip < cs (skip %d, cs %d)", skip, cs);
  SVI_REQUIRE(start >= 0 && (long long)start + cs <= F, "svi_window_accumulate: window %d..%d outside %d frames", start,
              start + cs - 1, F);
  SVI_REQUIRE(window::aligned16(win) && window::aligned16(sum), "svi_window_accumulate: pointers must be 16-byte aligned");
  const long long win_bytes = (long long)C * cs * hw * 4, sum_bytes = (long long)C * F * hw * 4;
  SVI_REQUIRE(!window::overlap(win, win_bytes, sum, sum_bytes), "svi_window_accumulate: win must not overlap sum");
  const long long hw4 = hw / 4, total = (long long)C * (cs - skip) * hw4;
  SVI_REQUIRE(window::blocks(total) <= 0x7fffffffLL, "svi_window_accumulate: too many elements");
  window::accumulate_kernel<<<window::blocks(total), window::kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(win), cs, hw4, skip, cs - skip, reinterpret_cast<float4*>(sum), F, start, total);
  SVI_CUDA_LAUNCH_CHECK("svi_window_accumulate");
  return SVI_OK;
}

extern "C" int svi_window_normalize(const float* sum, const int32_t* count, int32_t C, int32_t F, int64_t hw, float* out,
                                    void* stream) {
  SVI_REQUIRE(sum && count && out, "svi_window_normalize: null pointer");
  SVI_REQUIRE(C > 0 && F > 0 && hw > 0, "svi_window_normalize: bad shape");
  SVI_REQUIRE(hw % 4 == 0, "svi_window_normalize: hw must be a multiple of 4 (got %lld)", (long long)hw);
  SVI_REQUIRE(window::aligned16(sum) && window::aligned16(out), "svi_window_normalize: pointers must be 16-byte aligned");
  const long long bytes = (long long)C * F * hw * 4;
  SVI_REQUIRE((const void*)sum == (const void*)out || !window::overlap(sum, bytes, out, bytes),
              "svi_window_normalize: out must be sum itself or not overlap it");
  SVI_REQUIRE(!window::overlap(count, (long long)F * 4, out, bytes), "svi_window_normalize: count must not overlap out");
  const long long hw4 = hw / 4, total = (long long)C * F * hw4;
  SVI_REQUIRE(window::blocks(total) <= 0x7fffffffLL, "svi_window_normalize: too many elements");
  window::normalize_kernel<<<window::blocks(total), window::kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(sum), count, F, hw4, reinterpret_cast<float4*>(out), total);
  SVI_CUDA_LAUNCH_CHECK("svi_window_normalize");
  return SVI_OK;
}
