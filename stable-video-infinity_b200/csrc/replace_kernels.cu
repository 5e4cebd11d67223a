// Replace-Anyone input staging: the masked video for the VAE encoder and the learn-in stem's first frame ring, in one
// pass (include/svi_b200_replace.h).
//
// An HBM-bound stream: one thread per pixel of one frame reads its three colour samples and its segmentation value and
// writes three f32 samples and one 8-byte group of four bf16 ring channels.  No atomics, a grid that covers every pixel
// once: a pixel's bytes depend only on its inputs.
#include "common.cuh"
#include "../../include/svi_b200_replace.h"

namespace svi {
namespace replace {

constexpr int kThreads = 256;

template <bool kU8>
__global__ void __launch_bounds__(kThreads)
mask_stage_kernel(const float* __restrict__ video, const void* __restrict__ seg, long long n, float* __restrict__ masked,
                  uint2* __restrict__ ring, long long ring_stride) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float s = kU8 ? (float)__ldg(static_cast<const unsigned char*>(seg) + i) : __ldg(static_cast<const float*>(seg) + i);
  const float keep = __fdiv_rn(s, 255.0f) > 0.0f ? 0.0f : 1.0f;
  float m[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) m[c] = __fmul_rn(__ldg(video + c * n + i), keep);
  if (masked) {
#pragma unroll
    for (int c = 0; c < 3; ++c) masked[c * n + i] = m[c];
  }
  ring[i * ring_stride] = make_uint2(pack_bf16x2(m[0], m[1]), pack_bf16x2(m[2], keep));
}

inline bool overlap(const void* a, long long a_bytes, const void* b, long long b_bytes) {
  const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), b0 = reinterpret_cast<uintptr_t>(b);
  return a0 < b0 + (uintptr_t)b_bytes && b0 < a0 + (uintptr_t)a_bytes;
}

}  // namespace replace
}  // namespace svi

using namespace svi;

extern "C" int svi_replace_mask_stage(const float* video, const void* seg, int32_t seg_type, int32_t T, int64_t hw,
                                      float* masked, void* ring, int32_t ldr, void* stream) {
  SVI_REQUIRE(video && seg && ring, "svi_replace_mask_stage: null pointer");
  SVI_REQUIRE(seg_type == SVI_SEG_U8 || seg_type == SVI_SEG_F32, "svi_replace_mask_stage: seg_type must be SVI_SEG_U8 "
              "or SVI_SEG_F32 (got %d)", seg_type);
  SVI_REQUIRE(T > 0 && hw > 0, "svi_replace_mask_stage: bad shape (T %d, hw %lld)", T, (long long)hw);
  SVI_REQUIRE(ldr >= 4 && ldr % 4 == 0, "svi_replace_mask_stage: ldr must be a multiple of 4 and at least 4 (got %d)", ldr);
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(ring) & 7) == 0, "svi_replace_mask_stage: ring must be 8-byte aligned");
  const long long n = (long long)T * hw;
  const long long video_bytes = 3 * n * 4, seg_bytes = n * (seg_type == SVI_SEG_U8 ? 1 : 4), ring_bytes = n * ldr * 2;
  SVI_REQUIRE(!replace::overlap(ring, ring_bytes, video, video_bytes) && !replace::overlap(ring, ring_bytes, seg, seg_bytes),
              "svi_replace_mask_stage: ring must not overlap video or seg");
  SVI_REQUIRE(!masked || (!replace::overlap(masked, video_bytes, video, video_bytes) &&
                          !replace::overlap(masked, video_bytes, seg, seg_bytes) &&
                          !replace::overlap(masked, video_bytes, ring, ring_bytes)),
              "svi_replace_mask_stage: masked must not overlap video, seg or ring");
  const long long blocks = (n + replace::kThreads - 1) / replace::kThreads;
  SVI_REQUIRE(blocks <= 0x7fffffffLL, "svi_replace_mask_stage: too many pixels");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  uint2* r = static_cast<uint2*>(ring);
  if (seg_type == SVI_SEG_U8)
    replace::mask_stage_kernel<true><<<(unsigned)blocks, replace::kThreads, 0, s>>>(video, seg, n, masked, r, ldr / 4);
  else
    replace::mask_stage_kernel<false><<<(unsigned)blocks, replace::kThreads, 0, s>>>(video, seg, n, masked, r, ldr / 4);
  SVI_CUDA_LAUNCH_CHECK("svi_replace_mask_stage");
  return SVI_OK;
}
