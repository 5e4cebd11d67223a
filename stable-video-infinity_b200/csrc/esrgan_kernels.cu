// ESRGAN (RRDBNet): staging of the uint8 frames as conv_first's operand (include/svi_b200_esrgan.h).  The convolutions
// run on the conv mainloop of conv3d_wgmma.cu (svi_esrgan_conv2d).
//
// v = c / 255 as numpy's float32 division (ESRGAN.process_image), rounded to bf16; channels 3..7 are zero.  The rounding
// study (DESIGN.md §4) found no consistent gain from a two-term hi | lo operand here.  One thread per pixel, one 16-byte
// store.
#include "common.cuh"
#include "../../include/svi_b200_esrgan.h"

namespace svi {
namespace esrgan {

__global__ void stage_frames_kernel(const uint8_t* __restrict__ rgb, long long n, uint4* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* s = rgb + 3 * i;
  const float r = __fdiv_rn((float)s[0], 255.f), g = __fdiv_rn((float)s[1], 255.f), b = __fdiv_rn((float)s[2], 255.f);
  out[i] = make_uint4(pack_bf16x2(r, g), pack_bf16x2(b, 0.f), 0u, 0u);
}

}  // namespace esrgan
}  // namespace svi

extern "C" int svi_esrgan_stage_frames(const uint8_t* rgb, int64_t n_pix, void* out, void* stream) {
  using namespace svi;
  SVI_REQUIRE(rgb && out, "svi_esrgan_stage_frames: null pointer");
  SVI_REQUIRE(n_pix >= 0 && n_pix < (1LL << 40), "svi_esrgan_stage_frames: bad pixel count");
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "svi_esrgan_stage_frames: out must be 16-byte aligned");
  if (n_pix == 0) return SVI_OK;
  const int threads = 256;
  esrgan::stage_frames_kernel<<<(unsigned)((n_pix + threads - 1) / threads), threads, 0, static_cast<cudaStream_t>(stream)>>>(
      rgb, (long long)n_pix, reinterpret_cast<uint4*>(out));
  SVI_CUDA_LAUNCH_CHECK("svi_esrgan_stage_frames");
  return SVI_OK;
}
