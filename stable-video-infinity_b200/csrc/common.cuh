// Shared device/host helpers for the sm_90a kernels of the SVI clip-denoising hot path: inline PTX for mbarrier and TMA
// (cp.async.bulk.tensor), register redistribution, and the math helpers of the epilogues.  wgmma lives in wgmma.cuh.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace svi {

// ---------------------------------------------------------------------------------------------
// status codes of the C ABI (include/svi_b200.h)
// ---------------------------------------------------------------------------------------------
enum : int {
  SVI_OK = 0,
  SVI_ERR_INVALID_ARG = -1,
  SVI_ERR_UNSUPPORTED = -2,
  SVI_ERR_DRIVER = -3,
  SVI_ERR_LAUNCH = -4,
};

void set_last_error(const char* fmt, ...);

#define SVI_REQUIRE(cond, ...)                 \
  do {                                         \
    if (!(cond)) {                             \
      ::svi::set_last_error(__VA_ARGS__);      \
      return ::svi::SVI_ERR_INVALID_ARG;       \
    }                                          \
  } while (0)

#define SVI_CUDA_LAUNCH_CHECK(name)                                                    \
  do {                                                                                 \
    cudaError_t e__ = cudaGetLastError();                                              \
    if (e__ != cudaSuccess) {                                                          \
      ::svi::set_last_error("%s: launch failed: %s", name, cudaGetErrorString(e__));   \
      return ::svi::SVI_ERR_LAUNCH;                                                    \
    }                                                                                  \
  } while (0)

// Encode a 2-D bf16 (or fp32) row-major tensor map with 128-byte swizzle. `inner` is the contiguous
// dimension. Returns SVI_OK or an error code (message via set_last_error).
int make_tmap_2d(CUtensorMap* map, const void* base, int elem_bytes, uint64_t inner, uint64_t outer,
                 uint64_t row_pitch_bytes, uint32_t box_inner, uint32_t box_outer);

int sm_count();

#ifdef __CUDACC__
// ---------------------------------------------------------------------------------------------
// generic
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

// ---------------------------------------------------------------------------------------------
// mbarrier and TMA (32-bit shared-memory addresses: no generic 64-bit pointer arithmetic in the hot warps)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void mbar_init_a(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx_a(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive_a(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) break;
    // no printf here: a function call inside a wgmma pipeline makes ptxas serialise every wgmma of the kernel
    if (++spins > (1u << 26)) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d_a(uint32_t smem_dst, const CUtensorMap* m, uint32_t bar, int c_inner,
                                              int c_outer) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_dst),
      "l"(m), "r"(bar), "r"(c_inner), "r"(c_outer)
      : "memory");
}
// Register redistribution between the warpgroups of a warp-specialised CTA (producer warpgroup gives, consumers take).
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// The library is compiled WITHOUT --use_fast_math (fp32 norms / residual math stay IEEE); the two approximations the hot
// epilogues want are explicit: MUFU.EX2 (rel. error 2^-22) and MUFU.RCP (1 ulp).
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float gelu_tanh(float x) {
  // 0.5 x (1 + tanh(u)) = x * sigmoid(2u),  u = sqrt(2/pi) (x + 0.044715 x^3)   (torch.nn.GELU(approximate='tanh'));
  // two MUFU ops, relative error ~1e-6 (tanh.approx, which --use_fast_math would pick, is good to 2^-11 only)
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u = k0 * (x + k1 * x * x * x);
  return x * fast_rcp(1.0f + fast_ex2(-2.885390081777927f * u));   // exp(-2u) = 2^(-2 log2(e) u)
}
__device__ __forceinline__ float silu(float x) { return x * fast_rcp(1.0f + fast_ex2(-1.4426950408889634f * x)); }
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.7071067811865476f)); }
#endif  // __CUDACC__

}  // namespace svi
