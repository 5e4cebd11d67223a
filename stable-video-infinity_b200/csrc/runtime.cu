// Host-side runtime of the C ABI: error strings, device queries and the TMA tensor-map encoder
// (cuTensorMapEncodeTiled is fetched from the driver at run time, so the library links only cudart).
#include <stdarg.h>
#include <string.h>

#include "common.cuh"
#include "../../include/svi_b200.h"

namespace svi {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) {
    set_last_error("cuTensorMapEncodeTiled not available from the driver (%s)",
                   e != cudaSuccess ? cudaGetErrorString(e) : "entry point missing");
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

int make_tmap_2d(CUtensorMap* map, const void* base, int elem_bytes, uint64_t inner, uint64_t outer,
                 uint64_t row_pitch_bytes, uint32_t box_inner, uint32_t box_outer, bool swizzle_128b) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return SVI_ERR_DRIVER;
  CUtensorMapDataType dt;
  if (elem_bytes == 2) dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  else if (elem_bytes == 4) dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  else if (elem_bytes == 1) dt = CU_TENSOR_MAP_DATA_TYPE_UINT8;
  else { set_last_error("make_tmap_2d: unsupported element size %d", elem_bytes); return SVI_ERR_INVALID_ARG; }
  if (box_inner * (uint32_t)elem_bytes > 128 || box_outer > 256) {
    set_last_error("make_tmap_2d: box %ux%u too large (inner box at most 128 bytes, outer at most 256 rows)", box_inner,
                   box_outer);
    return SVI_ERR_INVALID_ARG;
  }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_pitch_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, dt, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_128b ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed (CUresult %d): base=%p inner=%llu outer=%llu pitch=%llu box=%ux%u",
                   (int)r, base, (unsigned long long)inner, (unsigned long long)outer,
                   (unsigned long long)row_pitch_bytes, box_inner, box_outer);
    return SVI_ERR_DRIVER;
  }
  return SVI_OK;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
    set_last_error("sm_count: cudaGetDevice failed");
    return -1;
  }
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      set_last_error("sm_count: cudaDeviceGetAttribute failed");
      return -1;
    }
    cached[dev] = n;
  }
  return cached[dev];
}

}  // namespace svi

extern "C" int svi_abi_version(void) { return 4; }  // 4: LayerNorm-fold GEMM epilogues, conv epilogue feeding the next conv, svi_frames_to_uint8
extern "C" const char* svi_last_error(void) { return svi::g_err; }
extern "C" int svi_sm_count(void) { return svi::sm_count(); }
