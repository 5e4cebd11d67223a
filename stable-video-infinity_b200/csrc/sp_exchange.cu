// Sequence-parallel K|V exchange over NVLink peer memory (one process per GPU).
//
// Replaces the reference's xfuser wiring for the self-attention exchange (diffsynth/distributed/
// xdit_context_parallel.py:108-129: xFuserLongContextAttention = Ulysses all-to-all / ring passes through NCCL).
//
// Every rank of a sequence-parallel group owns one symmetric allocation (cudaMalloc, exported with a CUDA IPC
// handle and mapped by its peers): the full [L, 2d] K|V buffer of a layer plus one 32-bit arrival flag per source
// rank.  After a rank has produced its own rows (K|V GEMM + RMSNorm/RoPE epilogue kernels) it PUSHES them into the
// same rows of every peer's buffer with copy-engine peer copies on a side stream, each followed by a 4-byte copy
// of the layer's epoch number into the peer's flag word (same stream, so it lands after the rows; no SM is
// involved, so the push can never wait for an SM that a spinning attention CTA holds).  The consumer is the attention kernel itself (attn_wgmma.cu): its TMA producer warp
// starts on the rank's own rows and polls a chunk's flag (ld.acquire.sys) only when the K/V stream reaches rows
// owned by another rank, so the transfer overlaps the attention math tile by tile and no SM time is spent copying.
#include <string.h>

#include "common.cuh"
#include "../../include/svi_b200.h"

extern "C" int svi_sp_alloc(size_t bytes, void** ptr, unsigned char* handle64) {
  using namespace svi;
  SVI_REQUIRE(ptr && handle64 && bytes > 0, "svi_sp_alloc: bad arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle is 64 bytes");
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {
    set_last_error("svi_sp_alloc: cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    return SVI_ERR_DRIVER;
  }
  e = cudaMemset(p, 0, bytes);
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    set_last_error("svi_sp_alloc: cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
    cudaFree(p);
    return SVI_ERR_DRIVER;
  }
  memcpy(handle64, &h, 64);
  *ptr = p;
  return SVI_OK;
}

extern "C" int svi_sp_free(void* ptr) {
  using namespace svi;
  cudaError_t e = cudaFree(ptr);
  if (e != cudaSuccess) {
    set_last_error("svi_sp_free: %s", cudaGetErrorString(e));
    return SVI_ERR_DRIVER;
  }
  return SVI_OK;
}

extern "C" int svi_sp_open(const unsigned char* handle64, void** peer_ptr) {
  using namespace svi;
  SVI_REQUIRE(handle64 && peer_ptr, "svi_sp_open: null pointer");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    set_last_error("svi_sp_open: cudaIpcOpenMemHandle failed: %s (peers must be NVLink/P2P reachable GPUs of one node)",
                   cudaGetErrorString(e));
    return SVI_ERR_DRIVER;
  }
  *peer_ptr = p;
  return SVI_OK;
}

extern "C" int svi_sp_close(void* peer_ptr) {
  using namespace svi;
  cudaError_t e = cudaIpcCloseMemHandle(peer_ptr);
  if (e != cudaSuccess) {
    set_last_error("svi_sp_close: %s", cudaGetErrorString(e));
    return SVI_ERR_DRIVER;
  }
  return SVI_OK;
}

extern "C" int svi_sp_push(const void* src, void* const* peer_dst, void* const* peer_flag, int32_t n_peers,
                           size_t bytes, const void* epoch_word, void* stream) {
  using namespace svi;
  SVI_REQUIRE(src && peer_dst && peer_flag && epoch_word && n_peers >= 0 && bytes > 0, "svi_sp_push: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int i = 0; i < n_peers; ++i) {
    SVI_REQUIRE(peer_dst[i] && peer_flag[i], "svi_sp_push: null peer pointer (peer %d)", i);
    cudaError_t e = cudaMemcpyAsync(peer_dst[i], src, bytes, cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) {
      set_last_error("svi_sp_push: peer copy %d failed: %s", i, cudaGetErrorString(e));
      return SVI_ERR_LAUNCH;
    }
    // stream order puts the flag after the copy engine has finished the rows
    e = cudaMemcpyAsync(peer_flag[i], epoch_word, 4, cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) {
      set_last_error("svi_sp_push: flag copy %d failed: %s", i, cudaGetErrorString(e));
      return SVI_ERR_LAUNCH;
    }
  }
  return SVI_OK;
}
