// Persistent warp-specialised bf16 GEMM for sm_90a:  out = epilogue(A[M,K] @ W[N,K]^T).
//
//   warpgroup 0     : TMA producer (one lane; 128B-swizzled 128x64 A and 256x64 W tiles into a 4-stage ring), 40 registers
//   warpgroups 1, 2 : consumers, rows [0, 64) and [64, 128) of the 128 x 256 tile: wgmma m64n256k16 with the fp32
//                     accumulator in registers, then the epilogue straight from those registers, 232 registers
//
// The producer runs ahead into the next tile while the consumers drain the previous one, so operand loads overlap the
// epilogue.  Tiles are visited in groups of GROUP_M row blocks so that the CTAs resident together share A and W tiles in L2.
// Replaces every F.linear of the reference's DiT (see include/svi_b200.h for the line map).
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/svi_b200.h"

namespace svi {
namespace gemm {

constexpr int BM = 128;
constexpr int BN = 256;
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int STAGES = 4;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int B_STAGE_BYTES = BN * BK * 2;  // 32 KB
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr int NUM_THREADS = 384;
constexpr int GROUP_M = 8;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 65536
static_assert(A_STAGE_BYTES % 1024 == 0 && STAGE_BYTES % 1024 == 0, "operand tiles must stay 1024-byte aligned");

struct Epi {
  void* out;
  long long ldo;
  int out_is_f32;
  int act;
  const float* bias;
  const float* gate;
  const float* residual;
  long long ldr;
  float* sumsq;
  int sumsq_groups;
  int sumsq_group_cols;
  int sumsq_parts;
  // LayerNorm folded into this GEMM (consumer side): A holds bf16(x * g) of the UN-normalised rows x; with the row statistics
  // (sum x, sum x^2) the epilogue reconstructs  LN(x)*g + t  times W^T  =  r_m (acc - mu_m u_n) + c_n,  u = W g, c = W t + b
  // (c arrives as `bias`)
  const float* ln_stats;   // [M, 2] or null
  const float* ln_u;       // [N]
  float ln_inv_d, ln_eps;
  // producer side: besides out, emit the NEXT GEMM's folded operand and row statistics from the final value v
  __nv_bfloat16* a_next;   // [M, ld_an] = bf16(v * g_next[n]) or null
  long long ld_an;
  const float* g_next;     // [N]
  float* row_stats;        // [M, 2] += (sum v, sum v^2) over this launch's columns (atomicAdd)
};

__device__ __forceinline__ void tile_coords(int tile, int num_m, int num_n, int& m_blk, int& n_blk) {
  const int per_group = GROUP_M * num_n;
  const int g = tile / per_group;
  const int first_m = g * GROUP_M;
  const int rows = min(GROUP_M, num_m - first_m);
  const int idx = tile - g * per_group;
  m_blk = first_m + idx % rows;
  n_blk = idx / rows;
}

// Activation with the switch outside the element loop (act is uniform over the launch).
__device__ __forceinline__ void apply_act2(float& a, float& b, int act) {
  if (act == SVI_ACT_GELU_TANH) {
    a = gelu_tanh(a); b = gelu_tanh(b);
  } else if (act == SVI_ACT_SILU) {
    a = silu(a); b = silu(b);
  } else if (act == SVI_ACT_GELU_ERF) {
    a = gelu_erf(a); b = gelu_erf(b);
  } else if (act == SVI_ACT_RELU) {
    a = fmaxf(a, 0.f); b = fmaxf(b, 0.f);
  }
}

// Sum over the four lanes that hold one accumulator row.
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// Row sums of squares per column group (the full-width q / k RMS norms, wan_video_dit.py:150-151).  sumsq_parts == 0:
// atomicAdd into [M, groups] (the order of the adds varies from run to run, and with it the last bit).  sumsq_parts == P > 0
// (P = group_cols / 128): every 128-column segment STORES its partial sum into [M, groups * P]; the consumers add a group's
// P partials in index order, so the result is bit-reproducible and the buffer needs no zeroing.
__device__ __forceinline__ void sumsq_flush(const Epi& ep, int row, bool ok, int lane, float ss, int key) {
  ss = quad_sum(ss);   // warp-uniform call: every lane takes part in the shuffles
  if (key < 0 || !ok || (lane & 3) != 0) return;
  if (ep.sumsq_parts) {
    const int segs = ep.sumsq_groups * ep.sumsq_parts;
    if (key < segs) ep.sumsq[(long long)row * segs + key] = ss;
  } else if (key < ep.sumsq_groups) {
    atomicAdd(&ep.sumsq[(long long)row * ep.sumsq_groups + key], ss);
  }
}

// Epilogue of one warp's 16 x 256 accumulator slice: rows row0 + g and row0 + g + 8, columns n_base + 8j + 2c (+1).
__device__ __forceinline__ void epilogue(const Epi& ep, float (&acc)[BN / 2], int M, int N, int row0, int n_base, int lane) {
  const int g = lane >> 2, c = lane & 3;
  const int rows[2] = {row0 + g, row0 + g + 8};
  const bool ok[2] = {rows[0] < M, rows[1] < M};
  float ln_r[2] = {1.f, 1.f}, ln_nmu[2] = {0.f, 0.f};
  if (ep.ln_stats) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!ok[h]) continue;
      const float2 st = __ldg(reinterpret_cast<const float2*>(ep.ln_stats) + rows[h]);
      const float mean = st.x * ep.ln_inv_d;
      ln_r[h] = rsqrtf(fmaxf(st.y * ep.ln_inv_d - mean * mean, 0.f) + ep.ln_eps);
      ln_nmu[h] = -mean;
    }
  }
  float ss[2] = {0.f, 0.f};
  int key = -1;
  float ps[2] = {0.f, 0.f}, pq[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n0 = n_base + 8 * j;
    if (n0 < N) {   // warp-uniform (N % 8 == 0)
      const int n = n0 + 2 * c;
      if (ep.sumsq) {
        const int k = ep.sumsq_parts ? (n0 >> 7) : n0 / ep.sumsq_group_cols;
        if (k != key) {
          sumsq_flush(ep, rows[0], ok[0], lane, ss[0], key);
          sumsq_flush(ep, rows[1], ok[1], lane, ss[1], key);
          ss[0] = ss[1] = 0.f;
          key = k;
        }
      }
      const float2 bv = ep.bias ? __ldg(reinterpret_cast<const float2*>(ep.bias + n)) : make_float2(0.f, 0.f);
      const float2 gv = ep.gate ? __ldg(reinterpret_cast<const float2*>(ep.gate + n)) : make_float2(1.f, 1.f);
      const float2 uv = ep.ln_stats ? __ldg(reinterpret_cast<const float2*>(ep.ln_u + n)) : make_float2(0.f, 0.f);
      const float2 gn = ep.a_next ? __ldg(reinterpret_cast<const float2*>(ep.g_next + n)) : make_float2(0.f, 0.f);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (ep.ln_stats) {
          v0 = ln_r[h] * fmaf(ln_nmu[h], uv.x, v0);
          v1 = ln_r[h] * fmaf(ln_nmu[h], uv.y, v1);
        }
        v0 += bv.x; v1 += bv.y;
        if (ep.act != SVI_ACT_NONE) apply_act2(v0, v1, ep.act);
        ss[h] += v0 * v0 + v1 * v1;
        v0 *= gv.x; v1 *= gv.y;
        if (ok[h]) {
          if (ep.residual) {
            const float2 r = *reinterpret_cast<const float2*>(ep.residual + (long long)rows[h] * ep.ldr + n);
            v0 += r.x; v1 += r.y;
          }
          if (ep.a_next) {
            ps[h] += v0 + v1;
            pq[h] = fmaf(v1, v1, fmaf(v0, v0, pq[h]));
            *reinterpret_cast<uint32_t*>(ep.a_next + (long long)rows[h] * ep.ld_an + n) = pack_bf16x2(v0 * gn.x, v1 * gn.y);
          }
          if (ep.out_is_f32) {
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(ep.out) + (long long)rows[h] * ep.ldo + n) = make_float2(v0, v1);
          } else {
            *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(ep.out) + (long long)rows[h] * ep.ldo + n) =
                pack_bf16x2(v0, v1);
          }
        }
      }
    }
  }
  if (ep.sumsq) {
    sumsq_flush(ep, rows[0], ok[0], lane, ss[0], key);
    sumsq_flush(ep, rows[1], ok[1], lane, ss[1], key);
  }
  if (ep.a_next) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float a = quad_sum(ps[h]), b = quad_sum(pq[h]);
      if (ok[h] && c == 0) {
        atomicAdd(&ep.row_stats[2LL * rows[h]], a);
        atomicAdd(&ep.row_stats[2LL * rows[h] + 1], b);
      }
    }
  }
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, int M, int N, int K,
                 const __grid_constant__ Epi ep) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bars = sbase + STAGES * STAGE_BYTES;
  auto full_bar = [&](int s) { return bars + 8u * s; };
  auto empty_bar = [&](int s) { return bars + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int num_m = (M + BM - 1) / BM;
  const int num_n = (N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_k = (K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init_a(full_bar(i), 1);
      mbar_init_a(empty_bar(i), 8);   // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------- TMA producer -------------------------------
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        tile_coords(tile, num_m, num_n, m_blk, n_blk);
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait_a(empty_bar(stage), phase ^ 1);
          mbar_expect_tx_a(full_bar(stage), STAGE_BYTES);
          const uint32_t sa = sbase + stage * STAGE_BYTES;
          tma_load_2d_a(sa, &tmap_a, full_bar(stage), kb * BK, m_blk * BM);
          tma_load_2d_a(sa + A_STAGE_BYTES, &tmap_b, full_bar(stage), kb * BK, n_blk * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------- consumers ----------------------------------
    setmaxnreg_inc<CONSUMER_REGS>();
    const int cw = wg - 1;   // rows [64 cw, 64 cw + 64) of the tile
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int m_blk, n_blk;
      tile_coords(tile, num_m, num_n, m_blk, n_blk);
      int prev = -1;
      for (int kb = 0; kb < num_k; ++kb) {
        mbar_wait_a(full_bar(stage), phase);
        const uint32_t sa = sbase + stage * STAGE_BYTES;
        const uint64_t da = wgmma_desc(sa + cw * 64 * 128, 16, 1024);
        const uint64_t db = wgmma_desc(sa + A_STAGE_BYTES, 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)   // +32 B per K-step = +2 in the 16-byte address field
          Wgmma<BN>::ss(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();   // the previous stage's MMAs have retired: its slot goes back to the producer
        if (prev >= 0 && lane == 0) mbar_arrive_a(empty_bar(prev));
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (lane == 0) mbar_arrive_a(empty_bar(prev));
      epilogue(ep, acc, M, N, m_blk * BM + cw * 64 + (warp & 3) * 16, n_blk * BN, lane);
    }
  }
}

}  // namespace gemm
}  // namespace svi

extern "C" int svi_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, int32_t M,
                             int32_t N, int32_t K, const svi_gemm_epilogue* e, void* stream) {
  using namespace svi;
  using namespace svi::gemm;
  SVI_REQUIRE(A && W && e && e->out, "svi_gemm_bf16: null pointer");
  SVI_REQUIRE(M > 0 && N > 0 && K > 0, "svi_gemm_bf16: M,N,K must be positive (got %d,%d,%d)", M, N, K);
  SVI_REQUIRE(K % 8 == 0 && N % 8 == 0, "svi_gemm_bf16: K and N must be multiples of 8 (K=%d N=%d)", K, N);
  SVI_REQUIRE(lda % 8 == 0 && ldw % 8 == 0 && lda >= K && ldw >= K,
              "svi_gemm_bf16: lda/ldw must be multiples of 8 and >= K");
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
              "svi_gemm_bf16: A and W must be 16-byte aligned");
  SVI_REQUIRE(e->ldo >= N && e->ldo % (e->out_is_f32 ? 4 : 8) == 0 &&
                  (reinterpret_cast<uintptr_t>(e->out) & 15) == 0,
              "svi_gemm_bf16: out must be 16-byte aligned with ldo >= N and 16-byte row pitch");
  SVI_REQUIRE(e->act >= 0 && e->act <= 4, "svi_gemm_bf16: unknown activation %d", e->act);
  if (e->residual)
    SVI_REQUIRE(e->ldr >= N && e->ldr % 4 == 0 && (reinterpret_cast<uintptr_t>(e->residual) & 15) == 0,
                "svi_gemm_bf16: residual must be 16-byte aligned with ldr >= N, ldr %% 4 == 0");
  if (e->bias) SVI_REQUIRE((reinterpret_cast<uintptr_t>(e->bias) & 15) == 0, "svi_gemm_bf16: bias alignment");
  if (e->gate) SVI_REQUIRE((reinterpret_cast<uintptr_t>(e->gate) & 15) == 0, "svi_gemm_bf16: gate alignment");
  if (e->sumsq)
    SVI_REQUIRE(e->sumsq_groups > 0 && e->sumsq_group_cols > 0 && e->sumsq_group_cols % 32 == 0,
                "svi_gemm_bf16: sumsq_group_cols must be a positive multiple of 32");
  if (e->sumsq && e->sumsq_parts)
    SVI_REQUIRE(e->sumsq_group_cols % 128 == 0 && e->sumsq_parts == e->sumsq_group_cols / 128,
                "svi_gemm_bf16: sumsq_parts must be 0 (atomic accumulation) or sumsq_group_cols / 128 with sumsq_group_cols %% 128 == 0");
  if (e->ln_stats)
    SVI_REQUIRE(e->ln_u && e->ln_dim > 0 && (reinterpret_cast<uintptr_t>(e->ln_stats) & 7) == 0 &&
                    (reinterpret_cast<uintptr_t>(e->ln_u) & 7) == 0,
                "svi_gemm_bf16: ln fold needs ln_u (8-byte aligned), ln_dim > 0 and 8-byte aligned ln_stats");
  if (e->a_next)
    SVI_REQUIRE(e->g_next && e->row_stats && e->ld_an >= N && e->ld_an % 8 == 0 &&
                    (reinterpret_cast<uintptr_t>(e->a_next) & 15) == 0 && (reinterpret_cast<uintptr_t>(e->g_next) & 7) == 0,
                "svi_gemm_bf16: a_next needs g_next, row_stats, ld_an >= N (multiple of 8) and 16-byte alignment");

  CUtensorMap ta, tb;
  int rc = make_tmap_2d(&ta, A, 2, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, BK, BM);
  if (rc) return rc;
  rc = make_tmap_2d(&tb, W, 2, (uint64_t)K, (uint64_t)N, (uint64_t)ldw * 2, BK, BN);
  if (rc) return rc;

  Epi ep;
  ep.out = e->out; ep.ldo = e->ldo; ep.out_is_f32 = e->out_is_f32; ep.act = e->act;
  ep.bias = e->bias; ep.gate = e->gate; ep.residual = e->residual; ep.ldr = e->ldr;
  ep.sumsq = e->sumsq; ep.sumsq_groups = e->sumsq_groups; ep.sumsq_group_cols = e->sumsq_group_cols; ep.sumsq_parts = e->sumsq_parts;
  ep.ln_stats = e->ln_stats; ep.ln_u = e->ln_u; ep.ln_inv_d = e->ln_dim > 0 ? 1.0f / (float)e->ln_dim : 0.f; ep.ln_eps = e->ln_eps;
  ep.a_next = reinterpret_cast<__nv_bfloat16*>(e->a_next); ep.ld_an = e->ld_an; ep.g_next = e->g_next; ep.row_stats = e->row_stats;

  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t ce = cudaFuncSetAttribute(gemm_bf16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (ce != cudaSuccess) {
      set_last_error("svi_gemm_bf16: cudaFuncSetAttribute failed: %s", cudaGetErrorString(ce));
      return SVI_ERR_LAUNCH;
    }
    attr_set = true;
  }
  const int num_tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
  const int sms = sm_count();
  if (sms <= 0) return SVI_ERR_DRIVER;
  const int grid = num_tiles < sms ? num_tiles : sms;
  gemm_bf16_kernel<<<grid, NUM_THREADS, SMEM_BYTES, static_cast<cudaStream_t>(stream)>>>(ta, tb, M, N, K, ep);
  SVI_CUDA_LAUNCH_CHECK("svi_gemm_bf16");
  return SVI_OK;
}
