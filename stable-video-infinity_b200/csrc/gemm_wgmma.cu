// Persistent warp-specialised bf16 GEMM for sm_90a:  out = epilogue(A[M,K] @ W[N,K]^T).
//
//   warpgroup 0     : TMA producer (one lane; 128B-swizzled 128x64 A and 256x64 W tiles into a 4-stage ring), 40 registers
//   warpgroups 1, 2 : consumers sharing each 128 x 256 tile: warpgroup w takes rows [64 w, 64 w + 64) as one m64n256k16
//                     per k16 step, fp32 accumulators in registers (128 per thread), then runs the epilogue straight from
//                     those registers in two 128-column passes, 232 registers
//
// The wide tile is for the operand feed: per k16 step each warpgroup reads the 256-row W slice from shared memory once for
// 64 x 256 outputs, and a tile moves 48 KB of operands from L2 per 4.2 MFLOP.  Its epilogue does not overlap MMAs of the
// same CTA; the producer keeps filling the ring with the next tile's k-blocks meanwhile.
//
// e4m3 weights (svi_gemm_epilogue.w_e4m3 = 1; the reference's weight-only FP8 mode): the producer lane TMA-loads the
// 256 x 64 e4m3 W tile (16 KB, unswizzled) into a staging ring instead, and warps 1-3 of warpgroup 0 (idle in the bf16
// instantiation) convert it, exactly, into the bf16 W tile in the same 128B-swizzled layout the bf16 TMA load produces.
// The consumers, their wgmma descriptors and the epilogue are the same code, so the result is bit-identical to the bf16
// GEMM on bf16(W).  Shared memory: 4 bf16 stages (192 KB) + 2 staging stages (32 KB), against 4 x 48 KB for bf16.
//
// The producer runs ahead across tiles, so operand loads overlap the epilogues.  Tiles are visited in groups of GROUP_M
// row blocks so that the CTAs resident together share A and W tiles in L2.
// Replaces every F.linear of the reference's DiT (see include/svi_b200.h for the line map).
//
// LoRA segment (kLoRA, svi_gemm_lora_bf16 in include/svi_b200_lora.h): out = epilogue(A W^T + U_g(n) B^T).  After a tile's
// num_k k-blocks the producer loads R / 64 more into the same ring, from U [M, groups R] (column g R + 64 kb, g = the
// tile's column group) and B [N, R]; the consumers run them into the same accumulators, so every epilogue stage sees the
// LoRA term.  Those tiles are bf16 in both weight formats: with e4m3 W the producer TMA-loads the B tile straight into the
// swizzled W half and makes the converter warps' arrivals on the stage's full barrier itself; the converters step over it.
// Column groups of an odd multiple of 128 would straddle a 256-column tile; svi_gemm_lora_bf16 launches those one group
// at a time.
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/svi_b200.h"
#include "../../include/svi_b200_lora.h"

namespace svi {
namespace gemm {

constexpr int BM = 128;
constexpr int BN = 256;
constexpr int EPI_N = 128;  // columns per epilogue pass (one 128-column half of a warp's accumulators)
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int B_STAGE_BYTES = BN * BK * 2;  // 32 KB
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr int W8_STAGE_BYTES = BN * BK;     // 16 KB of e4m3 W
constexpr int NUM_THREADS = 384;
constexpr int NUM_CONVERTERS = 96;          // warps 1-3 of warpgroup 0 (e4m3 instantiation)
constexpr int GROUP_M = 8;                  // 16 measured no faster on 256-column tiles (DESIGN.md §4)
constexpr int RES_J = 4;                    // 8-column blocks whose residual, bias and gate loads go out together
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 65536
static_assert(A_STAGE_BYTES % 1024 == 0 && STAGE_BYTES % 1024 == 0, "operand tiles must stay 1024-byte aligned");
static_assert((EPI_N / 8) % RES_J == 0 && BN % EPI_N == 0, "residual batches must tile the warp's columns");

// Ring depths per weight format: bf16 stages (A + bf16 W) and e4m3 staging stages.
template <bool kE4M3> struct Rings;
// 4 bf16 stages: 3 measured slower on ffn.0 / ffn.2 (DESIGN.md §4)
template <> struct Rings<false> { static constexpr int STAGES = 4, W8_STAGES = 0; };
template <> struct Rings<true> { static constexpr int STAGES = 4, W8_STAGES = 2; };
template <bool kE4M3>
constexpr int smem_bytes() {
  return Rings<kE4M3>::STAGES * STAGE_BYTES + Rings<kE4M3>::W8_STAGES * W8_STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
}
static_assert(smem_bytes<true>() <= 227 * 1024 && smem_bytes<false>() <= 227 * 1024, "shared memory over the sm_90 limit");

// Four e4m3 codes (byte i = element i) -> bf16 elements 0,1 (.x) and 2,3 (.y), exactly.  Each code's sign goes to bit 15
// and its 7 exponent|mantissa bits to bits 4..10 of a bf16, which reads as the e4m3 value times 2^-120 (the 4-bit
// exponent field lands in the low bits of bf16's 8-bit one; code exponent 0 lands on bf16 subnormals, which is the e4m3
// subnormal scale); one bf16x2 multiply by 2^120 is exact and restores the value, +-0 included.  The NaN codes 0x7F / 0xFF
// (which would read as +-480) get their exponent and top mantissa bits set instead.
__device__ __forceinline__ uint2 e4m3x4_to_bf16x4(uint32_t w) {
  const uint32_t q = __byte_perm(w, 0, 0x3120);              // bytes [b0, b2, b1, b3]
  const uint32_t q0 = q << 8;                                // halves hold b0 | b1 in their high bytes
  uint32_t lo = (q0 & 0x80008000u) | ((q0 & 0x7F007F00u) >> 4);
  uint32_t hi = (q & 0x80008000u) | ((q & 0x7F007F00u) >> 4); // b2 | b3
  asm("mul.rn.bf16x2 %0, %0, %1;" : "+r"(lo) : "r"(0x7B807B80u));   // 2^120 in both halves
  asm("mul.rn.bf16x2 %0, %0, %1;" : "+r"(hi) : "r"(0x7B807B80u));
  const uint32_t nan = ((w & 0x7F7F7F7Fu) + 0x01010101u) & 0x80808080u;   // bit 7 of every byte whose code is +-NaN
  if (nan) {
    lo |= ((nan & 0x80u) ? 0x7FC0u : 0u) | ((nan & 0x8000u) ? 0x7FC00000u : 0u);
    hi |= ((nan & 0x800000u) ? 0x7FC0u : 0u) | ((nan & 0x80000000u) ? 0x7FC00000u : 0u);
  }
  return make_uint2(lo, hi);
}

// One 256 x 64 e4m3 staging tile (row-major, 64 B per row) -> the bf16 W tile as the 128B-swizzled TMA load lays it out:
// row r at byte 128 r, its 16-byte chunk j at chunk position j ^ (r & 7).  Thread t takes 16-byte source chunks t, t + 96, ...
// (row i / 4, bf16 chunks 2 (i % 4) and 2 (i % 4) + 1); a quarter-warp's stores hit eight distinct bank groups.
__device__ __forceinline__ void convert_w_tile(uint32_t src, uint32_t dst, int t) {
#pragma unroll 2
  for (int i = t; i < W8_STAGE_BYTES / 16; i += NUM_CONVERTERS) {
    uint32_t w0, w1, w2, w3;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(w0), "=r"(w1), "=r"(w2), "=r"(w3) : "r"(src + 16u * i));
    const uint2 e0 = e4m3x4_to_bf16x4(w0), e1 = e4m3x4_to_bf16x4(w1), e2 = e4m3x4_to_bf16x4(w2), e3 = e4m3x4_to_bf16x4(w3);
    const int r = i >> 2, j = 2 * (i & 3);
    const uint32_t row = dst + 128u * r;
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(row + 16u * (j ^ (r & 7))), "r"(e0.x), "r"(e0.y), "r"(e1.x),
                 "r"(e1.y) : "memory");
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(row + 16u * ((j + 1) ^ (r & 7))), "r"(e2.x), "r"(e2.y),
                 "r"(e3.x), "r"(e3.y) : "memory");
  }
}

struct Epi {
  void* out;
  long long ldo;
  const float* bias;
  const float* gate;
  const float* residual;
  long long ldr;
  float* sumsq;
  int sumsq_groups;
  int sumsq_group_cols;
  int sumsq_parts;
  int sumsq_col0;          // the column that this launch's column 0 is in the row sums' column grouping
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

// The LoRA segment of a launch: empty in the plain instantiations, whose parameter list and code stay as they were.
template <bool kLoRA> struct LoRAArgs {};
template <> struct LoRAArgs<true> {
  CUtensorMap u;    // U [M, groups R] bf16, 64 x 128 boxes (BM rows), 128B swizzle
  CUtensorMap b;    // B [N, R] bf16, 64 x 256 boxes (BN rows), 128B swizzle
  int kb;           // R / BK
  int group_cols;   // 0: one group; else a multiple of BN (svi_gemm_lora_bf16 launches narrower groups one by one)
};

__device__ __forceinline__ void mbar_arrive_cnt_a(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}

__device__ __forceinline__ void tile_coords(int tile, int num_m, int num_n, int& m_blk, int& n_blk) {
  const int per_group = GROUP_M * num_n;
  const int g = tile / per_group;
  const int first_m = g * GROUP_M;
  const int rows = min(GROUP_M, num_m - first_m);
  const int idx = tile - g * per_group;
  m_blk = first_m + idx % rows;
  n_blk = idx / rows;
}

// The activation, the output type and the LayerNorm fold are template parameters of the kernel: the epilogue is unrolled
// over all 64 accumulator pairs of a warp's slice, so runtime switches put the code of every variant into that unrolled
// body.  One kernel held about 17 000 SASS instructions that way, and at K = 1536 the bare GEMM ran at 190 TFLOP/s against
// 490 with one kernel per variant (H100 80GB HBM3, 700 W, tools/gemm_bench.py).
template <int kAct>
__device__ __forceinline__ void apply_act2(float& a, float& b) {
  if constexpr (kAct == SVI_ACT_GELU_TANH) {
    a = gelu_tanh(a); b = gelu_tanh(b);
  } else if constexpr (kAct == SVI_ACT_SILU) {
    a = silu(a); b = silu(b);
  } else if constexpr (kAct == SVI_ACT_GELU_ERF) {
    a = gelu_erf(a); b = gelu_erf(b);
  } else if constexpr (kAct == SVI_ACT_RELU) {
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

// Epilogue of one warp's 16 x 128 accumulator slice: rows row0 + g and row0 + g + 8, columns n_base + 8j + 2c (+1).
// The residual may be `out` itself (each element is read and then written by the same lane only), so the compiler may not
// move a load above an earlier store: the residual, bias and gate loads of RES_J column blocks are issued together, ahead
// of their stores, which makes one memory round trip per batch instead of one per column block.
template <int kAct, bool kF32, bool kFold>
__device__ __forceinline__ void epilogue(const Epi& ep, float (&acc)[EPI_N / 2], int M, int N, int row0, int n_base, int lane) {
  const int g = lane >> 2, c = lane & 3;
  const int rows[2] = {row0 + g, row0 + g + 8};
  const bool ok[2] = {rows[0] < M, rows[1] < M};
  float ln_r[2] = {1.f, 1.f}, ln_nmu[2] = {0.f, 0.f};
  if (kFold && ep.ln_stats) {
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
  float2 res[RES_J][2], bvs[RES_J], gvs[RES_J];
  // this lane's first column in each of its two rows: column block j is then a constant offset of 8 j elements
  const long long col0 = (long long)n_base + 2 * c;
  const float* res_row[2];
  void* out_row[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    res_row[h] = ep.residual ? ep.residual + rows[h] * ep.ldr + col0 : nullptr;
    out_row[h] = kF32 ? (void*)(reinterpret_cast<float*>(ep.out) + rows[h] * ep.ldo + col0)
                      : (void*)(reinterpret_cast<__nv_bfloat16*>(ep.out) + rows[h] * ep.ldo + col0);
  }
#pragma unroll
  for (int j = 0; j < EPI_N / 8; ++j) {
    if (j % RES_J == 0) {
#pragma unroll
      for (int i = 0; i < RES_J; ++i) {
        const int nb = n_base + 8 * (j + i);
        const bool in = nb < N;
        bvs[i] = ep.bias && in ? __ldg(reinterpret_cast<const float2*>(ep.bias + nb + 2 * c)) : make_float2(0.f, 0.f);
        gvs[i] = ep.gate && in ? __ldg(reinterpret_cast<const float2*>(ep.gate + nb + 2 * c)) : make_float2(1.f, 1.f);
        if (ep.residual) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
            res[i][h] = ok[h] && in ? *reinterpret_cast<const float2*>(res_row[h] + 8 * (j + i)) : make_float2(0.f, 0.f);
        }
      }
    }
    const int n0 = n_base + 8 * j;
    if (n0 < N) {   // warp-uniform (N % 8 == 0)
      const int n = n0 + 2 * c;
      if (ep.sumsq && j % 4 == 0) {   // a group starts only on a 32-column boundary (sumsq_group_cols % 32 == 0)
        const int k = ep.sumsq_parts ? ((n0 + ep.sumsq_col0) >> 7) : (n0 + ep.sumsq_col0) / ep.sumsq_group_cols;
        if (k != key) {
          sumsq_flush(ep, rows[0], ok[0], lane, ss[0], key);
          sumsq_flush(ep, rows[1], ok[1], lane, ss[1], key);
          ss[0] = ss[1] = 0.f;
          key = k;
        }
      }
      const float2 bv = bvs[j % RES_J], gv = gvs[j % RES_J];
      const float2 uv = kFold && ep.ln_stats ? __ldg(reinterpret_cast<const float2*>(ep.ln_u + n)) : make_float2(0.f, 0.f);
      const float2 gn = kFold && ep.a_next ? __ldg(reinterpret_cast<const float2*>(ep.g_next + n)) : make_float2(0.f, 0.f);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (kFold && ep.ln_stats) {
          v0 = ln_r[h] * fmaf(ln_nmu[h], uv.x, v0);
          v1 = ln_r[h] * fmaf(ln_nmu[h], uv.y, v1);
        }
        v0 += bv.x; v1 += bv.y;
        apply_act2<kAct>(v0, v1);
        ss[h] += fmaf(v0, v0, v1 * v1);   // contraction spelled out: identical in both weight-format instantiations
        v0 *= gv.x; v1 *= gv.y;
        if (ok[h]) {
          if (ep.residual) {
            v0 += res[j % RES_J][h].x; v1 += res[j % RES_J][h].y;
          }
          if (kFold && ep.a_next) {
            ps[h] += v0 + v1;
            pq[h] = fmaf(v1, v1, fmaf(v0, v0, pq[h]));
            *reinterpret_cast<uint32_t*>(ep.a_next + (long long)rows[h] * ep.ld_an + n) = pack_bf16x2(v0 * gn.x, v1 * gn.y);
          }
          if constexpr (kF32) {
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(out_row[h]) + 8 * j) = make_float2(v0, v1);
          } else {
            *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(out_row[h]) + 8 * j) = pack_bf16x2(v0, v1);
          }
        }
      }
    }
  }
  if (ep.sumsq) {
    sumsq_flush(ep, rows[0], ok[0], lane, ss[0], key);
    sumsq_flush(ep, rows[1], ok[1], lane, ss[1], key);
  }
  if (kFold && ep.a_next) {
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

template <bool kE4M3, int kAct, bool kF32, bool kFold, bool kLoRA>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, int M, int N, int K,
                 const __grid_constant__ Epi ep, const __grid_constant__ LoRAArgs<kLoRA> lora) {
  constexpr int STAGES = Rings<kE4M3>::STAGES, W8_STAGES = Rings<kE4M3>::W8_STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t s8base = sbase + STAGES * STAGE_BYTES;          // e4m3 staging ring (e4m3 instantiation)
  const uint32_t bars = s8base + W8_STAGES * W8_STAGE_BYTES;
  auto full_bar = [&](int s) { return bars + 8u * s; };
  auto empty_bar = [&](int s) { return bars + 8u * (STAGES + s); };
  auto full8_bar = [&](int s) { return bars + 8u * (2 * STAGES + s); };               // staging tile landed
  auto empty8_bar = [&](int s) { return bars + 8u * (2 * STAGES + W8_STAGES + s); };  // staging tile converted

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int num_m = (M + BM - 1) / BM;
  const int num_n = (N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_k = (K + BK - 1) / BK;
  int num_kt = num_k;   // k-blocks per tile, LoRA segment included
  if constexpr (kLoRA) num_kt += lora.kb;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init_a(full_bar(i), kE4M3 ? 1 + NUM_CONVERTERS / 32 : 1);   // e4m3: + one arrive per converter warp
      mbar_init_a(empty_bar(i), 8);   // one arrive per consumer warp
    }
    for (int i = 0; i < W8_STAGES; ++i) {
      mbar_init_a(full8_bar(i), 1);
      mbar_init_a(empty8_bar(i), NUM_CONVERTERS / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------- TMA producer -------------------------------
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      int stage = 0, stage8 = 0;
      uint32_t phase = 0, phase8 = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        tile_coords(tile, num_m, num_n, m_blk, n_blk);
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait_a(empty_bar(stage), phase ^ 1);
          const uint32_t sa = sbase + stage * STAGE_BYTES;
          if constexpr (kE4M3) {
            mbar_expect_tx_a(full_bar(stage), A_STAGE_BYTES);
            tma_load_2d_a(sa, &tmap_a, full_bar(stage), kb * BK, m_blk * BM);
            mbar_wait_a(empty8_bar(stage8), phase8 ^ 1);
            mbar_expect_tx_a(full8_bar(stage8), W8_STAGE_BYTES);
            tma_load_2d_a(s8base + stage8 * W8_STAGE_BYTES, &tmap_b, full8_bar(stage8), kb * BK, n_blk * BN);
            if (++stage8 == W8_STAGES) { stage8 = 0; phase8 ^= 1; }
          } else {
            mbar_expect_tx_a(full_bar(stage), STAGE_BYTES);
            tma_load_2d_a(sa, &tmap_a, full_bar(stage), kb * BK, m_blk * BM);
            tma_load_2d_a(sa + A_STAGE_BYTES, &tmap_b, full_bar(stage), kb * BK, n_blk * BN);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        if constexpr (kLoRA) {
          const int g = lora.group_cols ? n_blk * BN / lora.group_cols : 0;   // a tile never straddles two groups
          for (int kb = 0; kb < lora.kb; ++kb) {
            mbar_wait_a(empty_bar(stage), phase ^ 1);
            const uint32_t sa = sbase + stage * STAGE_BYTES;
            // e4m3: no converter touches this stage, so the producer makes their arrivals (before its own, which comes
            // with the expected bytes: the phase cannot complete before both tiles land)
            if constexpr (kE4M3) mbar_arrive_cnt_a(full_bar(stage), NUM_CONVERTERS / 32);
            mbar_expect_tx_a(full_bar(stage), STAGE_BYTES);
            tma_load_2d_a(sa, &lora.u, full_bar(stage), (g * lora.kb + kb) * BK, m_blk * BM);
            tma_load_2d_a(sa + A_STAGE_BYTES, &lora.b, full_bar(stage), kb * BK, n_blk * BN);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    } else if (kE4M3 && warp >= 1) {
      // ------------------------------- e4m3 -> bf16 W converters -------------------------------
      // The staging tile of k-block i lands after the producer saw bf16 stage (i mod STAGES) freed by the consumers, so its
      // W half may be written once full8 completes.  The writes are generic-proxy stores that wgmma (async proxy) reads:
      // every writer fences before its warp's arrive on the stage's full barrier.
      const int t = threadIdx.x - 32;
      int stage = 0, stage8 = 0;
      uint32_t phase8 = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait_a(full8_bar(stage8), phase8);
          convert_w_tile(s8base + stage8 * W8_STAGE_BYTES, sbase + stage * STAGE_BYTES + A_STAGE_BYTES, t);
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
          if (lane == 0) {
            mbar_arrive_a(empty8_bar(stage8));
            mbar_arrive_a(full_bar(stage));
          }
          if (++stage8 == W8_STAGES) { stage8 = 0; phase8 ^= 1; }
          if (++stage == STAGES) stage = 0;
        }
        if constexpr (kLoRA) stage = (stage + lora.kb) % STAGES;   // the LoRA k-blocks arrive in bf16
      }
    }
  } else {
    // ------------------------------- consumers ----------------------------------
    setmaxnreg_inc<CONSUMER_REGS>();
    // Both warpgroups share every tile: warpgroup cw takes rows [64 cw, 64 cw + 64) as one m64n256k16 per k16 step.
    const int cw = wg - 1;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int m_blk, n_blk;
      tile_coords(tile, num_m, num_n, m_blk, n_blk);
      int prev = -1;
      for (int kb = 0; kb < num_kt; ++kb) {
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
      const int row0 = m_blk * BM + cw * 64 + (warp & 3) * 16;
#pragma unroll
      for (int h = 0; h < BN / EPI_N; ++h)
        epilogue<kAct, kF32, kFold>(ep, *reinterpret_cast<float(*)[EPI_N / 2]>(acc + h * EPI_N / 2), M, N, row0,
                                    n_blk * BN + h * EPI_N, lane);
    }
  }
}

// Sets the dynamic shared-memory size of one instantiation once per process, then launches it.
template <bool kE4M3, int kAct, bool kF32, bool kFold, bool kLoRA>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, int M, int N, int K, const Epi& ep, const LoRAArgs<kLoRA>& lora,
           cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t ce = cudaFuncSetAttribute(gemm_bf16_kernel<kE4M3, kAct, kF32, kFold, kLoRA>,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<kE4M3>());
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
  gemm_bf16_kernel<kE4M3, kAct, kF32, kFold, kLoRA><<<grid, NUM_THREADS, smem_bytes<kE4M3>(), stream>>>(ta, tb, M, N, K, ep, lora);
  SVI_CUDA_LAUNCH_CHECK("svi_gemm_bf16");
  return SVI_OK;
}

// The LoRA instantiations cover what the DiT blocks use: no activation or GELU-tanh (ffn.0), no LayerNorm fold.
template <bool kE4M3, bool kF32, bool kFold, bool kLoRA>
int launch_act(const CUtensorMap& ta, const CUtensorMap& tb, int M, int N, int K, int act, const Epi& ep,
               const LoRAArgs<kLoRA>& lora, cudaStream_t stream) {
  if constexpr (kLoRA) {
    return act == SVI_ACT_GELU_TANH ? launch<kE4M3, SVI_ACT_GELU_TANH, kF32, kFold>(ta, tb, M, N, K, ep, lora, stream)
                                    : launch<kE4M3, SVI_ACT_NONE, kF32, kFold>(ta, tb, M, N, K, ep, lora, stream);
  } else {
    switch (act) {
      case SVI_ACT_GELU_TANH: return launch<kE4M3, SVI_ACT_GELU_TANH, kF32, kFold>(ta, tb, M, N, K, ep, lora, stream);
      case SVI_ACT_SILU: return launch<kE4M3, SVI_ACT_SILU, kF32, kFold>(ta, tb, M, N, K, ep, lora, stream);
      case SVI_ACT_GELU_ERF: return launch<kE4M3, SVI_ACT_GELU_ERF, kF32, kFold>(ta, tb, M, N, K, ep, lora, stream);
      case SVI_ACT_RELU: return launch<kE4M3, SVI_ACT_RELU, kF32, kFold>(ta, tb, M, N, K, ep, lora, stream);
      default: return launch<kE4M3, SVI_ACT_NONE, kF32, kFold>(ta, tb, M, N, K, ep, lora, stream);   // act was checked to be in [0, 4]
    }
  }
}

// One kernel per (weight format, activation, output type, LayerNorm fold on / off, LoRA segment on / off).
template <bool kE4M3, bool kLoRA>
int launch_kind(const CUtensorMap& ta, const CUtensorMap& tb, int M, int N, int K, int act, bool f32, bool fold, const Epi& ep,
                const LoRAArgs<kLoRA>& lora, cudaStream_t stream) {
  if constexpr (kLoRA) {   // the fold was rejected
    return f32 ? launch_act<kE4M3, true, false>(ta, tb, M, N, K, act, ep, lora, stream)
               : launch_act<kE4M3, false, false>(ta, tb, M, N, K, act, ep, lora, stream);
  } else {
    if (f32)
      return fold ? launch_act<kE4M3, true, true>(ta, tb, M, N, K, act, ep, lora, stream)
                  : launch_act<kE4M3, true, false>(ta, tb, M, N, K, act, ep, lora, stream);
    return fold ? launch_act<kE4M3, false, true>(ta, tb, M, N, K, act, ep, lora, stream)
                : launch_act<kE4M3, false, false>(ta, tb, M, N, K, act, ep, lora, stream);
  }
}

int make_w_tmap(CUtensorMap* tb, const void* W, int64_t ldw, int N, int K, bool e4m3) {
  if (e4m3)   // the converters swizzle; the staging tile is plain 64-byte rows
    return make_tmap_2d(tb, W, 1, (uint64_t)K, (uint64_t)N, (uint64_t)ldw, BK, BN, /*swizzle_128b=*/false);
  return make_tmap_2d(tb, W, 2, (uint64_t)K, (uint64_t)N, (uint64_t)ldw * 2, BK, BN);
}

// The arguments of one GEMM as both entry points take them: checked, then turned into the operand tensor maps and the
// kernel's epilogue block.  `fn` names the entry point in the messages.
int prepare(const char* fn, const void* A, int64_t lda, const void* W, int64_t ldw, int32_t M, int32_t N, int32_t K,
            const svi_gemm_epilogue* e, CUtensorMap* ta, CUtensorMap* tb, Epi* ep) {
  SVI_REQUIRE(A && W && e && e->out, "%s: null pointer", fn);
  SVI_REQUIRE(M > 0 && N > 0 && K > 0, "%s: M,N,K must be positive (got %d,%d,%d)", fn, M, N, K);
  SVI_REQUIRE(K % 8 == 0 && N % 8 == 0, "%s: K and N must be multiples of 8 (K=%d N=%d)", fn, K, N);
  SVI_REQUIRE(lda % 8 == 0 && ldw % 8 == 0 && lda >= K && ldw >= K, "%s: lda/ldw must be multiples of 8 and >= K", fn);
  SVI_REQUIRE(e->w_e4m3 == 0 || e->w_e4m3 == 1, "%s: w_e4m3 must be 0 (bf16 W) or 1 (e4m3 W), got %d", fn, e->w_e4m3);
  if (e->w_e4m3)
    SVI_REQUIRE(K % 16 == 0 && ldw % 16 == 0,
                "%s: e4m3 W needs K and ldw to be multiples of 16 (16-byte row pitch; K=%d ldw=%lld)", fn, K, (long long)ldw);
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
              "%s: A and W must be 16-byte aligned", fn);
  SVI_REQUIRE(e->ldo >= N && e->ldo % (e->out_is_f32 ? 4 : 8) == 0 &&
                  (reinterpret_cast<uintptr_t>(e->out) & 15) == 0,
              "%s: out must be 16-byte aligned with ldo >= N and 16-byte row pitch", fn);
  SVI_REQUIRE(e->act >= 0 && e->act <= 4, "%s: unknown activation %d", fn, e->act);
  if (e->residual)
    SVI_REQUIRE(e->ldr >= N && e->ldr % 4 == 0 && (reinterpret_cast<uintptr_t>(e->residual) & 15) == 0,
                "%s: residual must be 16-byte aligned with ldr >= N, ldr %% 4 == 0", fn);
  if (e->bias) SVI_REQUIRE((reinterpret_cast<uintptr_t>(e->bias) & 15) == 0, "%s: bias alignment", fn);
  if (e->gate) SVI_REQUIRE((reinterpret_cast<uintptr_t>(e->gate) & 15) == 0, "%s: gate alignment", fn);
  if (e->sumsq)
    SVI_REQUIRE(e->sumsq_groups > 0 && e->sumsq_group_cols > 0 && e->sumsq_group_cols % 32 == 0,
                "%s: sumsq_group_cols must be a positive multiple of 32", fn);
  if (e->sumsq && e->sumsq_parts)
    SVI_REQUIRE(e->sumsq_group_cols % 128 == 0 && e->sumsq_parts == e->sumsq_group_cols / 128,
                "%s: sumsq_parts must be 0 (atomic accumulation) or sumsq_group_cols / 128 with sumsq_group_cols %% 128 == 0", fn);
  if (e->ln_stats)
    SVI_REQUIRE(e->ln_u && e->ln_dim > 0 && (reinterpret_cast<uintptr_t>(e->ln_stats) & 7) == 0 &&
                    (reinterpret_cast<uintptr_t>(e->ln_u) & 7) == 0,
                "%s: ln fold needs ln_u (8-byte aligned), ln_dim > 0 and 8-byte aligned ln_stats", fn);
  if (e->a_next)
    SVI_REQUIRE(e->g_next && e->row_stats && e->ld_an >= N && e->ld_an % 8 == 0 &&
                    (reinterpret_cast<uintptr_t>(e->a_next) & 15) == 0 && (reinterpret_cast<uintptr_t>(e->g_next) & 7) == 0,
                "%s: a_next needs g_next, row_stats, ld_an >= N (multiple of 8) and 16-byte alignment", fn);

  int rc = make_tmap_2d(ta, A, 2, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, BK, BM);
  if (rc) return rc;
  rc = make_w_tmap(tb, W, ldw, N, K, e->w_e4m3 != 0);
  if (rc) return rc;

  ep->out = e->out; ep->ldo = e->ldo;
  ep->bias = e->bias; ep->gate = e->gate; ep->residual = e->residual; ep->ldr = e->ldr;
  ep->sumsq = e->sumsq; ep->sumsq_groups = e->sumsq_groups; ep->sumsq_group_cols = e->sumsq_group_cols;
  ep->sumsq_parts = e->sumsq_parts; ep->sumsq_col0 = 0;
  ep->ln_stats = e->ln_stats; ep->ln_u = e->ln_u; ep->ln_inv_d = e->ln_dim > 0 ? 1.0f / (float)e->ln_dim : 0.f;
  ep->ln_eps = e->ln_eps;
  ep->a_next = reinterpret_cast<__nv_bfloat16*>(e->a_next); ep->ld_an = e->ld_an; ep->g_next = e->g_next;
  ep->row_stats = e->row_stats;
  return SVI_OK;
}

}  // namespace gemm
}  // namespace svi

extern "C" int svi_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, int32_t M,
                             int32_t N, int32_t K, const svi_gemm_epilogue* e, void* stream) {
  using namespace svi;
  using namespace svi::gemm;
  CUtensorMap ta, tb;
  Epi ep;
  const int rc = prepare("svi_gemm_bf16", A, lda, W, ldw, M, N, K, e, &ta, &tb, &ep);
  if (rc) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool f32 = e->out_is_f32 != 0, fold = e->ln_stats || e->a_next;
  const LoRAArgs<false> none{};
  return e->w_e4m3 ? launch_kind<true>(ta, tb, M, N, K, e->act, f32, fold, ep, none, st)
                   : launch_kind<false>(ta, tb, M, N, K, e->act, f32, fold, ep, none, st);
}

extern "C" int svi_gemm_lora_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, int32_t M, int32_t N, int32_t K,
                                  const svi_gemm_epilogue* e, const svi_gemm_lora* lora, void* stream) {
  using namespace svi;
  using namespace svi::gemm;
  CUtensorMap ta, tb;
  Epi ep;
  int rc = prepare("svi_gemm_lora_bf16", A, lda, W, ldw, M, N, K, e, &ta, &tb, &ep);
  if (rc) return rc;
  SVI_REQUIRE(lora && lora->U && lora->B, "svi_gemm_lora_bf16: null LoRA pointer");
  SVI_REQUIRE(lora->R > 0 && lora->R % BK == 0, "svi_gemm_lora_bf16: R must be a positive multiple of 64 (got %d)", lora->R);
  SVI_REQUIRE(lora->group_cols == 0 || (lora->group_cols > 0 && lora->group_cols % EPI_N == 0 && N % lora->group_cols == 0),
              "svi_gemm_lora_bf16: group_cols must be 0 or a multiple of 128 that divides N (got %d, N=%d)", lora->group_cols, N);
  const int64_t groups = lora->group_cols ? N / lora->group_cols : 1;
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(lora->U) & 15) == 0 && (reinterpret_cast<uintptr_t>(lora->B) & 15) == 0,
              "svi_gemm_lora_bf16: U and B must be 16-byte aligned");
  SVI_REQUIRE(lora->ldu >= groups * lora->R && lora->ldu % 8 == 0 && lora->ldb >= lora->R && lora->ldb % 8 == 0,
              "svi_gemm_lora_bf16: ldu must be >= groups * R and ldb >= R, both multiples of 8 (ldu=%lld ldb=%lld)",
              (long long)lora->ldu, (long long)lora->ldb);
  SVI_REQUIRE(e->act == SVI_ACT_NONE || e->act == SVI_ACT_GELU_TANH,
              "svi_gemm_lora_bf16: activation %d has no LoRA kernel (none or GELU-tanh)", e->act);
  SVI_REQUIRE(!e->ln_stats && !e->a_next, "svi_gemm_lora_bf16: the LayerNorm fold (ln_* / a_next) cannot take a LoRA segment");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool f32 = e->out_is_f32 != 0;
  LoRAArgs<true> la;
  la.kb = lora->R / BK;
  la.group_cols = lora->group_cols;
  if (lora->group_cols % BN == 0) {
    rc = make_tmap_2d(&la.u, lora->U, 2, (uint64_t)(groups * lora->R), (uint64_t)M, (uint64_t)lora->ldu * 2, BK, BM);
    if (rc) return rc;
    rc = make_tmap_2d(&la.b, lora->B, 2, (uint64_t)lora->R, (uint64_t)N, (uint64_t)lora->ldb * 2, BK, BN);
    if (rc) return rc;
    return e->w_e4m3 ? launch_kind<true>(ta, tb, M, N, K, e->act, f32, false, ep, la, st)
                     : launch_kind<false>(ta, tb, M, N, K, e->act, f32, false, ep, la, st);
  }
  // Groups of an odd multiple of 128 columns: a 256-column tile would straddle two groups, so each group is a launch of
  // its own on its columns of W, B and the epilogue operands, with its block of U.
  const int gc = lora->group_cols;
  la.group_cols = 0;
  for (int64_t g = 0; g < groups; ++g) {
    const int64_t c0 = g * gc;
    Epi eg = ep;
    eg.out = static_cast<char*>(ep.out) + c0 * (f32 ? 4 : 2);
    if (eg.bias) eg.bias += c0;
    if (eg.gate) eg.gate += c0;
    if (eg.residual) eg.residual += c0;
    eg.sumsq_col0 = (int)c0;
    CUtensorMap tw;
    rc = make_w_tmap(&tw, static_cast<const char*>(W) + c0 * ldw * (e->w_e4m3 ? 1 : 2), ldw, gc, K, e->w_e4m3 != 0);
    if (rc) return rc;
    rc = make_tmap_2d(&la.u, static_cast<const char*>(lora->U) + g * lora->R * 2, 2, (uint64_t)lora->R, (uint64_t)M,
                      (uint64_t)lora->ldu * 2, BK, BM);
    if (rc) return rc;
    rc = make_tmap_2d(&la.b, static_cast<const char*>(lora->B) + c0 * lora->ldb * 2, 2, (uint64_t)lora->R, (uint64_t)gc,
                      (uint64_t)lora->ldb * 2, BK, BN);
    if (rc) return rc;
    rc = e->w_e4m3 ? launch_kind<true>(ta, tw, M, gc, K, e->act, f32, false, eg, la, st)
                   : launch_kind<false>(ta, tw, M, gc, K, e->act, f32, false, eg, la, st);
    if (rc) return rc;
  }
  return SVI_OK;
}
