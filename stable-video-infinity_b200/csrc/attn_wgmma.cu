// Non-causal flash attention forward for sm_90a, head_dim 128, bf16 operands, fp32 softmax.
//
// One CTA owns one 128-row Q tile of one head and streams K/V tiles of 128 rows past it:
//
//   warpgroup 0     : TMA producer (one lane: Q once, then K_j / V_j into 2-stage rings, 128B-swizzled boxes)   40 registers
//   warpgroups 1, 2 : consumers, 64 Q rows each:  S = Q K_j^T (wgmma, both operands in shared memory, S in registers),
//                     online softmax in registers, O += P V_j (wgmma with P as the register A operand, V MN-major)  232 registers
//
// The two consumer warpgroups run independently, so the softmax of one overlaps the tensor-core work of the other.
// Work units are (head, Q tile).  The launch plan (plan_split, host side) runs `n_full` units whole and cuts each of the
// remaining ones into `split` slices of the K/V stream, so the last, partly filled wave of CTAs is spread over all SMs;
// sliced units leave (unnormalised O, row max, row sum) in a workspace and attn_merge_kernel combines them.  Without a
// workspace every unit runs whole.
// Replaces flash_attention(), reference wan_video_dit.py:116-147.
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/svi_b200.h"

namespace svi {
namespace attn {

constexpr int BQ = 128;
constexpr int BKV = 128;
constexpr int HD = 128;
constexpr int KV_STAGES = 2;
constexpr int HALF_BYTES = 128 * 64 * 2;   // one 128-row x 64-col swizzled box (16 KB)
constexpr int TILE_BYTES = 2 * HALF_BYTES;  // 128 x 128 bf16 (32 KB)
constexpr int NUM_THREADS = 384;
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
constexpr uint32_t OFF_Q = 0;
constexpr uint32_t OFF_K = TILE_BYTES;                          // [KV_STAGES][TILE_BYTES]
constexpr uint32_t OFF_V = OFF_K + KV_STAGES * TILE_BYTES;      // [KV_STAGES][TILE_BYTES]
constexpr uint32_t OFF_BAR = OFF_V + KV_STAGES * TILE_BYTES;
constexpr int SMEM_BYTES = OFF_BAR + 1024 + 256;
enum : uint32_t { Q_FULL = 0, K_FULL = 1, K_EMPTY = 3, V_FULL = 5, V_EMPTY = 7, NUM_BARS = 9 };

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct Params {
  __nv_bfloat16* O;
  long long ldo;
  int Lq, Lk;
  float scale_log2;  // softmax scale * log2(e)
  int accumulate;
  // sequence-parallel K/V stream (sp_exchange.cu); kv_flags == nullptr: plain attention
  const uint32_t* kv_flags;  // [n_chunks] arrival flag of each source rank's rows, written by that rank's push
  uint32_t kv_epoch;         // value a flag holds once the rows of this launch have landed
  int kv_chunk_rows;         // rows owned by each rank
  int kv_self_chunk;         // this rank's chunk: produced locally, never waited for
  int kv_first_tile;         // KV tile the stream starts on (first tile fully inside the local chunk)
  // launch plan: units [0, n_full) whole; unit n_full + t/split gets slice t%split of the K/V stream
  int n_qtiles;              // Q tiles per head
  int n_full;
  int split;
  float* ws_o;               // [slices][128 rows][128] unnormalised partial O
  float2* ws_ml;             // [slices][128 rows] (row max in scaled log2 units, row sum)
  // optional per-row RMS scale of Q (full-width RMSNorm folded into the softmax scale): row r of Q is used as
  // Q[r] * rsqrt(sum_{j < q_ss_parts} q_sumsq[r * q_ss_ld + j] * q_inv_d + q_eps); nullptr: none
  const float* q_sumsq;
  int q_ss_ld, q_ss_parts;
  float q_inv_d, q_eps;
};

__device__ __forceinline__ float q_row_sumsq(const Params& p, int qrow) {   // partials added in index order: reproducible
  const float* sp = p.q_sumsq + (long long)qrow * p.q_ss_ld;
  float s = __ldg(sp);
  for (int j = 1; j < p.q_ss_parts; ++j) s += __ldg(sp + j);
  return s;
}

// KV tile visited at iteration j: the stream starts on the rank's own rows and wraps around
__device__ __forceinline__ int kv_tile_at(int j, int first_tile, int n_kv) {
  const int t = j + first_tile;
  return t >= n_kv ? t - n_kv : t;
}

// Producer side of the K/V exchange: block until the rows of `chunk` have been pushed into this GPU's buffer.
__device__ __forceinline__ void wait_kv_chunk(const uint32_t* flags, int chunk, uint32_t epoch) {
  const uint32_t* f = flags + chunk;
  uint32_t v;
  uint32_t spins = 0;
  while (true) {
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
    if (v == epoch) break;
    __nanosleep(64);
    // > 2 s: a peer died or the protocol is broken -> visible error, not a hang (no printf: a function call anywhere in
    // the kernel makes ptxas serialise its wgmma pipeline)
    if (++spins > (1u << 25)) __trap();
  }
  asm volatile("fence.proxy.async.global;" ::: "memory");   // later TMA (async proxy) reads see the pushed rows
}

struct Unit {
  int head, q_row0, j_begin, n_kv, n_kv_total, slice_slot;
};
__device__ __forceinline__ Unit decode_unit(const Params& p) {
  Unit u;
  u.n_kv_total = (p.Lk + BKV - 1) / BKV;
  int unit = blockIdx.x;
  u.j_begin = 0;
  u.n_kv = u.n_kv_total;                            // K/V tiles THIS CTA streams, starting at j_begin
  u.slice_slot = (int)blockIdx.x - p.n_full;        // >= 0: this CTA computes one slice of a unit
  if (u.slice_slot >= 0) {
    unit = p.n_full + u.slice_slot / p.split;
    const int sl = u.slice_slot % p.split;
    u.j_begin = (int)((long long)u.n_kv_total * sl / p.split);
    u.n_kv = (int)((long long)u.n_kv_total * (sl + 1) / p.split) - u.j_begin;
  }
  u.head = unit / p.n_qtiles;
  u.q_row0 = (unit % p.n_qtiles) * BQ;
  return u;
}

// ------------------------------------ TMA producer (one lane) ------------------------------------
__device__ __forceinline__ void producer(const CUtensorMap* tmap_q, const CUtensorMap* tmap_k, const CUtensorMap* tmap_v,
                                         const Params& p, uint32_t sbase) {
  const Unit u = decode_unit(p);
  const uint32_t bars = sbase + OFF_BAR;
  const int col0 = u.head * HD;
  auto load_tile = [&](uint32_t dst, const CUtensorMap* m, uint32_t bar, int row) {
    mbar_expect_tx_a(bar, TILE_BYTES);
    tma_load_2d_a(dst, m, bar, col0, row);
    tma_load_2d_a(dst + HALF_BYTES, m, bar, col0 + 64, row);
  };
  load_tile(sbase + OFF_Q, tmap_q, bars + 8 * Q_FULL, u.q_row0);
  int landed = p.kv_self_chunk;   // most recent remote chunk known to be present (chunks are visited in runs)
  for (int j = 0; j < u.n_kv; ++j) {
    const int s = j % KV_STAGES;
    const uint32_t ph = (j / KV_STAGES) & 1;
    const int row = kv_tile_at(u.j_begin + j, p.kv_first_tile, u.n_kv_total) * BKV;
    if (p.kv_flags) {
      const int c0 = row / p.kv_chunk_rows;
      const int c1 = (min(row + BKV, p.Lk) - 1) / p.kv_chunk_rows;
      for (int c = c0; c <= c1; ++c) {
        if (c == p.kv_self_chunk || c == landed) continue;
        wait_kv_chunk(p.kv_flags, c, p.kv_epoch);
        landed = c;
      }
    }
    mbar_wait_a(bars + 8 * (K_EMPTY + s), ph ^ 1);
    load_tile(sbase + OFF_K + s * TILE_BYTES, tmap_k, bars + 8 * (K_FULL + s), row);
    mbar_wait_a(bars + 8 * (V_EMPTY + s), ph ^ 1);
    load_tile(sbase + OFF_V + s * TILE_BYTES, tmap_v, bars + 8 * (V_FULL + s), row);
  }
}

// ------------------------------------ consumer warpgroup (64 Q rows) ------------------------------
// Thread fragment of S and O (wgmma m64n128): rows r0 = 16 * warp + g and r0 + 8 (g = lane / 4), columns 8j + 2c, +1
// (c = lane % 4) for j = 0..15: element 4j + 2h + e is (row r0 + 8h, column 8j + 2c + e).
__device__ __forceinline__ void consumer(const Params& p, uint32_t sbase, int cw, int warp, int lane) {
  const Unit u = decode_unit(p);
  const uint32_t bars = sbase + OFF_BAR;
  const int g = lane >> 2, c = lane & 3;
  const int r_tile = cw * 64 + warp * 16 + g;   // row inside the Q tile (and + 8)
  float cs[2] = {p.scale_log2, p.scale_log2};
  if (p.q_sumsq) {          // the Q row carries its RMSNorm factor in the softmax scale
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int qrow = min(u.q_row0 + r_tile + 8 * h, p.Lq - 1);
      cs[h] *= rsqrtf(q_row_sumsq(p, qrow) * p.q_inv_d + p.q_eps);
    }
  }
  float m_cur[2] = {-INFINITY, -INFINITY};  // running row max (scaled, log2 domain); reference point of P and O
  float l[2] = {0.f, 0.f};                  // this thread's share of the running row sum of P
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  const uint32_t q_rows = sbase + OFF_Q + cw * 64 * 128;   // this warpgroup's 64 rows inside each 128-row box

  mbar_wait_a(bars + 8 * Q_FULL, 0);
  for (int j = 0; j < u.n_kv; ++j) {
    const int s = j % KV_STAGES;
    const uint32_t ph = (j / KV_STAGES) & 1;
    float sc[64];
    mbar_wait_a(bars + 8 * (K_FULL + s), ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {   // 8 K-steps: 4 per 64-column box, +32 B each
      const uint32_t box = (kk >> 2) * HALF_BYTES, koff = (kk & 3) * 32;
      Wgmma<128>::ss(sc, wgmma_desc(q_rows + box + koff, 16, 1024),
                     wgmma_desc(sbase + OFF_K + s * TILE_BYTES + box + koff, 16, 1024), kk != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    if (lane == 0) mbar_arrive_a(bars + 8 * (K_EMPTY + s));

    const int limit = p.Lk - kv_tile_at(u.j_begin + j, p.kv_first_tile, u.n_kv_total) * BKV;  // valid key columns
    if (limit < BKV) {
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (8 * (i >> 2) + 2 * c + (i & 1) >= limit) sc[i] = -INFINITY;
    }
    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(sc[4 * jj + 2 * h], sc[4 * jj + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_cur[h], mx * cs[h]);
      alpha[h] = ex2(m_cur[h] - m_new);   // 0 on the first tile (m_cur = -inf)
      m_cur[h] = m_new;
      l[h] *= alpha[h];
    }
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] *= alpha[(i >> 1) & 1];
    // P = exp2(S * c - m) (masked columns: exp2(-inf) = 0) -> bf16 A fragments of the P V MMA
    uint32_t pa[8][4];
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int h = (i >> 1) & 1;
      const float p0 = ex2(fmaf(sc[i], cs[h], -m_cur[h]));
      const float p1 = ex2(fmaf(sc[i + 1], cs[h], -m_cur[h]));
      l[h] += p0 + p1;
      pa[i >> 3][(i >> 1) & 3] = pack_bf16x2(p0, p1);
    }
    mbar_wait_a(bars + 8 * (V_FULL + s), ph);
    wgmma_fence();
#pragma unroll
    for (int t = 0; t < BKV / 16; ++t)   // 16 K/V rows per step = two 8-row swizzle groups = 2048 B; LBO = next 64 columns
      Wgmma<128>::rs_tb(o, pa[t], wgmma_desc(sbase + OFF_V + s * TILE_BYTES + t * 2048, HALF_BYTES, 1024), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    if (lane == 0) mbar_arrive_a(bars + 8 * (V_EMPTY + s));
  }

#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
  }
  if (u.slice_slot >= 0 && p.split > 1) {
    // one slice of the K/V stream: leave (O, m, l) for attn_merge_kernel
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long prow = (long long)u.slice_slot * BQ + r_tile + 8 * h;
      float* dst = p.ws_o + prow * HD + 2 * c;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
        *reinterpret_cast<float2*>(dst + 8 * jj) = make_float2(o[4 * jj + 2 * h], o[4 * jj + 2 * h + 1]);
      if (c == 0) p.ws_ml[prow] = make_float2(m_cur[h], l[h]);
    }
  } else {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = u.q_row0 + r_tile + 8 * h;
      if (row >= p.Lq) continue;
      const float inv_l = 1.0f / l[h];
      __nv_bfloat16* orow = p.O + (long long)row * p.ldo + u.head * HD + 2 * c;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        float v0 = o[4 * jj + 2 * h] * inv_l, v1 = o[4 * jj + 2 * h + 1] * inv_l;
        uint32_t* dst = reinterpret_cast<uint32_t*>(orow + 8 * jj);
        if (p.accumulate) {
          const uint32_t old = *dst;
          const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&old));
          v0 += f.x;
          v1 += f.y;
        }
        *dst = pack_bf16x2(v0, v1);
      }
    }
  }
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ Params p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    const uint32_t bars = sbase + OFF_BAR;
    for (uint32_t b = 0; b < NUM_BARS; ++b)
      mbar_init_a(bars + 8 * b, (b == K_EMPTY || b == K_EMPTY + 1 || b == V_EMPTY || b == V_EMPTY + 1) ? 8u : 1u);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) producer(&tmap_q, &tmap_k, &tmap_v, p, sbase);
  } else {
    setmaxnreg_inc<CONSUMER_REGS>();
    consumer(p, sbase, (warp >> 2) - 1, warp & 3, lane);
  }
}

constexpr size_t SLICE_BYTES = (size_t)BQ * HD * 4 + (size_t)BQ * 8;   // partial O + (m, l) of one slice
constexpr int MAX_SPLIT = 8;
constexpr int MIN_SLICE_TILES = 8;   // a slice shorter than this is dominated by its prologue / epilogue

// Combines the slices of the sliced units: one warp per Q row (lane = 4 output columns), 8 rows per block.
__global__ void __launch_bounds__(256)
attn_merge_kernel(const float* __restrict__ ws_o, const float2* __restrict__ ws_ml, int split, int n_full, int n_qtiles,
                  int Lq, __nv_bfloat16* __restrict__ O, long long ldo) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x / (BQ / 8);                       // sliced unit
  const int r = (blockIdx.x % (BQ / 8)) * 8 + warp;          // row inside the unit's 128
  const int unit = n_full + t;
  const int head = unit / n_qtiles;
  const int row = (unit % n_qtiles) * BQ + r;
  if (row >= Lq) return;
  float m = -INFINITY;
  for (int s = 0; s < split; ++s) m = fmaxf(m, ws_ml[((long long)t * split + s) * BQ + r].x);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float l = 0.f;
  for (int s = 0; s < split; ++s) {
    const long long prow = ((long long)t * split + s) * BQ + r;
    const float2 ml = ws_ml[prow];
    const float w = ex2(ml.x - m);
    const float4 o = __ldcs(reinterpret_cast<const float4*>(ws_o + prow * HD) + lane);
    acc.x += o.x * w; acc.y += o.y * w; acc.z += o.z * w; acc.w += o.w * w;
    l += ml.y * w;
  }
  const float inv = 1.0f / l;
  uint2 pk;
  pk.x = pack_bf16x2(acc.x * inv, acc.y * inv);
  pk.y = pack_bf16x2(acc.z * inv, acc.w * inv);
  *reinterpret_cast<uint2*>(O + (long long)row * ldo + head * HD + lane * 4) = pk;
}

// Launch plan: `units` equal CTAs on `sms` SMs cost ceil(units/sms) rounds.  Running r rounds of whole units and cutting
// the remaining t units into S slices costs r + ceil(t*S/sms)/S rounds (+ a little for the merge).  Returns the cheapest
// (n_full, split) that fits the workspace; (units, 1) when slicing does not pay.
static void plan_split(int units, int n_kv, int sms, size_t ws_bytes, int* n_full, int* split) {
  *n_full = units;
  *split = 1;
  if (ws_bytes < SLICE_BYTES || units <= 0) return;
  const int rounds = units / sms;
  double best = (double)((units + sms - 1) / sms);
  const double need = best * 0.985;   // must save at least 1.5 %
  for (int r = rounds; r >= 0 && r >= rounds - 1; --r) {
    const int t = units - r * sms;
    if (t <= 0) continue;
    for (int S = 2; S <= MAX_SPLIT; ++S) {
      if (n_kv / S < MIN_SLICE_TILES) break;
      const long long slices = (long long)t * S;
      if ((size_t)slices * SLICE_BYTES > ws_bytes) break;
      const double cost = r + (double)((slices + sms - 1) / sms) / S + 0.04 * (double)t / sms + 0.01 * S;
      if (cost < best && cost < need) {
        best = cost;
        *n_full = units - t;
        *split = S;
      }
    }
  }
}

struct QScale {
  const float* sumsq = nullptr;
  int ld = 0;
  int parts = 1;
  int dim = 1;
  float eps = 0.f;
};

static int launch_attn(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* O,
                       int64_t ldo, int32_t Lq, int32_t Lk, int32_t num_heads, float scale, int32_t accumulate,
                       const uint32_t* kv_flags, uint32_t kv_epoch, int kv_chunk_rows, int kv_self_chunk, void* workspace,
                       size_t workspace_bytes, void* stream, const char* who, QScale qs = QScale()) {
  SVI_REQUIRE(Q && K && V && O, "%s: null pointer", who);
  SVI_REQUIRE(Lq > 0 && Lk > 0 && num_heads > 0, "%s: Lq, Lk, num_heads must be positive", who);
  const int64_t width = (int64_t)num_heads * HD;
  SVI_REQUIRE(ldq >= width && ldk >= width && ldv >= width && ldo >= width,
              "%s: leading dimensions must be >= num_heads*128", who);
  SVI_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0,
              "%s: leading dimensions must be multiples of 8 elements", who);
  SVI_REQUIRE(((reinterpret_cast<uintptr_t>(Q) | reinterpret_cast<uintptr_t>(K) |
                reinterpret_cast<uintptr_t>(V) | reinterpret_cast<uintptr_t>(O)) & 15) == 0,
              "%s: pointers must be 16-byte aligned", who);
  CUtensorMap tq, tk, tv;
  int rc = make_tmap_2d(&tq, Q, 2, (uint64_t)width, (uint64_t)Lq, (uint64_t)ldq * 2, 64, BQ);
  if (rc) return rc;
  rc = make_tmap_2d(&tk, K, 2, (uint64_t)width, (uint64_t)Lk, (uint64_t)ldk * 2, 64, BKV);
  if (rc) return rc;
  rc = make_tmap_2d(&tv, V, 2, (uint64_t)width, (uint64_t)Lk, (uint64_t)ldv * 2, 64, BKV);
  if (rc) return rc;

  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t ce = cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          SMEM_BYTES);
    if (ce != cudaSuccess) {
      set_last_error("%s: cudaFuncSetAttribute failed: %s", who, cudaGetErrorString(ce));
      return SVI_ERR_LAUNCH;
    }
    attr_set = true;
  }
  Params p;
  p.O = reinterpret_cast<__nv_bfloat16*>(O);
  p.ldo = ldo;
  p.Lq = Lq;
  p.Lk = Lk;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.accumulate = accumulate;
  p.kv_flags = kv_flags;
  p.kv_epoch = kv_epoch;
  p.kv_chunk_rows = kv_chunk_rows;
  p.kv_self_chunk = kv_self_chunk;
  p.q_sumsq = qs.sumsq;
  p.q_ss_ld = qs.ld;
  p.q_ss_parts = qs.parts;
  p.q_inv_d = 1.0f / (float)qs.dim;
  p.q_eps = qs.eps;
  p.kv_first_tile = 0;
  if (kv_flags) {
    const int n_kv = (Lk + BKV - 1) / BKV;
    const int first = (int)(((int64_t)kv_self_chunk * kv_chunk_rows + BKV - 1) / BKV);
    p.kv_first_tile = first >= n_kv ? 0 : first;
  }
  p.n_qtiles = (Lq + BQ - 1) / BQ;
  const int units = p.n_qtiles * num_heads;
  const int sms = sm_count();
  if (sms <= 0) return SVI_ERR_DRIVER;
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "%s: workspace must be 16-byte aligned", who);
  plan_split(units, (Lk + BKV - 1) / BKV, sms, (workspace && !accumulate) ? workspace_bytes : 0, &p.n_full, &p.split);
  const int n_sliced = units - p.n_full;
  const long long slices = (long long)n_sliced * p.split;
  p.ws_o = static_cast<float*>(workspace);
  p.ws_ml = reinterpret_cast<float2*>(static_cast<char*>(workspace) + (size_t)slices * BQ * HD * 4);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  attn_fwd_kernel<<<(unsigned)(p.n_full + slices), NUM_THREADS, SMEM_BYTES, st>>>(tq, tk, tv, p);
  SVI_CUDA_LAUNCH_CHECK(who);
  if (p.split > 1) {
    attn_merge_kernel<<<n_sliced * (BQ / 8), 256, 0, st>>>(p.ws_o, p.ws_ml, p.split, p.n_full, p.n_qtiles, Lq, p.O, ldo);
    SVI_CUDA_LAUNCH_CHECK(who);
  }
  return SVI_OK;
}

}  // namespace attn
}  // namespace svi

extern "C" int svi_attn_fwd(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V,
                            int64_t ldv, void* O, int64_t ldo, int32_t Lq, int32_t Lk,
                            int32_t num_heads, float scale, int32_t accumulate, void* workspace,
                            size_t workspace_bytes, void* stream) {
  return svi::attn::launch_attn(Q, ldq, K, ldk, V, ldv, O, ldo, Lq, Lk, num_heads, scale, accumulate, nullptr, 0, 1, 0,
                                workspace, workspace_bytes, stream, "svi_attn_fwd");
}

extern "C" int svi_attn_fwd_qscale(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv,
                                   void* O, int64_t ldo, int32_t Lq, int32_t Lk, int32_t num_heads, float scale,
                                   int32_t accumulate, const float* q_sumsq, int32_t q_ss_ld, int32_t q_ss_parts, int32_t q_dim,
                                   float q_eps, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace svi;
  SVI_REQUIRE(q_sumsq && q_ss_ld >= 1 && q_dim >= 1 && q_ss_parts >= 0 && q_ss_parts <= q_ss_ld,
              "svi_attn_fwd_qscale: need q_sumsq, q_ss_ld >= 1, q_dim >= 1, 0 <= q_ss_parts <= q_ss_ld");
  svi::attn::QScale qs;
  qs.sumsq = q_sumsq;
  qs.ld = q_ss_ld;
  qs.parts = q_ss_parts > 0 ? q_ss_parts : 1;
  qs.dim = q_dim;
  qs.eps = q_eps;
  return svi::attn::launch_attn(Q, ldq, K, ldk, V, ldv, O, ldo, Lq, Lk, num_heads, scale, accumulate, nullptr, 0, 1, 0,
                                workspace, workspace_bytes, stream, "svi_attn_fwd_qscale", qs);
}

extern "C" void svi_attn_plan(int32_t units, int32_t kv_tiles, int32_t sms, size_t workspace_bytes, int32_t* n_full,
                              int32_t* split) {
  int a = units, b = 1;
  if (sms > 0) svi::attn::plan_split(units, kv_tiles, sms, workspace_bytes, &a, &b);
  if (n_full) *n_full = a;
  if (split) *split = b;
}

extern "C" size_t svi_attn_workspace_bytes(int32_t Lq, int32_t Lk, int32_t num_heads) {
  // enough for the largest plan plan_split can choose: up to two rounds of units, each cut into MAX_SPLIT slices
  using namespace svi::attn;
  (void)Lk;
  const long long units = (long long)((Lq + BQ - 1) / BQ) * num_heads;
  const int sms = svi::sm_count();
  const long long tail = units < 2LL * sms ? units : 2LL * sms;
  return (size_t)tail * MAX_SPLIT * SLICE_BYTES;
}

extern "C" int svi_attn_fwd_sp(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V,
                               int64_t ldv, void* O, int64_t ldo, int32_t Lq, int32_t Lk,
                               int32_t num_heads, float scale, const void* kv_flags, uint32_t kv_epoch,
                               int32_t kv_chunk_rows, int32_t kv_self_chunk, void* workspace, size_t workspace_bytes,
                               void* stream) {
  using namespace svi;
  SVI_REQUIRE(kv_flags, "svi_attn_fwd_sp: kv_flags is null");
  SVI_REQUIRE(kv_chunk_rows >= 128 && kv_self_chunk >= 0 && (int64_t)kv_self_chunk * kv_chunk_rows < Lk,
              "svi_attn_fwd_sp: need kv_chunk_rows >= 128 and the local chunk inside [0, Lk)");
  return svi::attn::launch_attn(Q, ldq, K, ldk, V, ldv, O, ldo, Lq, Lk, num_heads, scale, 0,
                                static_cast<const uint32_t*>(kv_flags), kv_epoch, kv_chunk_rows, kv_self_chunk, workspace,
                                workspace_bytes, stream, "svi_attn_fwd_sp");
}
