// Memory-bound row / elementwise kernels of the DiT hot path (HBM-bound: vectorised 16-byte accesses,
// one pass over the data, fp32 math).  Each replaces a chain of separate torch elementwise launches
// in the reference (line map in include/svi_b200.h).
#include "common.cuh"
#include "../../include/svi_b200.h"

namespace svi {
namespace ew {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum for blockDim.x == 128 (4 warps); every thread gets the result
__device__ __forceinline__ float block_sum_128(float v, float* red /*[4]*/) {
  v = warp_sum(v);
  __syncthreads();  // protect `red` reuse
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  return red[0] + red[1] + red[2] + red[3];
}

// ---------------------------------------------------------------------------------------------
// LayerNorm (+affine) (+modulate) -> bf16.  One 128-thread block per row, row cached in registers.
// ---------------------------------------------------------------------------------------------
constexpr int LN_THREADS = 128;
constexpr int LN_MAX_VEC = 16;  // float4 per thread -> D <= 8192

// y_lo != nullptr: split output — y holds bf16(v), y_lo holds bf16(v - bf16(v)), so that y + y_lo carries ~16 mantissa
// bits of v (the A operand of the head GEMM is fed as two bf16 passes; DESIGN.md section 2).
__global__ void __launch_bounds__(LN_THREADS)
layernorm_modulate_kernel(const float* __restrict__ x, int D, float eps, const float* __restrict__ gamma,
                          const float* __restrict__ beta, const float* __restrict__ scale,
                          const float* __restrict__ shift, __nv_bfloat16* __restrict__ y, long long ldy,
                          __nv_bfloat16* __restrict__ y_lo) {
  __shared__ float red[4];
  const long long row = blockIdx.x;
  const float4* xr = reinterpret_cast<const float4*>(x + row * D);
  const int nvec = D >> 2;
  float4 v[LN_MAX_VEC];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    const int idx = threadIdx.x + i * LN_THREADS;
    if (idx < nvec) {
      v[i] = xr[idx];
      s += v[i].x + v[i].y + v[i].z + v[i].w;
    }
  }
  const float mean = block_sum_128(s, red) / (float)D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    const int idx = threadIdx.x + i * LN_THREADS;
    if (idx < nvec) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += a * a + b * b + c * c + d * d;
    }
  }
  const float rstd = rsqrtf(block_sum_128(q, red) / (float)D + eps);
  uint2* yr = reinterpret_cast<uint2*>(y + row * ldy);
  uint2* yl = y_lo ? reinterpret_cast<uint2*>(y_lo + row * ldy) : nullptr;
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    const int idx = threadIdx.x + i * LN_THREADS;
    if (idx < nvec) {
      float o[4] = {(v[i].x - mean) * rstd, (v[i].y - mean) * rstd, (v[i].z - mean) * rstd,
                    (v[i].w - mean) * rstd};
      if (gamma) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + idx);
        o[0] *= g.x; o[1] *= g.y; o[2] *= g.z; o[3] *= g.w;
      }
      if (beta) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + idx);
        o[0] += b.x; o[1] += b.y; o[2] += b.z; o[3] += b.w;
      }
      if (scale) {
        const float4 sc = __ldg(reinterpret_cast<const float4*>(scale) + idx);
        o[0] *= 1.f + sc.x; o[1] *= 1.f + sc.y; o[2] *= 1.f + sc.z; o[3] *= 1.f + sc.w;
      }
      if (shift) {
        const float4 sh = __ldg(reinterpret_cast<const float4*>(shift) + idx);
        o[0] += sh.x; o[1] += sh.y; o[2] += sh.z; o[3] += sh.w;
      }
      uint2 pk;
      pk.x = pack_bf16x2(o[0], o[1]);
      pk.y = pack_bf16x2(o[2], o[3]);
      yr[idx] = pk;
      if (yl) {
        const __nv_bfloat162* hb = reinterpret_cast<const __nv_bfloat162*>(&pk);
        const float2 h0 = __bfloat1622float2(hb[0]), h1 = __bfloat1622float2(hb[1]);
        uint2 lo;
        lo.x = pack_bf16x2(o[0] - h0.x, o[1] - h0.y);
        lo.y = pack_bf16x2(o[2] - h1.x, o[3] - h1.y);
        yl[idx] = lo;
      }
    }
  }
}


// Warp-per-row variant for D <= 2048 (the 1.3B model, D = 1536): no block barriers, the whole row is fetched with up
// to 16 independent 16-byte loads per lane before anything is reduced (memory-level parallelism is what an HBM-bound
// 6 KB-per-row kernel needs, and the block-per-row version above waits at its barriers with few loads in flight).
constexpr int LNW_WARPS = 8;
constexpr int LNW_MAX_VEC = 16;  // float4 per lane -> D <= 2048

// NV > 0: D == 128 * NV exactly (no bounds predicates, fewer registers -> 3 blocks per SM); NV == 0: any D <= 2048.
template <int NV>
__global__ void __launch_bounds__(LNW_WARPS * 32, NV > 0 ? 3 : 2)
layernorm_modulate_warp_kernel(const float* __restrict__ x, int M, int D, float eps, const float* __restrict__ gamma,
                               const float* __restrict__ beta, const float* __restrict__ scale,
                               const float* __restrict__ shift, __nv_bfloat16* __restrict__ y) {
  constexpr int CAP = NV > 0 ? NV : LNW_MAX_VEC;
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * LNW_WARPS + (threadIdx.x >> 5);
  if (row >= M) return;
  const float4* xr = reinterpret_cast<const float4*>(x + row * D);
  const int nvec = NV > 0 ? NV * 32 : (D >> 2);
  float4 v[CAP];
#pragma unroll
  for (int i = 0; i < CAP; ++i) {
    const int idx = lane + i * 32;
    if (NV > 0 || idx < nvec) v[i] = __ldcs(xr + idx);   // streaming: the fp32 residual row is not re-read soon
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < CAP; ++i)
    if (NV > 0 || lane + i * 32 < nvec) s += v[i].x + v[i].y + v[i].z + v[i].w;
  const float mean = warp_sum(s) / (float)D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < CAP; ++i)
    if (NV > 0 || lane + i * 32 < nvec) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += a * a + b * b + c * c + d * d;
    }
  const float rstd = rsqrtf(warp_sum(q) / (float)D + eps);
  uint2* yr = reinterpret_cast<uint2*>(y + row * D);
#pragma unroll
  for (int i = 0; i < CAP; ++i) {
    const int idx = lane + i * 32;
    if (NV > 0 || idx < nvec) {
      float o[4] = {(v[i].x - mean) * rstd, (v[i].y - mean) * rstd, (v[i].z - mean) * rstd, (v[i].w - mean) * rstd};
      if (gamma) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + idx);
        o[0] *= g.x; o[1] *= g.y; o[2] *= g.z; o[3] *= g.w;
      }
      if (beta) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + idx);
        o[0] += b.x; o[1] += b.y; o[2] += b.z; o[3] += b.w;
      }
      if (scale) {
        const float4 sc = __ldg(reinterpret_cast<const float4*>(scale) + idx);
        o[0] *= 1.f + sc.x; o[1] *= 1.f + sc.y; o[2] *= 1.f + sc.z; o[3] *= 1.f + sc.w;
      }
      if (shift) {
        const float4 sh = __ldg(reinterpret_cast<const float4*>(shift) + idx);
        o[0] += sh.x; o[1] += sh.y; o[2] += sh.z; o[3] += sh.w;
      }
      uint2 pk;
      pk.x = pack_bf16x2(o[0], o[1]);
      pk.y = pack_bf16x2(o[2], o[3]);
      __stcs(yr + idx, pk);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// full-width RMSNorm (row sum of squares supplied by the GEMM epilogue) + interleaved-pair RoPE,
// in place on bf16.  One thread = 8 consecutive columns (4 rotation pairs).
// ---------------------------------------------------------------------------------------------
// groups == 2: the row holds two D-wide vectors side by side (q | k of the fused QKV buffer), normalised with
// sumsq columns sumsq_col / sumsq_col + 1 and weights w / w2 — one launch instead of two.
__global__ void __launch_bounds__(256)
rmsnorm_rope_kernel(__nv_bfloat16* __restrict__ t, long long ldt, int M, int D, int groups,
                    const float* __restrict__ sumsq, int sumsq_ld, int sumsq_col, int parts, float eps,
                    const float* __restrict__ w, const float* __restrict__ w2, const float* __restrict__ rope_cos,
                    const float* __restrict__ rope_sin, int row_offset) {
  const int vec_per_row = (D >> 3) * groups;
  const long long total = (long long)M * vec_per_row;
  const float inv_d = 1.0f / (float)D;
  const bool warp_row = ((D >> 3) & 31) == 0;       // a warp's 32 x 8 columns never straddle a row or a group (D % 256 == 0)
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(i / vec_per_row);
    const int cc = (int)(i % vec_per_row) * 8;      // column inside the row (both groups)
    const int grp = cc >= D ? 1 : 0;
    const int c0 = cc - grp * D;                     // column inside the group
    // this thread's 8 values and weights first: the loads below them in program order would otherwise wait behind the
    // partial-sum loads and the shuffles (two serialized memory latencies per thread)
    uint4* ptr = reinterpret_cast<uint4*>(t + (long long)m * ldt + cc);
    const uint4 raw = *ptr;
    const float* wg = grp ? w2 : w;
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(wg + c0));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(wg + c0 + 4));
    // the group's sum of squares: one value (atomically accumulated) or `parts` partials added in index order (reproducible)
    const float* sp = sumsq + (long long)m * sumsq_ld + (long long)(sumsq_col + grp) * parts;
    float ssum;
    if (parts > 1 && warp_row) {
      // every lane of this warp works on the same (row, group): the partials are read once per warp (lane q takes partials q,
      // q + 32, ...) and added by a butterfly — commutative at every level, so all lanes hold the same bits, and the tree is
      // fixed, so the sum is reproducible.  (Every thread summing all partials itself made the pass L1-bound: 101 -> 133 us.)
      float a = 0.f;
      for (int q = threadIdx.x & 31; q < parts; q += 32) a += __ldg(sp + q);
#pragma unroll
      for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      ssum = a;
    } else if ((parts & 3) == 0 && (sumsq_ld & 3) == 0) {      // 16-byte loads, index order
      float4 a = __ldg(reinterpret_cast<const float4*>(sp));
      ssum = ((a.x + a.y) + a.z) + a.w;
      for (int q = 4; q < parts; q += 4) {
        a = __ldg(reinterpret_cast<const float4*>(sp + q));
        ssum = (((ssum + a.x) + a.y) + a.z) + a.w;
      }
    } else {
      ssum = sp[0];
      for (int q = 1; q < parts; ++q) ssum += sp[q];
    }
    const float rs = rsqrtf(ssum * inv_d + eps);
    const __nv_bfloat162* b2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
    float v[8];
    {
      const float2 a = __bfloat1622float2(b2[0]), b = __bfloat1622float2(b2[1]),
                   c = __bfloat1622float2(b2[2]), d = __bfloat1622float2(b2[3]);
      v[0] = a.x * rs * w0.x; v[1] = a.y * rs * w0.y; v[2] = b.x * rs * w0.z; v[3] = b.y * rs * w0.w;
      v[4] = c.x * rs * w1.x; v[5] = c.y * rs * w1.y; v[6] = d.x * rs * w1.z; v[7] = d.y * rs * w1.w;
    }
    if (rope_cos) {
      const int pair0 = (c0 & 127) >> 1;  // pair index inside the head (0..63), multiple of 4
      const long long ro = (long long)(m + row_offset) * 64 + pair0;
      const float4 cs = __ldg(reinterpret_cast<const float4*>(rope_cos + ro));
      const float4 sn = __ldg(reinterpret_cast<const float4*>(rope_sin + ro));
      const float cc[4] = {cs.x, cs.y, cs.z, cs.w};
      const float ss[4] = {sn.x, sn.y, sn.z, sn.w};
#pragma unroll
      for (int pidx = 0; pidx < 4; ++pidx) {
        const float re = v[2 * pidx], im = v[2 * pidx + 1];
        v[2 * pidx] = re * cc[pidx] - im * ss[pidx];
        v[2 * pidx + 1] = re * ss[pidx] + im * cc[pidx];
      }
    }
    uint4 pk;
    pk.x = pack_bf16x2(v[0], v[1]);
    pk.y = pack_bf16x2(v[2], v[3]);
    pk.z = pack_bf16x2(v[4], v[5]);
    pk.w = pack_bf16x2(v[6], v[7]);
    *ptr = pk;
  }
}

// ---------------------------------------------------------------------------------------------
// patchify gather / unpatchify scatter
// ---------------------------------------------------------------------------------------------
// split != 0: tok has 2*Kpad columns, [0, Kpad) = bf16(v), [Kpad, 2 Kpad) = bf16(v - bf16(v))
__global__ void __launch_bounds__(256)
patchify_gather_kernel(const float* __restrict__ x, int C0, const float* __restrict__ y, int C1, int F,
                       int H, int W, __nv_bfloat16* __restrict__ tok, int Kpad, int split) {
  const int h2 = H >> 1, w2 = W >> 1;
  const long long L = (long long)F * h2 * w2;
  const int C = C0 + C1;
  const int groups = Kpad >> 2;  // 4 columns (one channel's 2x2 patch) per thread
  const long long total = L * groups;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long tokn = i % L;  // token fastest -> coalesced reads along w
    const int c = (int)(i / L);
    uint2 pk = make_uint2(0u, 0u), lo = make_uint2(0u, 0u);
    if (c < C) {
      const int f = (int)(tokn / (h2 * w2));
      const int rem = (int)(tokn % (h2 * w2));
      const int hh = rem / w2, ww = rem % w2;
      const float* src = (c < C0) ? (x + (long long)c * F * H * W) : (y + (long long)(c - C0) * F * H * W);
      const float* p0 = src + ((long long)f * H + 2 * hh) * W + 2 * ww;
      const float2 r0 = *reinterpret_cast<const float2*>(p0);
      const float2 r1 = *reinterpret_cast<const float2*>(p0 + W);
      pk.x = pack_bf16x2(r0.x, r0.y);
      pk.y = pack_bf16x2(r1.x, r1.y);
      if (split) {
        const __nv_bfloat162* hb = reinterpret_cast<const __nv_bfloat162*>(&pk);
        const float2 h0 = __bfloat1622float2(hb[0]), h1 = __bfloat1622float2(hb[1]);
        lo.x = pack_bf16x2(r0.x - h0.x, r0.y - h0.y);
        lo.y = pack_bf16x2(r1.x - h1.x, r1.y - h1.y);
      }
    }
    const long long ld = split ? 2LL * Kpad : Kpad;
    *reinterpret_cast<uint2*>(tok + tokn * ld + c * 4) = pk;
    if (split) *reinterpret_cast<uint2*>(tok + tokn * ld + Kpad + c * 4) = lo;
  }
}

__global__ void __launch_bounds__(256)
unpatchify_kernel(const float* __restrict__ ho, long long ldh, int C, int F, int H, int W,
                  float* __restrict__ out) {
  const int h2 = H >> 1, w2 = W >> 1;
  const long long total = (long long)C * F * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(i % W);
    const int Y = (int)((i / W) % H);
    const int f = (int)((i / ((long long)W * H)) % F);
    const int c = (int)(i / ((long long)W * H * F));
    const long long tokn = ((long long)f * h2 + (Y >> 1)) * w2 + (X >> 1);
    const int col = (((Y & 1) << 1) | (X & 1)) * C + c;
    out[i] = ho[tokn * ldh + col];
  }
}

// ---------------------------------------------------------------------------------------------
// small elementwise kernels
// ---------------------------------------------------------------------------------------------
__global__ void cfg_euler_kernel(float* __restrict__ lat, const float* __restrict__ vc,
                                 const float* __restrict__ vu, long long n, float cfg, float dsigma) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float v = vc[i];
    if (vu) {
      const float u = vu[i];
      v = u + cfg * (v - u);
    }
    lat[i] += v * dsigma;
  }
}

// out = alpha * a + beta * b (TeaCache residual bookkeeping on the [L, d] token stream)
__global__ void axpby_kernel(const float4* __restrict__ a, float alpha, const float4* __restrict__ b, float beta,
                             float4* __restrict__ out, long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 x = a[i], y = b[i];
    out[i] = make_float4(alpha * x.x + beta * y.x, alpha * x.y + beta * y.y, alpha * x.z + beta * y.z,
                         alpha * x.w + beta * y.w);
  }
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ s, __nv_bfloat16* __restrict__ d,
                                     long long n, int act) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float v = s[i];
    if (act == SVI_ACT_SILU) v = silu(v);
    else if (act == SVI_ACT_GELU_TANH) v = gelu_tanh(v);
    else if (act == SVI_ACT_GELU_ERF) v = gelu_erf(v);
    d[i] = __float2bfloat16_rn(v);
  }
}
// dst[m, k] = bf16(v), dst[m, lo_col + k] = bf16(v - bf16(v)), v = act(src[m, k])
__global__ void split_f32_bf16x2_kernel(const float* __restrict__ s, long long lds, int M, int K, int act,
                                        __nv_bfloat16* __restrict__ d, long long ldd, int lo_col) {
  const long long n = (long long)M * K;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(i / K), k = (int)(i % K);
    float v = s[(long long)m * lds + k];
    if (act == SVI_ACT_SILU) v = silu(v);
    else if (act == SVI_ACT_GELU_TANH) v = gelu_tanh(v);
    else if (act == SVI_ACT_GELU_ERF) v = gelu_erf(v);
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    d[(long long)m * ldd + k] = hi;
    d[(long long)m * ldd + lo_col + k] = __float2bfloat16_rn(v - __bfloat162float(hi));
  }
}
__global__ void cast_bf16_f32_kernel(const __nv_bfloat16* __restrict__ s, float* __restrict__ d,
                                     long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    d[i] = __bfloat162float(s[i]);
}
__global__ void add_rows_kernel(const float* __restrict__ table, const float* __restrict__ t, int rows,
                                int rows_t, int D, float* __restrict__ out) {
  const long long n = (long long)rows * D;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / D), c = (int)(i % D);
    out[i] = table[i] + t[(long long)(r % rows_t) * D + c];
  }
}

// LN fold, per timestep: from the modulation rows of every block build (a) the fp32 column scales g = 1 + scale the
// producer epilogues multiply into the next operand and (b) the two-term bf16 rows [g_hi; g_lo; t_hi; t_lo] whose products
// with W give u = W g and W t.   mods f32 [6 L, D] rows (shift_a, scale_a, gate_a, shift_m, scale_m, gate_m) per block;
// g_out f32 [L, 2, D]; rows_out bf16 [L, 2, 4, D]  (index 1: 0 = self-attention LN, 1 = FFN LN).
__global__ void fold_prepare_kernel(const float* __restrict__ mods, int L, int D, float* __restrict__ g_out,
                                    __nv_bfloat16* __restrict__ rows_out) {
  const long long n = (long long)L * 2 * D;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % D);
    const int which = (int)((i / D) % 2);
    const int l = (int)(i / (2LL * D));
    const float shift = mods[((long long)l * 6 + which * 3 + 0) * D + k];
    const float g = 1.0f + mods[((long long)l * 6 + which * 3 + 1) * D + k];
    g_out[i] = g;
    __nv_bfloat16* r = rows_out + ((long long)l * 2 + which) * 4 * D + k;
    const __nv_bfloat16 gh = __float2bfloat16_rn(g), th = __float2bfloat16_rn(shift);
    r[0] = gh;
    r[D] = __float2bfloat16_rn(g - __bfloat162float(gh));
    r[2 * D] = th;
    r[3 * D] = __float2bfloat16_rn(shift - __bfloat162float(th));
  }
}
// u[n] = o4[0,n] + o4[1,n];  c[n] = o4[2,n] + o4[3,n] + bias[n]   (o4 = the [4, N] products of the rows above with W)
__global__ void fold_combine_kernel(const float* __restrict__ o4, int N, const float* __restrict__ bias,
                                    float* __restrict__ u, float* __restrict__ c) {
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) {
    u[n] = o4[n] + o4[N + n];
    c[n] = o4[2LL * N + n] + o4[3LL * N + n] + (bias ? bias[n] : 0.f);
  }
}

inline int grid_for(long long n, int block) {
  long long g = (n + block - 1) / block;
  const long long cap = 16LL * sm_count();   // grid-stride loops: 16 blocks per SM
  if (cap > 0 && g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace ew
}  // namespace svi

using namespace svi;
using namespace svi::ew;

extern "C" int svi_layernorm_modulate(const float* x, int32_t M, int32_t D, float eps, const float* gamma,
                                      const float* beta, const float* scale, const float* shift,
                                      void* y_bf16, void* stream) {
  SVI_REQUIRE(x && y_bf16, "svi_layernorm_modulate: null pointer");
  SVI_REQUIRE(M > 0 && D > 0 && D % 8 == 0 && D <= 4 * LN_THREADS * LN_MAX_VEC,
              "svi_layernorm_modulate: need M>0, D %% 8 == 0, D <= 8192 (M=%d D=%d)", M, D);
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y_bf16) & 7) == 0,
              "svi_layernorm_modulate: alignment");
  const int wgrid = (M + LNW_WARPS - 1) / LNW_WARPS;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  __nv_bfloat16* yb = reinterpret_cast<__nv_bfloat16*>(y_bf16);
  if (D == 1536)        // Wan 1.3B
    layernorm_modulate_warp_kernel<12><<<wgrid, LNW_WARPS * 32, 0, st>>>(x, M, D, eps, gamma, beta, scale, shift, yb);
  else if (D == 1280)   // CLIP ViT-H
    layernorm_modulate_warp_kernel<10><<<wgrid, LNW_WARPS * 32, 0, st>>>(x, M, D, eps, gamma, beta, scale, shift, yb);
  else if (D <= 128 * LNW_MAX_VEC)
    layernorm_modulate_warp_kernel<0><<<wgrid, LNW_WARPS * 32, 0, st>>>(x, M, D, eps, gamma, beta, scale, shift, yb);
  else
    layernorm_modulate_kernel<<<M, LN_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        x, D, eps, gamma, beta, scale, shift, reinterpret_cast<__nv_bfloat16*>(y_bf16), D, nullptr);
  SVI_CUDA_LAUNCH_CHECK("svi_layernorm_modulate");
  return SVI_OK;
}

extern "C" int svi_layernorm_modulate_split(const float* x, int32_t M, int32_t D, float eps, const float* gamma,
                                            const float* beta, const float* scale, const float* shift,
                                            void* y_bf16, int64_t ldy, int32_t lo_col, void* stream) {
  SVI_REQUIRE(x && y_bf16, "svi_layernorm_modulate_split: null pointer");
  SVI_REQUIRE(M > 0 && D > 0 && D % 8 == 0 && D <= 4 * LN_THREADS * LN_MAX_VEC,
              "svi_layernorm_modulate_split: need M>0, D %% 8 == 0, D <= 8192 (M=%d D=%d)", M, D);
  SVI_REQUIRE(lo_col >= D && lo_col % 4 == 0 && ldy >= (int64_t)lo_col + D && ldy % 4 == 0,
              "svi_layernorm_modulate_split: need lo_col >= D, ldy >= lo_col + D, both multiples of 4");
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y_bf16) & 7) == 0,
              "svi_layernorm_modulate_split: alignment");
  __nv_bfloat16* yb = reinterpret_cast<__nv_bfloat16*>(y_bf16);
  layernorm_modulate_kernel<<<M, LN_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(x, D, eps, gamma, beta, scale, shift,
                                                                                    yb, ldy, yb + lo_col);
  SVI_CUDA_LAUNCH_CHECK("svi_layernorm_modulate_split");
  return SVI_OK;
}

extern "C" int svi_rmsnorm_rope(void* t_bf16, int64_t ldt, int32_t M, int32_t D, const float* sumsq,
                                int32_t sumsq_ld, int32_t sumsq_col, int32_t sumsq_parts, float eps, const float* w,
                                const float* rope_cos, const float* rope_sin, int32_t row_offset,
                                void* stream) {
  SVI_REQUIRE(t_bf16 && sumsq && w, "svi_rmsnorm_rope: null pointer");
  SVI_REQUIRE(M > 0 && D > 0 && D % 8 == 0 && ldt >= D && ldt % 8 == 0,
              "svi_rmsnorm_rope: need D %% 8 == 0, ldt %% 8 == 0, ldt >= D");
  SVI_REQUIRE((rope_cos == nullptr) == (rope_sin == nullptr), "svi_rmsnorm_rope: cos/sin must both be given");
  if (rope_cos) SVI_REQUIRE(D % 128 == 0, "svi_rmsnorm_rope: RoPE needs D %% 128 == 0 (head_dim 128)");
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(t_bf16) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0,
              "svi_rmsnorm_rope: alignment");
  const long long total = (long long)M * (D / 8);
  rmsnorm_rope_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<__nv_bfloat16*>(t_bf16), ldt, M, D, 1, sumsq, sumsq_ld, sumsq_col, sumsq_parts > 0 ? sumsq_parts : 1, eps, w, w, rope_cos,
      rope_sin, row_offset);
  SVI_CUDA_LAUNCH_CHECK("svi_rmsnorm_rope");
  return SVI_OK;
}

extern "C" int svi_qk_norm_rope(void* qk_bf16, int64_t ld, int32_t M, int32_t D, const float* sumsq, int32_t sumsq_ld,
                                int32_t sumsq_parts,
                                float eps, const float* wq, const float* wk, const float* rope_cos,
                                const float* rope_sin, int32_t row_offset, void* stream) {
  SVI_REQUIRE(qk_bf16 && sumsq && wq && wk && rope_cos && rope_sin, "svi_qk_norm_rope: null pointer");
  SVI_REQUIRE(M > 0 && D > 0 && D % 128 == 0 && ld >= 2 * (int64_t)D && ld % 8 == 0 && sumsq_ld >= 2,
              "svi_qk_norm_rope: need D %% 128 == 0, ld %% 8 == 0, ld >= 2 D, sumsq_ld >= 2");
  SVI_REQUIRE(((reinterpret_cast<uintptr_t>(qk_bf16) | reinterpret_cast<uintptr_t>(wq) | reinterpret_cast<uintptr_t>(wk)) & 15) == 0,
              "svi_qk_norm_rope: alignment");
  const long long total = (long long)M * (D / 4);
  rmsnorm_rope_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<__nv_bfloat16*>(qk_bf16), ld, M, D, 2, sumsq, sumsq_ld, 0, sumsq_parts > 0 ? sumsq_parts : 1, eps, wq, wk, rope_cos, rope_sin,
      row_offset);
  SVI_CUDA_LAUNCH_CHECK("svi_qk_norm_rope");
  return SVI_OK;
}

extern "C" int svi_patchify_gather(const float* x, int32_t C0, const float* y, int32_t C1, int32_t F,
                                   int32_t H, int32_t W, void* tokens_bf16, int32_t Kpad, void* stream) {
  SVI_REQUIRE(x && tokens_bf16, "svi_patchify_gather: null pointer");
  SVI_REQUIRE(C0 > 0 && C1 >= 0 && (C1 == 0 || y), "svi_patchify_gather: bad channel split");
  SVI_REQUIRE(F > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, "svi_patchify_gather: H, W must be even");
  SVI_REQUIRE(Kpad % 8 == 0 && Kpad >= 4 * (C0 + C1), "svi_patchify_gather: Kpad must be a multiple of 8 >= 4*C");
  const long long total = (long long)F * (H / 2) * (W / 2) * (Kpad / 4);
  patchify_gather_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, C0, y, C1, F, H, W, reinterpret_cast<__nv_bfloat16*>(tokens_bf16), Kpad, 0);
  SVI_CUDA_LAUNCH_CHECK("svi_patchify_gather");
  return SVI_OK;
}

extern "C" int svi_patchify_gather_split(const float* x, int32_t C0, const float* y, int32_t C1, int32_t F, int32_t H,
                                         int32_t W, void* tokens_bf16, int32_t Kpad, void* stream) {
  SVI_REQUIRE(x && tokens_bf16, "svi_patchify_gather_split: null pointer");
  SVI_REQUIRE(C0 > 0 && C1 >= 0 && (C1 == 0 || y), "svi_patchify_gather_split: bad channel split");
  SVI_REQUIRE(F > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, "svi_patchify_gather_split: H, W must be even");
  SVI_REQUIRE(Kpad % 8 == 0 && Kpad >= 4 * (C0 + C1), "svi_patchify_gather_split: Kpad must be a multiple of 8 >= 4*C");
  const long long total = (long long)F * (H / 2) * (W / 2) * (Kpad / 4);
  patchify_gather_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, C0, y, C1, F, H, W, reinterpret_cast<__nv_bfloat16*>(tokens_bf16), Kpad, 1);
  SVI_CUDA_LAUNCH_CHECK("svi_patchify_gather_split");
  return SVI_OK;
}

extern "C" int svi_unpatchify(const float* head_out, int64_t ldh, int32_t C, int32_t F, int32_t H,
                              int32_t W, float* out, void* stream) {
  SVI_REQUIRE(head_out && out, "svi_unpatchify: null pointer");
  SVI_REQUIRE(C > 0 && F > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && ldh >= 4 * C,
              "svi_unpatchify: bad shape");
  const long long total = (long long)C * F * H * W;
  unpatchify_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(head_out, ldh, C, F,
                                                                                         H, W, out);
  SVI_CUDA_LAUNCH_CHECK("svi_unpatchify");
  return SVI_OK;
}

extern "C" int svi_cfg_euler_step(float* latents, const float* v_cond, const float* v_uncond, int64_t n,
                                  float cfg, float sigma, float sigma_next, void* stream) {
  SVI_REQUIRE(latents && v_cond && n > 0, "svi_cfg_euler_step: null pointer / empty");
  cfg_euler_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      latents, v_cond, v_uncond, n, cfg, sigma_next - sigma);
  SVI_CUDA_LAUNCH_CHECK("svi_cfg_euler_step");
  return SVI_OK;
}

extern "C" int svi_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream) {
  SVI_REQUIRE(src && dst && n > 0, "svi_cast_f32_to_bf16: null pointer / empty");
  cast_f32_bf16_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, reinterpret_cast<__nv_bfloat16*>(dst), n, SVI_ACT_NONE);
  SVI_CUDA_LAUNCH_CHECK("svi_cast_f32_to_bf16");
  return SVI_OK;
}
extern "C" int svi_act_f32_to_bf16(const float* src, void* dst, int64_t n, int32_t act, void* stream) {
  SVI_REQUIRE(src && dst && n > 0, "svi_act_f32_to_bf16: null pointer / empty");
  SVI_REQUIRE(act >= 0 && act <= 3, "svi_act_f32_to_bf16: unknown activation %d", act);
  cast_f32_bf16_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, reinterpret_cast<__nv_bfloat16*>(dst), n, act);
  SVI_CUDA_LAUNCH_CHECK("svi_act_f32_to_bf16");
  return SVI_OK;
}
extern "C" int svi_split_f32_to_bf16x2(const float* src, int64_t lds, int32_t M, int32_t K, int32_t act, void* dst_bf16,
                                       int64_t ldd, int32_t lo_col, void* stream) {
  SVI_REQUIRE(src && dst_bf16 && M > 0 && K > 0, "svi_split_f32_to_bf16x2: null pointer / empty");
  SVI_REQUIRE(act >= 0 && act <= 3, "svi_split_f32_to_bf16x2: unknown activation %d", act);
  SVI_REQUIRE(lds >= K && lo_col >= K && ldd >= (int64_t)lo_col + K, "svi_split_f32_to_bf16x2: need lds >= K, lo_col >= K, ldd >= lo_col + K");
  split_f32_bf16x2_kernel<<<grid_for((long long)M * K, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, lds, M, K, act, reinterpret_cast<__nv_bfloat16*>(dst_bf16), ldd, lo_col);
  SVI_CUDA_LAUNCH_CHECK("svi_split_f32_to_bf16x2");
  return SVI_OK;
}
extern "C" int svi_ln_fold_prepare(const float* mods, int32_t layers, int32_t D, float* g_out, void* rows_bf16, void* stream) {
  SVI_REQUIRE(mods && g_out && rows_bf16 && layers > 0 && D > 0, "svi_ln_fold_prepare: bad arguments");
  fold_prepare_kernel<<<grid_for((long long)layers * 2 * D, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      mods, layers, D, g_out, reinterpret_cast<__nv_bfloat16*>(rows_bf16));
  SVI_CUDA_LAUNCH_CHECK("svi_ln_fold_prepare");
  return SVI_OK;
}
extern "C" int svi_ln_fold_combine(const float* o4, int32_t N, const float* bias, float* u, float* c, void* stream) {
  SVI_REQUIRE(o4 && u && c && N > 0, "svi_ln_fold_combine: bad arguments");
  fold_combine_kernel<<<grid_for(N, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(o4, N, bias, u, c);
  SVI_CUDA_LAUNCH_CHECK("svi_ln_fold_combine");
  return SVI_OK;
}
extern "C" int svi_zero(void* ptr, size_t bytes, void* stream) {
  SVI_REQUIRE(ptr && bytes > 0, "svi_zero: null pointer / empty");
  cudaError_t e = cudaMemsetAsync(ptr, 0, bytes, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) {
    set_last_error("svi_zero: cudaMemsetAsync failed: %s", cudaGetErrorString(e));
    return SVI_ERR_LAUNCH;
  }
  return SVI_OK;
}
extern "C" int svi_cast_bf16_to_f32(const void* src, float* dst, int64_t n, void* stream) {
  SVI_REQUIRE(src && dst && n > 0, "svi_cast_bf16_to_f32: null pointer / empty");
  cast_bf16_f32_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(src), dst, n);
  SVI_CUDA_LAUNCH_CHECK("svi_cast_bf16_to_f32");
  return SVI_OK;
}
extern "C" int svi_axpby(const float* a, float alpha, const float* b, float beta, float* out, int64_t n, void* stream) {
  SVI_REQUIRE(a && b && out && n > 0 && n % 4 == 0, "svi_axpby: null pointer or n not a multiple of 4");
  SVI_REQUIRE(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
              "svi_axpby: pointers must be 16-byte aligned");
  axpby_kernel<<<grid_for(n / 4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(a), alpha, reinterpret_cast<const float4*>(b), beta, reinterpret_cast<float4*>(out), n / 4);
  SVI_CUDA_LAUNCH_CHECK("svi_axpby");
  return SVI_OK;
}

extern "C" int svi_add_rows(const float* table, const float* t, int32_t rows, int32_t rows_t, int32_t D,
                            float* out, void* stream) {
  SVI_REQUIRE(table && t && out, "svi_add_rows: null pointer");
  SVI_REQUIRE(rows > 0 && D > 0 && rows_t > 0 && rows % rows_t == 0, "svi_add_rows: rows must be a multiple of rows_t");
  add_rows_kernel<<<grid_for((long long)rows * D, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      table, t, rows, rows_t, D, out);
  SVI_CUDA_LAUNCH_CHECK("svi_add_rows");
  return SVI_OK;
}
