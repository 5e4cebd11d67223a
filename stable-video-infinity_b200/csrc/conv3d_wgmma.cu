// Causal 3-D / 2-D convolution of the Wan VAE as an implicit GEMM on wgmma (sm_90a).
//
// Activations are channels-last bf16 "frame rings"  [slots][H][W][C];  one CTA tile = 128 output pixels (a BH x BW patch of
// one frame, accumulator row = pixel) x BN output channels.  The K loop walks (k_t, k_h, k_w, 64-channel chunk): for every
// step ONE 4-D TMA box {64ch, BW, BH, 1 frame} of the input ring, shifted by the tap offset, lands in shared memory as a
// canonical 128-row x 128-byte swizzled K-major operand tile — spatial zero padding comes for free from TMA out-of-bounds
// zero fill, temporal causality from the (output frame, k_t) -> ring slot table (history frames stay in the ring: no F.pad /
// torch.cat cache copies as in the reference, wan_video_vae.py:44-52, 214-232).  Weights are pre-packed
// [C_out, (k_t,k_h,k_w,C_in padded to 64)] and stream through a 2-D TMA like a GEMM B operand.
// Warp roles are those of gemm_wgmma.cu: a TMA producer warpgroup and two consumer warpgroups of 64 pixels each, persistent
// over the tiles, operand ring of 4..8 stages depending on the N tile.  Epilogue (from the accumulator registers):
// + bias, + fp32 residual (ResidualBlock skip), optional channel split into two frames (upsample3d time_conv,
// wan_video_vae.py:153-156), fp32 NHWC out — and, fused, the NEXT conv's input: RMS_norm + SiLU (:55-70, 206-210) of the
// output pixel (its whole channel vector sits in one accumulator row) written as bf16 straight into the next conv's frame
// ring, so the activation between the two convs of a ResidualBlock never exists in fp32 and no staging pass runs.
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/svi_b200.h"

namespace svi {
namespace conv {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int MAX_STAGES = 8;
constexpr int MAX_BN = 256;
constexpr int A_STAGE_BYTES = BM * BK * 2;
constexpr int RING_BYTES = 4 * (A_STAGE_BYTES + MAX_BN * BK * 2);   // 192 KB of operand stages: 4 at BN = 256 ... 8 at BN <= 64
constexpr int NUM_THREADS = 384;
constexpr int SMEM_BYTES = RING_BYTES + 1024 + 256;
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;

struct Params {
  int H, W, T;                 // output height / width / frames of this launch
  int kt, kh, kw;              // kernel extent
  int pad_h, pad_w;            // input coordinate = output coordinate + k - pad
  int slot[4][3];              // ring slot of the input frame for (output frame, k_t)
  int cin_chunks;              // ceil(C_in / 64)
  int C_out, BW, BH;           // BH * BW == 128
  float* out;                  // fp32 channels-last [frame][H][W][out_ld]
  long long out_frame_stride;  // elements between output frames
  int out_ld;                  // channels per output pixel in memory
  int n_split;                 // columns >= n_split are written to out + split_offset (column - n_split); 0 = off
  long long split_offset;
  const float* bias;           // [C_out]
  const float* residual;       // same layout as out (frame stride res_frame_stride, ld res_ld) or null
  long long res_frame_stride;
  int res_ld;
  int stages, stage_bytes;     // operand ring: stage_bytes = A tile + BN x 64 bf16 rounded to 1 KB
  // fused producer of the NEXT conv's input (RMS_norm + SiLU + bf16 staging, wan_video_vae.py:55-70,206-210):
  __nv_bfloat16* next_ring;    // bf16 [slots][H][W][next_ld] or null
  long long next_frame_stride; // elements between ring slots
  int next_ld;
  int next_slot[4];            // ring slot of output frame t
  const float* next_gamma;     // [C_out] RMS-norm weight, null: plain cast
  int next_silu;
  int write_f32;               // 0: the fp32 output is not needed (only the normalised bf16 is consumed)
};

__device__ __forceinline__ void tma_load_4d_a(uint32_t smem_dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                              int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_dst),
      "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// Epilogue of one warp's 16-pixel x BN accumulator slice: pixels (tile rows) r0 + g and r0 + g + 8, channels
// col0 + 8j + 2c (+1).  Pass 1: v = acc + bias (+ residual) -> fp32 out (if write_f32), sum of v^2 over the pixel's channels.
// Pass 2 (fused producer of the next conv's input; the launch side guarantees one N tile): RMS norm + SiLU -> bf16 ring.
template <int BN>
__device__ __forceinline__ void epilogue(const Params& p, float (&acc)[BN / 2], int t, int h0, int w0, int r0, int col0,
                                         int lane) {
  const int g = lane >> 2, c = lane & 3;
  long long pix[2];
  bool ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + g + 8 * h;
    const int hh = h0 + r / p.BW, ww = w0 + r % p.BW;
    ok[h] = hh < p.H && ww < p.W;
    pix[h] = (long long)hh * p.W + ww;
  }
  float ssq[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = col0 + 8 * j + 2 * c;
    if (n < p.C_out) {   // C_out % 4 == 0: n + 1 is a channel too
      const float2 b = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + n)) : make_float2(0.f, 0.f);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!ok[h]) continue;
        float v0 = acc[4 * j + 2 * h] + b.x, v1 = acc[4 * j + 2 * h + 1] + b.y;
        if (p.residual) {
          const float2 r = *reinterpret_cast<const float2*>(p.residual + (long long)t * p.res_frame_stride + pix[h] * p.res_ld + n);
          v0 += r.x; v1 += r.y;
        }
        ssq[h] += v0 * v0 + v1 * v1;
        if (p.write_f32) {
          float* dst;
          if (p.n_split > 0 && n >= p.n_split)
            dst = p.out + p.split_offset + (long long)t * p.out_frame_stride + pix[h] * p.out_ld + (n - p.n_split);
          else
            dst = p.out + (long long)t * p.out_frame_stride + pix[h] * p.out_ld + n;
          *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
        }
        acc[4 * j + 2 * h] = v0;
        acc[4 * j + 2 * h + 1] = v1;
      }
    }
  }
  if (!p.next_ring) return;
  float mul[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float s = ssq[h];
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    mul[h] = p.next_gamma ? sqrtf((float)p.C_out) / fmaxf(sqrtf(s), 1e-12f) : 1.f;
  }
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = col0 + 8 * j + 2 * c;
    if (n < p.C_out) {
      const float2 gm = p.next_gamma ? __ldg(reinterpret_cast<const float2*>(p.next_gamma + n)) : make_float2(1.f, 1.f);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!ok[h]) continue;
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (p.next_gamma) {
          v0 *= mul[h] * gm.x;
          v1 *= mul[h] * gm.y;
        }
        if (p.next_silu) {
          v0 = silu(v0);
          v1 = silu(v1);
        }
        __nv_bfloat16* nrow = p.next_ring + (long long)p.next_slot[t] * p.next_frame_stride + pix[h] * p.next_ld;
        *reinterpret_cast<uint32_t*>(nrow + n) = pack_bf16x2(v0, v1);
      }
    }
  }
}

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
            const __grid_constant__ Params p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bars = sbase + RING_BYTES;
  auto full_bar = [&](int s) { return bars + 8u * s; };
  auto empty_bar = [&](int s) { return bars + 8u * (MAX_STAGES + s); };
  const int STAGES = p.stages;
  const int STAGE_BYTES = p.stage_bytes;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int tiles_w = (p.W + p.BW - 1) / p.BW;
  const int tiles_h = (p.H + p.BH - 1) / p.BH;
  const int num_n = (p.C_out + BN - 1) / BN;
  const int tiles_per_frame = tiles_h * tiles_w;
  const int num_tiles = p.T * tiles_per_frame * num_n;
  const int num_k = p.kt * p.kh * p.kw * p.cin_chunks;
  const uint32_t stage_tx = A_STAGE_BYTES + BN * BK * 2;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_w);
    for (int i = 0; i < MAX_STAGES; ++i) {
      mbar_init_a(full_bar(i), 1);
      mbar_init_a(empty_bar(i), 8);   // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  // tile index -> (n block fastest, then spatial tile, then frame): CTAs running together share the input patch
  auto decode_tile = [&](int tile, int& t, int& h0, int& w0, int& n_blk) {
    n_blk = tile % num_n;
    int r = tile / num_n;
    const int sp = r % tiles_per_frame;
    t = r / tiles_per_frame;
    h0 = (sp / tiles_w) * p.BH;
    w0 = (sp % tiles_w) * p.BW;
  };

  if (wg == 0) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int t, h0, w0, n_blk;
        decode_tile(tile, t, h0, w0, n_blk);
        int kcol = 0;
        for (int a = 0; a < p.kt; ++a) {
          const int slot = p.slot[t][a];
          for (int b = 0; b < p.kh; ++b) {
            for (int c = 0; c < p.kw; ++c) {
              for (int cc = 0; cc < p.cin_chunks; ++cc) {
                mbar_wait_a(empty_bar(stage), phase ^ 1);
                mbar_expect_tx_a(full_bar(stage), stage_tx);
                const uint32_t sa = sbase + stage * STAGE_BYTES;
                tma_load_4d_a(sa, &tmap_x, full_bar(stage), cc * BK, w0 + c - p.pad_w, h0 + b - p.pad_h, slot);
                tma_load_2d_a(sa + A_STAGE_BYTES, &tmap_w, full_bar(stage), kcol, n_blk * BN);
                kcol += BK;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
              }
            }
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<CONSUMER_REGS>();
    const int cw = wg - 1;   // pixels [64 cw, 64 cw + 64) of the tile
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int t, h0, w0, n_blk;
      decode_tile(tile, t, h0, w0, n_blk);
      int prev = -1;
      for (int kb = 0; kb < num_k; ++kb) {
        mbar_wait_a(full_bar(stage), phase);
        const uint32_t sa = sbase + stage * STAGE_BYTES;
        const uint64_t da = wgmma_desc(sa + cw * 64 * 128, 16, 1024);
        const uint64_t db = wgmma_desc(sa + A_STAGE_BYTES, 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) Wgmma<BN>::ss(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();   // the previous stage's MMAs have retired: its slot goes back to the producer
        if (prev >= 0 && lane == 0) mbar_arrive_a(empty_bar(prev));
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (lane == 0) mbar_arrive_a(empty_bar(prev));
      epilogue<BN>(p, acc, t, h0, w0, cw * 64 + (warp & 3) * 16, n_blk * BN, lane);
    }
  }
}

void* encode_tiled_fn() {
  static void* fn = nullptr;
  if (!fn) {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess || !fp) {
      set_last_error("svi_conv3d_causal: cuTensorMapEncodeTiled unavailable");
      return nullptr;
    }
    fn = fp;
  }
  return fn;
}

template <int BN>
int launch(const CUtensorMap& tx, const CUtensorMap& tw, Params p, int tiles, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t ce = cudaFuncSetAttribute(conv_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (ce != cudaSuccess) {
      set_last_error("svi_conv3d_causal: cudaFuncSetAttribute failed: %s", cudaGetErrorString(ce));
      return SVI_ERR_LAUNCH;
    }
    attr_set = true;
  }
  p.stage_bytes = (A_STAGE_BYTES + BN * BK * 2 + 1023) / 1024 * 1024;
  p.stages = RING_BYTES / p.stage_bytes;
  if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
  const int sms = sm_count();
  if (sms <= 0) return SVI_ERR_DRIVER;
  conv_kernel<BN><<<tiles < sms ? tiles : sms, NUM_THREADS, SMEM_BYTES, stream>>>(tx, tw, p);
  SVI_CUDA_LAUNCH_CHECK("svi_conv3d_causal");
  return SVI_OK;
}

}  // namespace conv
}  // namespace svi

extern "C" int svi_conv3d_causal(const svi_conv_desc* d, void* stream) {
  using namespace svi;
  using namespace svi::conv;
  SVI_REQUIRE(d && d->x_ring && d->w_packed && (d->out || (d->next_ring && !d->write_f32)), "svi_conv3d_causal: null pointer");
  SVI_REQUIRE(d->H > 0 && d->W > 0 && d->T > 0 && d->T <= 4, "svi_conv3d_causal: need 1 <= T <= 4, H, W > 0");
  SVI_REQUIRE(d->kt >= 1 && d->kt <= 3 && d->kh >= 1 && d->kh <= 3 && d->kw >= 1 && d->kw <= 3,
              "svi_conv3d_causal: kernel extents must be in [1,3]");
  SVI_REQUIRE(d->C_in > 0 && d->C_in % 8 == 0, "svi_conv3d_causal: C_in must be a multiple of 8 (got %d)", d->C_in);
  SVI_REQUIRE(d->C_out > 0 && d->C_out % 4 == 0 && d->out_ld % 4 == 0, "svi_conv3d_causal: C_out, out_ld %% 4");
  SVI_REQUIRE(d->ring_slots > 0 && d->in_H > 0 && d->in_W > 0, "svi_conv3d_causal: bad ring geometry");
  SVI_REQUIRE(d->tile_w == 8 || d->tile_w == 16 || d->tile_w == 32 || d->tile_w == 64 || d->tile_w == 128,
              "svi_conv3d_causal: tile_w must be 8, 16, 32, 64 or 128");
  for (int t = 0; t < d->T; ++t)
    for (int a = 0; a < d->kt; ++a)
      SVI_REQUIRE(d->slot[t * 3 + a] >= 0 && d->slot[t * 3 + a] < d->ring_slots, "svi_conv3d_causal: slot out of range");
  const int cin_chunks = (d->C_in + BK - 1) / BK;
  const int cpad = cin_chunks * BK;
  const int ktot = d->kt * d->kh * d->kw * cpad;
  SVI_REQUIRE(d->w_ld >= ktot && d->w_ld % 8 == 0, "svi_conv3d_causal: packed weight ld must be >= kt*kh*kw*ceil64(C_in)");
  int BN = d->C_out <= MAX_BN ? ((d->C_out + 15) / 16) * 16 : 0;
  if (BN == 0) {  // split wide outputs into equal tiles that are multiples of 16
    for (int parts = 2; parts <= 8 && BN == 0; ++parts)
      if (d->C_out % parts == 0 && (d->C_out / parts) % 16 == 0 && d->C_out / parts <= MAX_BN) BN = d->C_out / parts;
    if (BN == 0) BN = MAX_BN;
  }
  // the N tiles the kernel is instantiated for (wgmma widths): the smallest that covers BN
  static const int kWidths[] = {16, 32, 64, 96, 128, 192, 256};
  for (int w : kWidths)
    if (w >= BN) { BN = w; break; }
  SVI_REQUIRE(d->w_rows >= d->C_out, "svi_conv3d_causal: packed weight has fewer rows than C_out");
  // variant: kept in the descriptor so that callers of the C ABI stay valid; every value runs the one kernel of this file
  SVI_REQUIRE(d->variant >= 0 && d->variant <= 2, "svi_conv3d_causal: variant must be 0 (auto), 1 or 2");
  SVI_REQUIRE(d->variant != 2 || (d->kw == 3 && d->pad_w == 1), "svi_conv3d_causal: variant 2 needs k_w = 3 and pad_w = 1");

  Params p;
  p.H = d->H; p.W = d->W; p.T = d->T;
  p.kt = d->kt; p.kh = d->kh; p.kw = d->kw;
  p.pad_h = d->pad_h; p.pad_w = d->pad_w;
  for (int t = 0; t < 4; ++t)
    for (int a = 0; a < 3; ++a) p.slot[t][a] = d->slot[t * 3 + a];
  p.cin_chunks = cin_chunks;
  p.C_out = d->C_out; p.BW = d->tile_w; p.BH = BM / d->tile_w;
  p.out = d->out; p.out_frame_stride = d->out_frame_stride; p.out_ld = d->out_ld;
  p.n_split = d->n_split; p.split_offset = d->split_offset;
  p.bias = d->bias; p.residual = d->residual; p.res_frame_stride = d->res_frame_stride; p.res_ld = d->res_ld;
  p.next_ring = reinterpret_cast<__nv_bfloat16*>(d->next_ring);
  p.next_frame_stride = d->next_frame_stride;
  p.next_ld = d->next_ld;
  for (int t = 0; t < 4; ++t) p.next_slot[t] = d->next_slot[t];
  p.next_gamma = d->next_gamma;
  p.next_silu = d->next_silu;
  p.write_f32 = d->next_ring ? d->write_f32 : 1;
  if (d->next_ring) {
    SVI_REQUIRE(d->C_out <= BN && d->n_split == 0, "svi_conv3d_causal: the fused next-input producer needs one N tile (C_out <= 256) and no channel split");
    SVI_REQUIRE(d->next_ld >= d->C_out && d->next_ld % 4 == 0, "svi_conv3d_causal: next_ld must be >= C_out and a multiple of 4");
    for (int t = 0; t < d->T; ++t) SVI_REQUIRE(d->next_slot[t] >= 0, "svi_conv3d_causal: next_slot must be >= 0");
  }

  typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  EncodeTiledFn enc = reinterpret_cast<EncodeTiledFn>(encode_tiled_fn());
  if (!enc) return SVI_ERR_DRIVER;
  const int BW = d->tile_w, BH = BM / BW;
  CUtensorMap tx, tw;
  {
    cuuint64_t dims[4] = {(cuuint64_t)d->C_in, (cuuint64_t)d->in_W, (cuuint64_t)d->in_H, (cuuint64_t)d->ring_slots};
    cuuint64_t strides[3] = {(cuuint64_t)d->C_in * 2, (cuuint64_t)d->in_W * d->C_in * 2,
                             (cuuint64_t)d->in_H * d->in_W * d->C_in * 2};
    cuuint32_t box[4] = {BK, (cuuint32_t)BW, (cuuint32_t)BH, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = enc(&tx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(d->x_ring), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_last_error("svi_conv3d_causal: input tensor map failed (CUresult %d) C=%d W=%d H=%d slots=%d", (int)r, d->C_in,
                     d->in_W, d->in_H, d->ring_slots);
      return SVI_ERR_DRIVER;
    }
  }
  int rc = make_tmap_2d(&tw, d->w_packed, 2, (uint64_t)ktot, (uint64_t)d->w_rows, (uint64_t)d->w_ld * 2, BK, BN);
  if (rc) return rc;

  const int tiles = d->T * ((d->H + BH - 1) / BH) * ((d->W + BW - 1) / BW) * ((d->C_out + BN - 1) / BN);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (BN) {
    case 16: return launch<16>(tx, tw, p, tiles, st);
    case 32: return launch<32>(tx, tw, p, tiles, st);
    case 64: return launch<64>(tx, tw, p, tiles, st);
    case 96: return launch<96>(tx, tw, p, tiles, st);
    case 128: return launch<128>(tx, tw, p, tiles, st);
    case 192: return launch<192>(tx, tw, p, tiles, st);
    default: return launch<256>(tx, tw, p, tiles, st);
  }
}
