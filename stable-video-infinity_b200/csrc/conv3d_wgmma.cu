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
//
// The same mainloop, instantiated with RifeParams, runs the 2-D convolutions of RIFE's IFNet (svi_rife_conv2d,
// include/svi_b200_rife.h): "frames" are the N images of a batch (no slot table, no cap on N), and the epilogue is
// bias -> PReLU -> + residual with the output columns split into sub-pixel phases and an optional space-to-depth bf16 copy.
//
// A third instantiation, with EsrganParams, runs ESRGAN's RRDBNet (svi_esrgan_conv2d, include/svi_b200_esrgan.h): the
// input map reads a channel prefix [0, C_in) of a wider pixel (pitch in_ld), and the epilogue is bias -> LeakyReLU -> up to
// two scaled residuals, with f32, bf16 (channel offset, optional nearest x2) and uint8 RGB outputs.
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/svi_b200.h"
#include "../../include/svi_b200_esrgan.h"
#include "../../include/svi_b200_rife.h"

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

// svi_rife_conv2d: the mainloop fields of Params, then the epilogue of svi_rife_conv_desc.  T = images, kt = 1.
struct RifeParams {
  int H, W, T;
  int kt, kh, kw;
  int pad_h, pad_w;
  int cin_chunks;
  int C_out, BW, BH;
  int stages, stage_bytes;
  int phase_cols, up;          // up = 2: four phases, destination grid 2H x 2W
  const float* bias;
  const float* prelu;
  const float* residual;
  float* out;
  long long out_img_stride;
  int out_ld;
  __nv_bfloat16* out_bf;
  long long bf_img_stride;
  int bf_ld, bf_s2d;
};

// svi_esrgan_conv2d: the mainloop fields of Params, then the epilogue of svi_esrgan_conv_desc.  T = images, kt = 1.
struct EsrganParams {
  int H, W, T;
  int kt, kh, kw;
  int pad_h, pad_w;
  int cin_chunks;
  int C_out, BW, BH;
  int stages, stage_bytes;
  const float* bias;
  float slope;                 // 0: no activation
  const float* residual;
  float res_scale;
  const float* residual2;
  float res2_scale;
  float* out;                  // f32 [T][H][W][f_ld]; residual and residual2 share the layout
  int f_ld;
  __nv_bfloat16* out_bf;       // bf16 [T][up H][up W][bf_ld]
  int bf_ld, bf_up2;
  uint8_t* out_u8;             // uint8 [T][H][W][3]
};

__device__ __forceinline__ int input_slot(const Params& p, int t, int a) { return p.slot[t][a]; }
__device__ __forceinline__ int input_slot(const RifeParams&, int t, int) { return t; }
__device__ __forceinline__ int input_slot(const EsrganParams&, int t, int) { return t; }

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

// RIFE epilogue of the same slice: v = acc + bias -> PReLU -> + residual; column n = q * phase_cols + c goes to channel c
// of destination pixel (up * y + q / 2, up * x + q % 2).  phase_cols is even, so the pair (n, n + 1) stays in one phase.
template <int BN>
__device__ __forceinline__ void epilogue(const RifeParams& p, float (&acc)[BN / 2], int t, int h0, int w0, int r0, int col0,
                                         int lane) {
  const int g = lane >> 2, c = lane & 3;
  const int Wd = p.W * p.up;
  int yy[2], xx[2];
  bool ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + g + 8 * h;
    yy[h] = h0 + r / p.BW;
    xx[h] = w0 + r % p.BW;
    ok[h] = yy[h] < p.H && xx[h] < p.W;
  }
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = col0 + 8 * j + 2 * c;
    if (n < p.C_out) {
      const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
      const float2 a = p.prelu ? __ldg(reinterpret_cast<const float2*>(p.prelu + n)) : make_float2(1.f, 1.f);
      const int q = n / p.phase_cols, ch = n - q * p.phase_cols;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!ok[h]) continue;
        const int Y = yy[h] * p.up + (q >> 1), X = xx[h] * p.up + (q & 1);
        float v0 = acc[4 * j + 2 * h] + b.x, v1 = acc[4 * j + 2 * h + 1] + b.y;
        v0 = v0 > 0.f ? v0 : v0 * a.x;
        v1 = v1 > 0.f ? v1 : v1 * a.y;
        const long long o = (long long)t * p.out_img_stride + ((long long)Y * Wd + X) * p.out_ld + ch;
        if (p.residual) {
          const float2 r = *reinterpret_cast<const float2*>(p.residual + o);
          v0 += r.x; v1 += r.y;
        }
        if (p.out) *reinterpret_cast<float2*>(p.out + o) = make_float2(v0, v1);
        if (p.out_bf) {
          const long long ob = p.bf_s2d
              ? (long long)t * p.bf_img_stride + ((long long)(Y >> 1) * (Wd >> 1) + (X >> 1)) * p.bf_ld +
                    ((Y & 1) * 2 + (X & 1)) * p.phase_cols + ch
              : (long long)t * p.bf_img_stride + ((long long)Y * Wd + X) * p.bf_ld + ch;
          *reinterpret_cast<uint32_t*>(p.out_bf + ob) = pack_bf16x2(v0, v1);
        }
      }
    }
  }
}

// ESRGAN epilogue of the same slice, in the reference's op order with every step rounded on its own (__fmul_rn /
// __fadd_rn keep ptxas from contracting the residual steps into FMAs).  The pair (n, n + 1) is one 4-byte bf16 store.
template <int BN>
__device__ __forceinline__ void epilogue(const EsrganParams& p, float (&acc)[BN / 2], int t, int h0, int w0, int r0,
                                         int col0, int lane) {
  const int g = lane >> 2, c = lane & 3;
  const int up = p.bf_up2 ? 2 : 1;
  const int Wd = p.W * up;
  int yy[2], xx[2];
  bool ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + g + 8 * h;
    yy[h] = h0 + r / p.BW;
    xx[h] = w0 + r % p.BW;
    ok[h] = yy[h] < p.H && xx[h] < p.W;
  }
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = col0 + 8 * j + 2 * c;
    if (n < p.C_out) {
      const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!ok[h]) continue;
        const long long pix = ((long long)t * p.H + yy[h]) * p.W + xx[h];
        const long long o = pix * p.f_ld + n;
        float v0 = __fadd_rn(acc[4 * j + 2 * h], b.x), v1 = __fadd_rn(acc[4 * j + 2 * h + 1], b.y);
        if (p.slope != 0.f) {
          v0 = v0 > 0.f ? v0 : __fmul_rn(v0, p.slope);
          v1 = v1 > 0.f ? v1 : __fmul_rn(v1, p.slope);
        }
        if (p.residual) {
          const float2 r = *reinterpret_cast<const float2*>(p.residual + o);
          v0 = __fadd_rn(__fmul_rn(v0, p.res_scale), r.x);
          v1 = __fadd_rn(__fmul_rn(v1, p.res_scale), r.y);
        }
        if (p.residual2) {
          const float2 r = *reinterpret_cast<const float2*>(p.residual2 + o);
          v0 = __fadd_rn(__fmul_rn(v0, p.res2_scale), r.x);
          v1 = __fadd_rn(__fmul_rn(v1, p.res2_scale), r.y);
        }
        if (p.out) *reinterpret_cast<float2*>(p.out + o) = make_float2(v0, v1);
        if (p.out_bf) {
          const uint32_t pk = pack_bf16x2(v0, v1);
          const long long img = (long long)t * p.H * up;
          for (int dy = 0; dy < up; ++dy)
            for (int dx = 0; dx < up; ++dx)
              *reinterpret_cast<uint32_t*>(
                  p.out_bf + ((img + yy[h] * up + dy) * Wd + xx[h] * up + dx) * p.bf_ld + n) = pk;
        }
        if (p.out_u8) {
          uint8_t* q = p.out_u8 + pix * 3;
          if (n < 3) q[n] = (uint8_t)fminf(fmaxf(__fmul_rn(v0, 255.f), 0.f), 255.f);
          if (n + 1 < 3) q[n + 1] = (uint8_t)fminf(fmaxf(__fmul_rn(v1, 255.f), 0.f), 255.f);
        }
      }
    }
  }
}

template <int BN, class P>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
            const __grid_constant__ P p) {
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
          const int slot = input_slot(p, t, a);
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

template <int BN, class P>
int launch(const CUtensorMap& tx, const CUtensorMap& tw, P p, int tiles, cudaStream_t stream, const char* name) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t ce = cudaFuncSetAttribute(conv_kernel<BN, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (ce != cudaSuccess) {
      set_last_error("%s: cudaFuncSetAttribute failed: %s", name, cudaGetErrorString(ce));
      return SVI_ERR_LAUNCH;
    }
    attr_set = true;
  }
  p.stage_bytes = (A_STAGE_BYTES + BN * BK * 2 + 1023) / 1024 * 1024;
  p.stages = RING_BYTES / p.stage_bytes;
  if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
  const int sms = sm_count();
  if (sms <= 0) return SVI_ERR_DRIVER;
  conv_kernel<BN, P><<<tiles < sms ? tiles : sms, NUM_THREADS, SMEM_BYTES, stream>>>(tx, tw, p);
  SVI_CUDA_LAUNCH_CHECK(name);
  return SVI_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 4-D tensor map of channels [0, C) of a channels-last bf16 stack [images][H][W][ld] with 64-channel x BW x BH x 1 boxes
// (OOB = zero: channels C .. ceil64(C) read as zero even where the pixel holds more channels).
int encode_input_map(CUtensorMap* tx, const void* base, int C, int ld, int W, int H, int images, int BW, int BH,
                     const char* name) {
  EncodeTiledFn enc = reinterpret_cast<EncodeTiledFn>(encode_tiled_fn());
  if (!enc) return SVI_ERR_DRIVER;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)images};
  cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)W * ld * 2, (cuuint64_t)H * W * ld * 2};
  cuuint32_t box[4] = {BK, (cuuint32_t)BW, (cuuint32_t)BH, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(tx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("%s: input tensor map failed (CUresult %d) C=%d W=%d H=%d images=%d", name, (int)r, C, W, H, images);
    return SVI_ERR_DRIVER;
  }
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
  // The epilogue moves channel pairs (n, n + 1), n even: float2 loads of bias / residual / next_gamma, float2 stores to out
  // and bf16x2 stores to next_ring.  Every offset added to n must therefore be even and every base aligned to the pair.
  const bool writes_out = !d->next_ring || d->write_f32;
  SVI_REQUIRE(d->n_split % 2 == 0, "svi_conv3d_causal: n_split must be even (got %d)", d->n_split);
  if (writes_out) {
    SVI_REQUIRE((reinterpret_cast<uintptr_t>(d->out) & 7) == 0, "svi_conv3d_causal: out must be 8-byte aligned");
    SVI_REQUIRE(d->out_frame_stride % 2 == 0, "svi_conv3d_causal: out_frame_stride must be even (got %lld)",
                (long long)d->out_frame_stride);
    if (d->n_split > 0) {
      SVI_REQUIRE(d->split_offset % 2 == 0, "svi_conv3d_causal: split_offset must be even (got %lld)",
                  (long long)d->split_offset);
      SVI_REQUIRE(d->out_ld >= d->n_split && d->out_ld >= d->C_out - d->n_split,
                  "svi_conv3d_causal: out_ld must be >= max(n_split, C_out - n_split) (got out_ld %d)", d->out_ld);
    } else {
      SVI_REQUIRE(d->out_ld >= d->C_out, "svi_conv3d_causal: out_ld must be >= C_out (got out_ld %d, C_out %d)", d->out_ld,
                  d->C_out);
    }
  }
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(d->bias) & 7) == 0, "svi_conv3d_causal: bias must be 8-byte aligned");
  if (d->residual) {
    SVI_REQUIRE((reinterpret_cast<uintptr_t>(d->residual) & 7) == 0, "svi_conv3d_causal: residual must be 8-byte aligned");
    SVI_REQUIRE(d->res_ld >= d->C_out && d->res_ld % 2 == 0, "svi_conv3d_causal: res_ld must be even and >= C_out (got %d)",
                d->res_ld);
    SVI_REQUIRE(d->res_frame_stride % 2 == 0, "svi_conv3d_causal: res_frame_stride must be even (got %lld)",
                (long long)d->res_frame_stride);
  }
  if (d->next_ring) {
    SVI_REQUIRE((reinterpret_cast<uintptr_t>(d->next_ring) & 3) == 0, "svi_conv3d_causal: next_ring must be 4-byte aligned");
    SVI_REQUIRE(d->next_frame_stride % 2 == 0, "svi_conv3d_causal: next_frame_stride must be even (got %lld)",
                (long long)d->next_frame_stride);
    SVI_REQUIRE((reinterpret_cast<uintptr_t>(d->next_gamma) & 7) == 0, "svi_conv3d_causal: next_gamma must be 8-byte aligned");
  }
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

  const int BW = d->tile_w, BH = BM / BW;
  CUtensorMap tx, tw;
  int rc = encode_input_map(&tx, d->x_ring, d->C_in, d->C_in, d->in_W, d->in_H, d->ring_slots, BW, BH, "svi_conv3d_causal");
  if (rc) return rc;
  rc = make_tmap_2d(&tw, d->w_packed, 2, (uint64_t)ktot, (uint64_t)d->w_rows, (uint64_t)d->w_ld * 2, BK, BN);
  if (rc) return rc;

  const int tiles = d->T * ((d->H + BH - 1) / BH) * ((d->W + BW - 1) / BW) * ((d->C_out + BN - 1) / BN);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const char* nm = "svi_conv3d_causal";
  switch (BN) {
    case 16: return launch<16>(tx, tw, p, tiles, st, nm);
    case 32: return launch<32>(tx, tw, p, tiles, st, nm);
    case 64: return launch<64>(tx, tw, p, tiles, st, nm);
    case 96: return launch<96>(tx, tw, p, tiles, st, nm);
    case 128: return launch<128>(tx, tw, p, tiles, st, nm);
    case 192: return launch<192>(tx, tw, p, tiles, st, nm);
    default: return launch<256>(tx, tw, p, tiles, st, nm);
  }
}

extern "C" int svi_rife_conv2d(const svi_rife_conv_desc* d, void* stream) {
  using namespace svi;
  using namespace svi::conv;
  SVI_REQUIRE(d && d->x && d->w_packed && d->bias && (d->out || d->out_bf16), "svi_rife_conv2d: null pointer");
  SVI_REQUIRE(d->N > 0 && d->H > 0 && d->W > 0 && d->in_H > 0 && d->in_W > 0, "svi_rife_conv2d: N, H, W, in_H, in_W must be > 0");
  SVI_REQUIRE(d->kh >= 1 && d->kh <= 3 && d->kw >= 1 && d->kw <= 3, "svi_rife_conv2d: kernel extents must be in [1,3]");
  SVI_REQUIRE(d->pad_h >= 0 && d->pad_h < d->kh && d->pad_w >= 0 && d->pad_w < d->kw, "svi_rife_conv2d: need 0 <= pad < extent");
  SVI_REQUIRE(d->C_in > 0 && d->C_in % 8 == 0, "svi_rife_conv2d: C_in must be a multiple of 8 (got %d)", d->C_in);
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(d->x) & 15) == 0 && (reinterpret_cast<uintptr_t>(d->w_packed) & 15) == 0,
              "svi_rife_conv2d: x and w_packed must be 16-byte aligned");
  SVI_REQUIRE(d->phase_cols > 0 && d->phase_cols % 2 == 0 && d->C_out > 0 && d->C_out % d->phase_cols == 0 &&
                  (d->C_out / d->phase_cols == 1 || d->C_out / d->phase_cols == 4),
              "svi_rife_conv2d: phase_cols must be even and C_out must be 1 or 4 phases of it (C_out %d, phase_cols %d)",
              d->C_out, d->phase_cols);
  SVI_REQUIRE(d->tile_w == 8 || d->tile_w == 16 || d->tile_w == 32 || d->tile_w == 64 || d->tile_w == 128,
              "svi_rife_conv2d: tile_w must be 8, 16, 32, 64 or 128");
  const int cin_chunks = (d->C_in + BK - 1) / BK;
  const int ktot = d->kh * d->kw * cin_chunks * BK;
  SVI_REQUIRE(d->w_rows >= d->C_out && d->w_ld >= ktot && d->w_ld % 8 == 0,
              "svi_rife_conv2d: packed weight needs >= C_out rows and ld >= kh*kw*ceil64(C_in), ld %% 8 == 0");
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(d->bias) & 7) == 0 && (reinterpret_cast<uintptr_t>(d->prelu) & 7) == 0,
              "svi_rife_conv2d: bias and prelu must be 8-byte aligned");
  const int up = d->C_out / d->phase_cols == 4 ? 2 : 1;
  if (d->out || d->residual) {
    SVI_REQUIRE((reinterpret_cast<uintptr_t>(d->out) & 7) == 0 && (reinterpret_cast<uintptr_t>(d->residual) & 7) == 0,
                "svi_rife_conv2d: out and residual must be 8-byte aligned");
    SVI_REQUIRE(d->out_ld % 2 == 0 && d->out_ld >= d->phase_cols && d->out_img_stride % 2 == 0 &&
                    d->out_img_stride >= (long long)d->H * up * d->W * up * d->out_ld,
                "svi_rife_conv2d: out_ld must be even and >= phase_cols, out_img_stride even and >= one image");
  }
  if (d->out_bf16) {
    SVI_REQUIRE((reinterpret_cast<uintptr_t>(d->out_bf16) & 3) == 0, "svi_rife_conv2d: out_bf16 must be 4-byte aligned");
    SVI_REQUIRE(d->bf_s2d == 0 || d->bf_s2d == 1, "svi_rife_conv2d: bf_s2d must be 0 or 1");
    SVI_REQUIRE(!d->bf_s2d || ((d->H * up) % 2 == 0 && (d->W * up) % 2 == 0),
                "svi_rife_conv2d: a space-to-depth copy needs an even destination grid");
    const int need = d->bf_s2d ? 4 * d->phase_cols : d->phase_cols;
    SVI_REQUIRE(d->bf_ld % 2 == 0 && d->bf_ld >= need && d->bf_img_stride % 2 == 0 &&
                    d->bf_img_stride >= (long long)d->H * up * d->W * up / (d->bf_s2d ? 4 : 1) * d->bf_ld,
                "svi_rife_conv2d: bf_ld must be even and hold every channel of a pixel, bf_img_stride even and >= one image");
  }
  // N tiles: as few as the widest instantiated width (192) allows, then the smallest width that covers each
  const int n_tiles = (d->C_out + 191) / 192;
  const int per = (d->C_out + n_tiles - 1) / n_tiles;
  const int BN = per <= 32 ? 32 : per <= 64 ? 64 : per <= 96 ? 96 : 192;
  const int BW = d->tile_w, BH = BM / BW;
  const long long tiles = (long long)d->N * ((d->H + BH - 1) / BH) * ((d->W + BW - 1) / BW) * ((d->C_out + BN - 1) / BN);
  SVI_REQUIRE(tiles < (1LL << 31), "svi_rife_conv2d: too many tiles in one launch (%lld)", tiles);

  RifeParams p;
  p.H = d->H; p.W = d->W; p.T = d->N;
  p.kt = 1; p.kh = d->kh; p.kw = d->kw;
  p.pad_h = d->pad_h; p.pad_w = d->pad_w;
  p.cin_chunks = cin_chunks;
  p.C_out = d->C_out; p.BW = BW; p.BH = BH;
  p.stages = p.stage_bytes = 0;
  p.phase_cols = d->phase_cols; p.up = up;
  p.bias = d->bias; p.prelu = d->prelu; p.residual = d->residual;
  p.out = d->out; p.out_img_stride = d->out_img_stride; p.out_ld = d->out_ld;
  p.out_bf = reinterpret_cast<__nv_bfloat16*>(d->out_bf16); p.bf_img_stride = d->bf_img_stride;
  p.bf_ld = d->bf_ld; p.bf_s2d = d->bf_s2d;

  CUtensorMap tx, tw;
  int rc = encode_input_map(&tx, d->x, d->C_in, d->C_in, d->in_W, d->in_H, d->N, BW, BH, "svi_rife_conv2d");
  if (rc) return rc;
  rc = make_tmap_2d(&tw, d->w_packed, 2, (uint64_t)ktot, (uint64_t)d->w_rows, (uint64_t)d->w_ld * 2, BK, BN);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const char* nm = "svi_rife_conv2d";
  switch (BN) {
    case 32: return launch<32>(tx, tw, p, (int)tiles, st, nm);
    case 64: return launch<64>(tx, tw, p, (int)tiles, st, nm);
    case 96: return launch<96>(tx, tw, p, (int)tiles, st, nm);
    default: return launch<192>(tx, tw, p, (int)tiles, st, nm);
  }
}

extern "C" int svi_esrgan_conv2d(const svi_esrgan_conv_desc* d, void* stream) {
  using namespace svi;
  using namespace svi::conv;
  SVI_REQUIRE(d && d->x && d->w_packed && d->bias && (d->out || d->out_bf16 || d->out_u8), "svi_esrgan_conv2d: null pointer");
  SVI_REQUIRE(d->N > 0 && d->H > 0 && d->W > 0, "svi_esrgan_conv2d: N, H, W must be > 0");
  SVI_REQUIRE(d->C_in > 0 && d->C_in % 8 == 0 && d->in_ld % 8 == 0 && d->in_ld >= d->C_in,
              "svi_esrgan_conv2d: need C_in %% 8 == 0, in_ld %% 8 == 0 and in_ld >= C_in (got C_in %d, in_ld %d)", d->C_in,
              d->in_ld);
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(d->x) & 15) == 0 && (reinterpret_cast<uintptr_t>(d->w_packed) & 15) == 0,
              "svi_esrgan_conv2d: x and w_packed must be 16-byte aligned");
  SVI_REQUIRE(d->C_out > 0 && d->C_out % 2 == 0, "svi_esrgan_conv2d: C_out must be even and > 0 (got %d)", d->C_out);
  SVI_REQUIRE(d->tile_w == 8 || d->tile_w == 16 || d->tile_w == 32 || d->tile_w == 64 || d->tile_w == 128,
              "svi_esrgan_conv2d: tile_w must be 8, 16, 32, 64 or 128");
  const int cin_chunks = (d->C_in + BK - 1) / BK;
  const int ktot = 9 * cin_chunks * BK;
  SVI_REQUIRE(d->w_rows >= d->C_out && d->w_ld >= ktot && d->w_ld % 8 == 0,
              "svi_esrgan_conv2d: packed weight needs >= C_out rows and ld >= 9*ceil64(C_in), ld %% 8 == 0");
  SVI_REQUIRE((reinterpret_cast<uintptr_t>(d->bias) & 7) == 0, "svi_esrgan_conv2d: bias must be 8-byte aligned");
  if (d->out || d->residual || d->residual2) {
    SVI_REQUIRE(((reinterpret_cast<uintptr_t>(d->out) | reinterpret_cast<uintptr_t>(d->residual) |
                  reinterpret_cast<uintptr_t>(d->residual2)) & 7) == 0,
                "svi_esrgan_conv2d: out, residual and residual2 must be 8-byte aligned");
    SVI_REQUIRE(d->f_ld % 2 == 0 && d->f_ld >= d->C_out, "svi_esrgan_conv2d: f_ld must be even and >= C_out (got %d)", d->f_ld);
  }
  const long long in_bytes = (long long)d->N * d->H * d->W * d->in_ld * 2;
  if (d->out_bf16) {
    SVI_REQUIRE((reinterpret_cast<uintptr_t>(d->out_bf16) & 3) == 0,
                "svi_esrgan_conv2d: out_bf16 must be 4-byte aligned (an even channel offset)");
    SVI_REQUIRE(d->bf_up2 == 0 || d->bf_up2 == 1, "svi_esrgan_conv2d: bf_up2 must be 0 or 1");
    SVI_REQUIRE(d->bf_ld % 2 == 0 && d->bf_ld >= d->C_out, "svi_esrgan_conv2d: bf_ld must be even and >= C_out (got %d)",
                d->bf_ld);
    // The launch reads channels [0, C_in) of x while it writes: a destination in x's buffer must keep x's pixel layout
    // and lie past the read window, or a tile would read channels another tile is writing.
    const int up = d->bf_up2 ? 2 : 1;
    const long long out_bytes = (long long)d->N * d->H * up * d->W * up * d->bf_ld * 2;
    const char* xb = static_cast<const char*>(d->x);
    const char* ob = static_cast<const char*>(d->out_bf16);
    if (ob < xb + in_bytes && xb < ob + out_bytes) {
      SVI_REQUIRE(ob >= xb && !d->bf_up2 && d->bf_ld == d->in_ld,
                  "svi_esrgan_conv2d: a bf16 destination that overlaps x must lie in x's buffer with its pixel layout");
      const long long ch = (long long)(ob - xb) / 2 % d->in_ld;
      SVI_REQUIRE(ch >= d->C_in && ch + d->C_out <= d->in_ld,
                  "svi_esrgan_conv2d: the bf16 destination (channels %lld..%lld) lies inside the input's read window "
                  "[0, %d)", ch, ch + d->C_out, d->C_in);
    }
  }
  SVI_REQUIRE(!d->out_u8 || d->C_out >= 3, "svi_esrgan_conv2d: a uint8 RGB output needs C_out >= 3");
  const int BN = d->C_out <= 16 ? 16 : d->C_out <= 32 ? 32 : 64;
  const int BW = d->tile_w, BH = BM / BW;
  const long long tiles = (long long)d->N * ((d->H + BH - 1) / BH) * ((d->W + BW - 1) / BW) * ((d->C_out + BN - 1) / BN);
  SVI_REQUIRE(tiles < (1LL << 31), "svi_esrgan_conv2d: too many tiles in one launch (%lld)", tiles);

  EsrganParams p;
  p.H = d->H; p.W = d->W; p.T = d->N;
  p.kt = 1; p.kh = 3; p.kw = 3;
  p.pad_h = 1; p.pad_w = 1;
  p.cin_chunks = cin_chunks;
  p.C_out = d->C_out; p.BW = BW; p.BH = BH;
  p.stages = p.stage_bytes = 0;
  p.bias = d->bias; p.slope = d->slope;
  p.residual = d->residual; p.res_scale = d->res_scale;
  p.residual2 = d->residual2; p.res2_scale = d->res2_scale;
  p.out = d->out; p.f_ld = d->f_ld;
  p.out_bf = reinterpret_cast<__nv_bfloat16*>(d->out_bf16); p.bf_ld = d->bf_ld; p.bf_up2 = d->bf_up2;
  p.out_u8 = d->out_u8;

  CUtensorMap tx, tw;
  int rc = encode_input_map(&tx, d->x, d->C_in, d->in_ld, d->W, d->H, d->N, BW, BH, "svi_esrgan_conv2d");
  if (rc) return rc;
  rc = make_tmap_2d(&tw, d->w_packed, 2, (uint64_t)ktot, (uint64_t)d->w_rows, (uint64_t)d->w_ld * 2, BK, BN);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const char* nm = "svi_esrgan_conv2d";
  switch (BN) {
    case 16: return launch<16>(tx, tw, p, (int)tiles, st, nm);
    case 32: return launch<32>(tx, tw, p, (int)tiles, st, nm);
    default: return launch<64>(tx, tw, p, (int)tiles, st, nm);
  }
}
