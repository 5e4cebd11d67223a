/*
 * svi_b200_rife.h — RIFE frame interpolation (IFNet) on libsvi_b200.so (the same library as svi_b200.h).
 *
 * IFNet (diffsynth/extensions/RIFE) estimates, for a frame pair (img0, img1), a bidirectional flow and a blend mask in
 * three coarse-to-fine blocks, each run twice with shared weights (img0 -> img1 and img1 -> img0).  Four entry points
 * cover one block of a batch of pairs:
 *
 *   svi_rife_stage_frames   uint8 RGB frames -> f32 BGR in [0, 1] (the frames cross the bus once, as bytes)
 *   svi_rife_block_input    bilinear resize of the images / warped images / mask / flow, channel concat of both directions,
 *                           written in space-to-depth form as the first convolution's bf16 operand
 *   svi_rife_conv2d         a batch of 2-D convolutions on the implicit-GEMM wgmma conv mainloop of svi_conv3d_causal,
 *                           epilogue  v = acc + bias -> PReLU -> + residual,  f32 and / or bf16 out, sub-pixel phases
 *   svi_rife_update_warp    x s upsample of the heads' flow / mask, the averaged update, the two border warps, and (any
 *                           block) the sigmoid blend in f32, clipped if asked, and its uint8 RGB frame
 *
 * Layouts are channels-last.  Per-pair state (svi_rife_update.state): f32 [pairs][H][W][12] =
 *   warped img0 (B, G, R), warped img1 (B, G, R), mask, 0, flow img0 (x, y), flow img1 (x, y).
 * Frames: f32 [H][W][4] per frame = B, G, R, and a fourth channel no reader uses.
 * Conventions as in svi_b200.h: 0 on success, a negative status (and svi_last_error) on a rejected argument, in which
 * case nothing is launched; every launch is on `stream`, without atomics: the same input gives the same bytes.
 * A separate header so that svi_b200.h and its ABI version stay as they are.
 */
#ifndef SVI_B200_RIFE_H_
#define SVI_B200_RIFE_H_

#include <stdint.h>

#include "svi_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One svi_rife_conv2d launch: N images, output grid H x W per image, stride 1, input coordinate = output + tap - pad.
 * GEMM column n = q * phase_cols + c is output channel c of phase q.  One phase: a plain convolution.  Four phases: a
 * ConvTranspose2d(4, stride 2, padding 1) run as a 3x3 sub-pixel convolution; phase q = 2 dy + dx is written to output
 * pixel (2 y + dy, 2 x + dx), so the destination grid is 2H x 2W. */
typedef struct svi_rife_conv_desc {
  const void* x;            /* bf16 [N][in_H][in_W][C_in], 16-byte aligned */
  int32_t N, in_H, in_W, C_in;   /* C_in % 8 == 0 (the channel pitch; channels past it read as zero) */
  const void* w_packed;     /* bf16 [w_rows][w_ld]: row n = column n, (kh, kw, C_in padded to 64) taps; 16-byte aligned */
  int32_t w_rows;
  int64_t w_ld;
  int32_t kh, kw, pad_h, pad_w;  /* extents in [1, 3] */
  int32_t H, W;             /* output grid per image */
  int32_t C_out;            /* GEMM columns: phases * phase_cols */
  int32_t phase_cols;       /* even; C_out / phase_cols is 1 or 4 */
  int32_t tile_w;           /* pixels per tile row: 8, 16, 32, 64 or 128 (tile = 128 pixels) */
  const float* bias;        /* [C_out], 8-byte aligned */
  const float* prelu;       /* [C_out] PReLU slopes, or null (no activation) */
  const float* residual;    /* f32 in the layout of out, added after PReLU, or null; may equal out */
  float* out;               /* f32 [N] x out_img_stride: pixel (Y, X) of the destination grid at (Y * Wd + X) * out_ld, or null */
  int64_t out_img_stride;   /* even */
  int32_t out_ld;           /* even, >= phase_cols */
  void* out_bf16;           /* bf16 copy of the result, or null: [N] x bf_img_stride, */
  int64_t bf_img_stride;    /*   bf_s2d == 0: pixel (Y, X) at (Y * Wd + X) * bf_ld, channel c */
  int32_t bf_ld;            /*   bf_s2d == 1: space-to-depth, pixel (Y/2, X/2) at ((Y/2) * Wd/2 + X/2) * bf_ld, */
  int32_t bf_s2d;           /*   channel ((Y % 2) * 2 + X % 2) * phase_cols + c (the next stride-2 conv's operand) */
} svi_rife_conv_desc;

/* The first convolution's operand of one block, both directions of `pairs` pairs:
 * out bf16 [2 pairs][h/2][w/2][48], image p = direction 0 of pair p, image pairs + p = direction 1, channel
 * (dy * 2 + dx) * 11 + k of block-resolution pixel (2 y + dy, 2 x + dx), channels 44..47 zero; k:
 *   direction 0:  warped img0 (3), warped img1 (3),  mask, flow img0 (2), flow img1 (2)
 *   direction 1:  warped img1 (3), warped img0 (3), -mask, flow img1 (2), flow img0 (2)
 * each bilinearly resized from H x W to h x w as F.interpolate(scale_factor = 1 / s, align_corners = False,
 * recompute_scale_factor = False) does (source index src_scale * (d + 0.5) - 0.5, clamped at 0; src_scale = (float) s),
 * the flows then multiplied by flow_mul (= 1 / s).  state == null: the first block (warped = the images, mask = flow = 0). */
typedef struct svi_rife_block_input {
  const float* img0;        /* f32 frames of pair p at img0 + p * img_stride, and img1 + p * img_stride */
  const float* img1;
  int64_t img_stride;       /* floats between the pairs' frames, % 4 == 0 */
  const float* state;       /* f32 [pairs][H][W][12] or null */
  int32_t pairs, H, W, h, w;     /* h, w even */
  float src_scale, flow_mul;
  void* out;
} svi_rife_block_input;

/* The update after a block, per pixel of every pair: the heads' output of direction 0 (image p) and 1 (image pairs + p),
 * f32 [2 pairs][h][w][heads_ld] (flow 4, mask 1), upsampled to H x W as F.interpolate(scale_factor = s) with source scale
 * src_scale (= (float)(1 / s)), the flows times flow_mul (= s):
 *   flow += (f0 + swap(f1)) / 2,  mask += (m0 - m1) / 2   (swap: the two 2-channel halves exchanged)
 *   warped imgK = grid_sample(imgK, identity grid + flow K, bilinear, padding border, align_corners True)
 * state is read (unless first) and written.  merged (or null): f32 [H][W][4] per pair = B, G, R of
 * warped0 * sigmoid(mask) + warped1 * (1 - sigmoid(mask)), clipped to [0, 1] if clip, and sigmoid(mask).
 * rgb (or null): uint8 [H][W][3] per pair = R, G, B of (x * 255).clip(0, 255) truncated, x = the blend. */
typedef struct svi_rife_update {
  const float* heads;
  int32_t heads_ld;         /* % 4 == 0, >= 8 */
  int32_t pairs, H, W, h, w;
  float src_scale, flow_mul;
  const float* img0;        /* as in svi_rife_block_input */
  const float* img1;
  int64_t img_stride;
  float* state;
  int32_t first;
  float* merged;
  int64_t merged_stride;    /* floats between pairs, % 4 == 0 */
  int32_t clip;
  uint8_t* rgb;
  int64_t rgb_stride;       /* bytes between pairs */
} svi_rife_update;

/* f32 out [n][4] = B, G, R, 0 of uint8 rgb [n][3], each v / 255 (IEEE division, as numpy's float32 v / 255). */
int svi_rife_stage_frames(const uint8_t* rgb, int64_t n_pix, float* out, void* stream);
int svi_rife_block_input_launch(const svi_rife_block_input* d, void* stream);
int svi_rife_conv2d(const svi_rife_conv_desc* d, void* stream);
int svi_rife_update_warp(const svi_rife_update* d, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SVI_B200_RIFE_H_ */
