/*
 * svi_b200_esrgan.h — ESRGAN 4x upscaling (RRDBNet) on libsvi_b200.so (the same library as svi_b200.h).
 *
 * RRDBNet (diffsynth/extensions/ESRGAN) is a stack of 3x3, stride-1, padding-1 convolutions: conv_first, 23 RRDBs of
 * three residual dense blocks (five convs each, conv k reading the concatenation of the block input and the k - 1
 * outputs before it), conv_body, two nearest-x2 upsamplings each followed by a conv, conv_hr and conv_last.  Two entry
 * points run it:
 *
 *   svi_esrgan_stage_frames   uint8 RGB frames -> the bf16 operand of conv_first (the frames cross the bus once, as bytes)
 *   svi_esrgan_conv2d         a batch of 2-D convolutions on the implicit-GEMM wgmma conv mainloop of svi_conv3d_causal,
 *                             epilogue  v = acc + bias -> LeakyReLU -> scaled residual -> scaled residual, with f32, bf16
 *                             (at a channel offset, optionally nearest-x2 upsampled) and uint8 RGB outputs
 *
 * Layouts are channels-last.  The input of a convolution is read through a pitch: channels [0, C_in) of a buffer with
 * in_ld channels per pixel, so that a dense block's convolutions read growing prefixes of one buffer and write their
 * outputs just past them without copies.
 * Conventions as in svi_b200.h: 0 on success, a negative status (and svi_last_error) on a rejected argument, in which
 * case nothing is launched; every launch is on `stream`, without atomics: the same input gives the same bytes.
 * A separate header so that svi_b200.h and its ABI version stay as they are.
 */
#ifndef SVI_B200_ESRGAN_H_
#define SVI_B200_ESRGAN_H_

#include <stdint.h>

#include "svi_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One svi_esrgan_conv2d launch: N images of H x W pixels, 3x3 taps, stride 1, padding 1.  Per output element, in f32 and
 * in this order, each step rounded on its own (no fused multiply-add):
 *   v = acc + bias[n]
 *   slope != 0:     v = v > 0 ? v : v * slope
 *   residual:       v = v * res_scale + residual[pixel, n]
 *   residual2:      v = v * res2_scale + residual2[pixel, n]
 * Outputs (any non-empty subset):
 *   out       f32 [N][H][W][f_ld], channel n; may alias residual or residual2 (an element is read and written by one thread)
 *   out_bf16  bf16 [N][Hd][Wd][bf_ld], channel n, Hd x Wd = H x W, or 2H x 2W with bf_up2 (pixel (y, x) then goes to the
 *             four pixels (2y + dy, 2x + dx)); the pointer may sit at a channel offset into a wider pixel.  It may lie in
 *             the input buffer x only with x's pixel layout and outside the read window: channels [0, C_in) are read
 *             while the launch runs.
 *   out_u8    uint8 [N][H][W][3] of (v * 255).clip(0, 255), truncated, channels 0..2 (C_out >= 3). */
typedef struct svi_esrgan_conv_desc {
  const void* x;            /* bf16 [N][H][W][in_ld], 16-byte aligned; channels [0, C_in) are read, the rest of K is zero */
  int32_t N, H, W;
  int32_t C_in;             /* % 8 == 0, <= in_ld */
  int32_t in_ld;            /* % 8 == 0 */
  const void* w_packed;     /* bf16 [w_rows][w_ld]: row n = output channel n, (kh, kw, C_in padded to 64) taps; 16-byte aligned */
  int32_t w_rows;
  int64_t w_ld;
  int32_t C_out;            /* even */
  int32_t tile_w;           /* pixels per tile row: 8, 16, 32, 64 or 128 (tile = 128 pixels) */
  const float* bias;        /* [C_out], 8-byte aligned */
  float slope;              /* LeakyReLU negative slope; 0: no activation */
  const float* residual;    /* f32 in the layout of out, or null */
  float res_scale;
  const float* residual2;   /* f32 in the layout of out, or null */
  float res2_scale;
  float* out;               /* f32 [N][H][W][f_ld] or null; 8-byte aligned */
  int32_t f_ld;             /* even, >= C_out (also the pitch of residual and residual2) */
  void* out_bf16;           /* bf16 or null; 4-byte aligned */
  int32_t bf_ld;            /* even, >= C_out */
  int32_t bf_up2;           /* 0 or 1 */
  uint8_t* out_u8;          /* uint8 RGB or null */
} svi_esrgan_conv_desc;

/* conv_first's operand (C_in = 8, in_ld = 8) of uint8 rgb [n][3]: out bf16 [n][8] = R, G, B, 0, 0, 0, 0, 0, each
 * bf16(c / 255) of the IEEE f32 division. */
int svi_esrgan_stage_frames(const uint8_t* rgb, int64_t n_pix, void* out, void* stream);
int svi_esrgan_conv2d(const svi_esrgan_conv_desc* d, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SVI_B200_ESRGAN_H_ */
