/*
 * svi_b200_processors.h — the video processors of diffsynth/processors (contrast and sharpness editors, the RIFE
 * smoother's averaging mode) on libsvi_b200.so (the same library as svi_b200.h and svi_b200_rife.h).
 *
 * The editors reproduce Pillow's ImageEnhance byte for byte (Pillow 12.2: Image.blend over a degenerate image):
 *   svi_luma_sum_u8       per frame, the integer sum of L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16 (Contrast's
 *                         degenerate grey is int(sum / n_pix + 0.5), divided on the host in double as ImageStat does)
 *   svi_enhance_blend_u8  out = blend(degenerate, x, rate) with one degenerate value per frame (Contrast)
 *   svi_sharpen_u8        out = blend(SMOOTH(x), x, rate), the 3x3 smoothing fused into the blend (Sharpness)
 *   svi_rife_average_u8   the inner frames of RIFESmoother(interpolate=False): (frame + interpolation) / 2 as uint8 RGB
 *
 * blend(d, x, rate), per byte, as Pillow's ImagingBlend with a float alpha:  t = (float) d + rate * (float)(x - d), each
 * operation rounded on its own (no FMA);  0 <= rate <= 1: (uint8)(int) t;  otherwise 0 if t <= 0, 255 if t >= 255, else
 * (int) t.
 * SMOOTH (ImageFilter.SMOOTH, ImagingFilter 3x3): weights 1/13 around and 5/13 at the centre, each an fp32 quotient,
 * ss = sum of v * w from 0 in row-major tap order (row y - 1 first, x - 1 first), then 0 if ss <= 0, 255 if ss >= 255,
 * else (int)(ss + 0.5); the first and last rows and columns are copied unfiltered.
 *
 * Frames are uint8 RGB [frames][H][W][3], contiguous.  Conventions as in svi_b200.h: 0 on success, a negative status (and
 * svi_last_error) on a rejected argument, in which case nothing is launched; every launch is on `stream`.  Only
 * svi_luma_sum_u8 uses atomics, on integers, so every entry point gives the same bytes for the same input.
 * A separate header so that svi_b200.h and its ABI version stay as they are.
 */
#ifndef SVI_B200_PROCESSORS_H_
#define SVI_B200_PROCESSORS_H_

#include <stdint.h>

#include "svi_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* sums[f] = sum of L over the n_pix pixels of frame f (sums is zeroed on `stream` first).  frames <= 65535. */
int svi_luma_sum_u8(const uint8_t* rgb, int32_t frames, int64_t n_pix, uint64_t* sums, void* stream);

/* out = blend(degenerate[f], rgb, rate) for every byte of frame f; degenerate: f32 [frames] on the device, each a whole
 * number in [0, 255]; rate finite.  out may equal rgb. */
int svi_enhance_blend_u8(const uint8_t* rgb, int32_t frames, int64_t n_pix, const float* degenerate, float rate,
                         uint8_t* out, void* stream);

/* out = blend(SMOOTH(rgb), rgb, rate) per frame of H x W; rate finite.  out must not overlap rgb. */
int svi_sharpen_u8(const uint8_t* rgb, int32_t frames, int32_t H, int32_t W, float rate, uint8_t* out, void* stream);

/* For the inner frames f = 1 .. frames - 2:  out[f] = R, G, B of ((frame[f] + merged[f - 1]) / 2 * 255).clip(0, 255)
 * truncated, in fp32 in that order.  frame: f32 [frames][n_pix][4] (B, G, R, unused) as svi_rife_stage_frames writes it;
 * merged: f32 [frames - 2][n_pix][4] (B, G, R, mask) as svi_rife_update_warp writes it; out: uint8 [frames][n_pix][3].
 * Frames 0 and frames - 1 of out are not written: they keep the input bytes.  frames >= 3. */
int svi_rife_average_u8(const float* frame, const float* merged, int32_t frames, int64_t n_pix, uint8_t* out,
                        void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SVI_B200_PROCESSORS_H_ */
