/*
 * svi_b200_replace.h — input staging of the UniAnimate-DiT Replace-Anyone pipeline on libsvi_b200.so (the same library
 * as svi_b200.h).
 *
 * WanRepalceAnyoneVideoPipeline re-animates the masked person of a video.  Before its loop it needs the video with the
 * person cut out twice: as f32 planar frames for the VAE encoder, and as the first input of the learn-in stem (the
 * masked RGB plus the keep mask, four channels) in the bf16 channels-last frame ring of the conv kernel.  One pass over
 * the video and its segmentation writes both:
 *
 *   keep          = !((float)seg / 255.0f > 0.0f)                    (IEEE division; a NaN segmentation value keeps)
 *   masked[c]     = video[c] * (float)keep                           (c = 0..2; -0.0 and NaN as an IEEE multiply gives)
 *   ring[pixel]   = { bf16_rn(masked[0]), bf16_rn(masked[1]), bf16_rn(masked[2]), bf16(keep) }
 *
 * which is torch's `video * ~(seg / 255. > 0)` and `cat([that, (~seg).float()]).to(torch.bfloat16)` bit for bit.
 *
 * Layouts: `video` and `masked` are f32 [3][T][hw] (planar, the [1, 3, T, H, W] video), `seg` is uint8 or f32 [T][hw],
 * `ring` is bf16 [T][hw][ldr] (channels-last frames, ldr >= 4 and a multiple of 4, 8-byte aligned).  Ring channels
 * 4 .. ldr-1 are not written.  `masked` may be NULL (ring only).  Every pixel is computed by one thread, without atomics;
 * the result does not depend on the launch configuration.
 * Conventions as in svi_b200.h: 0 on success, a negative status (and svi_last_error) on a rejected argument, in which
 * case nothing is launched; every launch is on `stream`.
 * A separate header so that svi_b200.h and its ABI version stay as they are.
 */
#ifndef SVI_B200_REPLACE_H_
#define SVI_B200_REPLACE_H_

#include <stdint.h>

#include "svi_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define SVI_SEG_U8 0  /* seg is uint8 */
#define SVI_SEG_F32 1 /* seg is f32 */

/* See above.  T > 0, hw > 0; no output may overlap an input or the other output. */
int svi_replace_mask_stage(const float* video, const void* seg, int32_t seg_type, int32_t T, int64_t hw, float* masked,
                           void* ring, int32_t ldr, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SVI_B200_REPLACE_H_ */
