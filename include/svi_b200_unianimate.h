/*
 * svi_b200_unianimate.h — sliding-window accumulation of the UniAnimate-DiT long-video loop on libsvi_b200.so (the same
 * library as svi_b200.h).
 *
 * WanUniAnimateLongVideoPipeline denoises a video longer than one clip in overlapping windows of `cs` latent frames.
 * After each window's CFG + Euler step its frames are added into an f32 per-frame sum (window 0 adds all of its frames,
 * every later window skips its first two); after the last window each frame is its sum divided by the number of
 * windows that added to it:
 *
 *   svi_window_accumulate   sum[c][start + j][p] += win[c][j][p] for skip <= j < cs
 *   svi_window_normalize    out[c][f][p] = sum[c][f][p] / count[f]   (IEEE round-to-nearest division)
 *
 * Layouts: `win` is f32 [C][cs][hw], `sum` and `out` are f32 [C][F][hw] (the [1, C, F, h, w] latents), `count` is int32
 * [F], a table the host builds once from the window schedule.  hw must be a multiple of 4 and every pointer 16-byte
 * aligned.  Every output element is computed by one thread, without atomics: additions happen in the order the windows
 * are launched, and the result does not depend on the launch configuration.
 * Conventions as in svi_b200.h: 0 on success, a negative status (and svi_last_error) on a rejected argument, in which
 * case nothing is launched; every launch is on `stream`.
 * A separate header so that svi_b200.h and its ABI version stay as they are.
 */
#ifndef SVI_B200_UNIANIMATE_H_
#define SVI_B200_UNIANIMATE_H_

#include <stdint.h>

#include "svi_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* sum (f32 [C][F][hw]) frames start + skip .. start + cs - 1 += win (f32 [C][cs][hw]) frames skip .. cs - 1.
 * Needs 0 <= skip < cs, 0 <= start, start + cs <= F; win must not overlap sum. */
int svi_window_accumulate(const float* win, int32_t C, int32_t cs, int64_t hw, int32_t skip, float* sum, int32_t F,
                          int32_t start, void* stream);

/* out (f32 [C][F][hw]) = sum / count[f], count int32 [F] (each > 0; not checked on the device).  out may be sum itself
 * but must not overlap it otherwise. */
int svi_window_normalize(const float* sum, const int32_t* count, int32_t C, int32_t F, int64_t hw, float* out,
                         void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SVI_B200_UNIANIMATE_H_ */
