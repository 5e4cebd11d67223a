"""Time FastBlend's balanced and accurate modes and keyframe interpolation on an 81-frame clip at 832x480, with the
reference UI's defaults: window 15 and batch 8, and for interpolation minimum patch 15 with a keyframe every 10 frames
(two keyframes around each frame; the single-keyframe runner from the middle frame).

Each runner end to end: frames in, PIL frames out, so the host conversions, both transfers and the device work are inside
the timed window.  A 3-frame run of the same size warms each mode up.  Per mode one JSON line: seconds per video, the
number of estimate_nnf batches, candidate evaluations per second (each PatchMatch iteration evaluates 8 + 2T candidate
fields per pixel: the current one, four neighbour steps, three random steps and 2T tracking steps; counted from the level
shapes), the peak of torch's device allocations, and the card's name, power limit and SM clock, read in the same call.
With --profile, one more untimed run of each mode under torch.profiler prints the device time per kernel.

usage:  python tools/fastblend_modes_bench.py [--frames 81] [--size 832x480] [--modes balanced,accurate,interpolation,single]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-video-infinity_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

from tools.fastblend_bench import card  # noqa: E402
from tools.synth_fastblend import make_frames  # noqa: E402

CONFIG = dict(minimum_patch_size=5, threads_per_block=8, num_iter=5, gpu_id=0, guide_weight=10.0, initialize="identity",
              tracking_window_size=0)
WINDOW, BATCH, KEY_EVERY = 15, 8, 10


class Counter:
    """counts estimate_nnf batches and the candidate evaluations they make, from shapes"""

    def __init__(self, cls):
        self.batches = self.candidates = 0
        inner = cls.estimate_nnf_device

        def counted(engine, sg, tg, ss):
            self.batches += 1
            px = sum(h * w for h, w in zip(engine.pyramid_heights, engine.pyramid_widths))
            self.candidates += sg.shape[0] * px * engine.num_iter * (8 + 2 * engine.tracking_window_size)
            return inner(engine, sg, tg, ss)

        cls.estimate_nnf_device = counted


def call(mode, guide, style):
    from diffsynth.extensions.FastBlend import runners
    n = len(guide)
    if mode == "balanced":
        return runners.BalancedModeRunner().run(guide, style, BATCH, WINDOW, CONFIG)
    if mode == "accurate":
        return runners.AccurateModeRunner().run(guide, style, BATCH, WINDOW, CONFIG)
    if mode == "interpolation":
        keys = list(range(0, n, KEY_EVERY))
        return runners.InterpolationModeRunner().run(guide, [style[k] for k in keys], keys, BATCH,
                                                     dict(CONFIG, minimum_patch_size=15))
    return runners.InterpolationModeSingleFrameRunner().run(guide, [style[n // 2]], [n // 2], BATCH,
                                                            dict(CONFIG, minimum_patch_size=15))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=81)
    ap.add_argument("--size", default="832x480")
    ap.add_argument("--modes", default="balanced,accurate,interpolation,single")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    from diffsynth.extensions.FastBlend import PyramidPatchMatcher
    counter = Counter(PyramidPatchMatcher)
    W, H = (int(v) for v in a.size.split("x"))
    raw = make_frames(a.frames, H, W, seed=0)
    guide = [Image.fromarray(f) for f in raw]
    style = [Image.fromarray(np.ascontiguousarray(f[..., ::-1])) for f in raw]
    for mode in a.modes.split(","):
        call(mode, guide[:3], style[:3])
        torch.cuda.synchronize()
        counter.batches = counter.candidates = 0
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        out = call(mode, guide, style)
        dt = time.perf_counter() - t0
        assert len(out) == len(guide)
        name, power, sm, sm_max = card()
        print(json.dumps({"mode": mode, "size": a.size, "frames": a.frames, "s_per_video": round(dt, 3),
                          "estimate_nnf_batches": counter.batches,
                          "candidate_evals_per_s": float(f"{counter.candidates / dt:.4g}"),
                          "peak_alloc_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), "gpu": name,
                          "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}), flush=True)
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call(mode, guide, style)
                torch.cuda.synchronize()
            totals = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" and e.self_device_time_total > 0:
                    totals[e.key] = totals.get(e.key, 0.0) + e.self_device_time_total / 1e3
            top = sorted(totals.items(), key=lambda kv: -kv[1])[:8]
            print(json.dumps({"mode": mode, "device_ms_total": round(sum(totals.values()), 1),
                              "kernels_ms": {k[:80]: round(v, 1) for k, v in top}}), flush=True)


if __name__ == "__main__":
    main()
