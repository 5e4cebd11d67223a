"""Time FastBlend deflickering of an 81-frame clip at 832x480 and 1280x720 with the default config.

`FastBlendSmoother()(frames)` end to end: PIL frames in, PIL frames out, so the host conversions, both transfers and
the device work are inside the timed window (the call ends with the frames on the host).  A 3-frame clip of the same size
runs first as a warm-up.  Reports seconds per video, ms per frame, the number of estimate_nnf batches, candidate
evaluations per second (each PatchMatch iteration evaluates 8 candidate fields per pixel: the current one, four
neighbour steps and three random steps; counted from the level shapes) and the card's name, power limit and SM clock,
read in the same call, and the peak of torch's device allocations during the timed call.  The reference needs CuPy and is
not timed here.  Prints one JSON line per size.  With --profile, one more untimed run of the first size under
torch.profiler prints the device time per kernel (a separate run: tracing slows the host).

usage:  python tools/fastblend_bench.py [--frames 81] [--sizes 832x480,1280x720] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-video-infinity_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
from PIL import Image  # noqa: E402

from tools.synth_fastblend import make_frames  # noqa: E402

CANDIDATES_PER_ITERATION = 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    return [s.strip() for s in q.split(",")]


class Counter:
    """counts estimate_nnf batches and the candidate evaluations they make, from shapes"""

    def __init__(self, cls):
        self.batches = self.candidates = 0
        inner = cls.estimate_nnf_device

        def counted(engine, sg, tg, ss):
            self.batches += 1
            px = sum(h * w for h, w in zip(engine.pyramid_heights, engine.pyramid_widths))
            self.candidates += sg.shape[0] * px * engine.num_iter * CANDIDATES_PER_ITERATION
            return inner(engine, sg, tg, ss)

        cls.estimate_nnf_device = counted


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=81)
    ap.add_argument("--sizes", default="832x480,1280x720")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    from diffsynth.extensions.FastBlend import FastBlendSmoother, PyramidPatchMatcher
    counter = Counter(PyramidPatchMatcher)
    for size in a.sizes.split(","):
        W, H = (int(v) for v in size.split("x"))
        frames = [Image.fromarray(f) for f in make_frames(a.frames, H, W, seed=0)]
        smoother = FastBlendSmoother()
        smoother(frames[:3])
        torch.cuda.synchronize()
        counter.batches = counter.candidates = 0
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        out = smoother(frames)
        dt = time.perf_counter() - t0
        assert len(out) == len(frames)
        name, power, sm, sm_max = card()
        print(json.dumps({"size": size, "frames": a.frames, "s_per_video": round(dt, 3),
                          "ms_per_frame": round(1e3 * dt / a.frames, 2), "estimate_nnf_batches": counter.batches,
                          "candidate_evals_per_s": float(f"{counter.candidates / dt:.4g}"),
                          "peak_alloc_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), "gpu": name,
                          "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max,
                          "reference": "not measured (needs CuPy)"}), flush=True)
    if a.profile:
        W, H = (int(v) for v in a.sizes.split(",")[0].split("x"))
        frames = [Image.fromarray(f) for f in make_frames(a.frames, H, W, seed=0)]
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            FastBlendSmoother()(frames)
            torch.cuda.synchronize()
        totals = {}
        for e in prof.key_averages():
            if e.device_type.name == "CUDA" and e.self_device_time_total > 0:
                totals[e.key] = totals.get(e.key, 0.0) + e.self_device_time_total / 1e3
        top = sorted(totals.items(), key=lambda kv: -kv[1])[:10]
        print(json.dumps({"size": f"{W}x{H}", "device_ms_total": round(sum(totals.values()), 1),
                          "kernels_ms": {k[:80]: round(v, 1) for k, v in top}}), flush=True)


if __name__ == "__main__":
    main()
