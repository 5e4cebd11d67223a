"""Time the video processors (diffsynth.processors) on an 81-frame clip at 832x480 and 1280x720, PIL frames in and out.

Each native processor end to end (host conversions, both transfers and the device work inside the timed window):
ContrastEditor(1.5), SharpnessEditor(1.5), RIFESmoother (interpolate True and False, batch 4, synthetic full-size IFNet
weights) and FastBlendSmoother (fast mode, window 15, batch 8, guided by the frames themselves); next to them Pillow's
ImageEnhance Contrast / Sharpness frame by frame on the host, and the four-processor chain [FastBlend, RIFE, Contrast,
Sharpness] twice: as SequencialProcessor (frames staged once, kept on the device) and as the reference runs it, each
processor called with PIL frames.  A 3-frame run of each warms it up.  The cases then run in --repeats rounds, one run
of every case per round, so that a drift of the card or the host reaches all of them alike; per case one JSON line
with the fastest, median and slowest run, and the card's name, power limit and SM clock, read in the same call.

usage:  python tools/processors_bench.py [--frames 81] [--sizes 832x480,1280x720] [--repeats 5] [--cases a,b]
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

import torch  # noqa: E402
from PIL import ImageEnhance  # noqa: E402

from tools.fastblend_bench import card  # noqa: E402
from tools import synth_rife as S  # noqa: E402


def cases(model):
    from diffsynth.processors.FastBlend import FastBlendSmoother
    from diffsynth.processors.PILEditor import ContrastEditor, SharpnessEditor
    from diffsynth.processors.RIFE import RIFESmoother
    from diffsynth.processors.sequencial_processor import SequencialProcessor

    def chain():
        return [FastBlendSmoother(inference_mode="fast", batch_size=8, window_size=15),
                RIFESmoother(model, device="cuda", batch_size=4), ContrastEditor(1.5), SharpnessEditor(1.5)]

    def one_by_one(frames):
        for p in chain():
            frames = p(frames)
        return frames

    return {
        "contrast": ContrastEditor(1.5),
        "pillow_contrast": lambda fr: [ImageEnhance.Contrast(im).enhance(1.5) for im in fr],
        "sharpness": SharpnessEditor(1.5),
        "pillow_sharpness": lambda fr: [ImageEnhance.Sharpness(im).enhance(1.5) for im in fr],
        "rife_interpolate": RIFESmoother(model, device="cuda", batch_size=4, interpolate=True),
        "rife_average": RIFESmoother(model, device="cuda", batch_size=4, interpolate=False),
        "fastblend_fast": FastBlendSmoother(inference_mode="fast", batch_size=8, window_size=15),
        "chain_on_device": SequencialProcessor(chain()),
        "chain_through_pil": one_by_one,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=81)
    ap.add_argument("--sizes", default="832x480,1280x720")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--cases", default=None, help="comma-separated subset of the cases")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    from diffsynth.extensions.RIFE import IFNet
    model = IFNet().eval()
    model.load_state_dict(S.make_state_dict(seed=0))
    model = model.cuda()
    todo = cases(model)
    names = a.cases.split(",") if a.cases else list(todo)
    for size in a.sizes.split(","):
        W, H = (int(v) for v in size.split("x"))
        frames = S.make_frames(a.frames, H, W, seed=0)
        for name in names:
            todo[name](frames[:3])
        torch.cuda.synchronize()
        times = {name: [] for name in names}
        for _ in range(a.repeats):
            for name in names:
                t0 = time.perf_counter()
                out = todo[name](frames)
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t0)
                assert len(out) == len(frames)
        gpu, power, sm, sm_max = card()
        for name in names:
            t = sorted(times[name])
            print(json.dumps({"case": name, "size": size, "frames": a.frames, "runs": len(t), "s_min": round(t[0], 4),
                              "s_median": round(t[len(t) // 2], 4), "s_max": round(t[-1], 4), "gpu": gpu,
                              "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}), flush=True)


if __name__ == "__main__":
    main()
