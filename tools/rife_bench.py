"""Time RIFE frame doubling: an 81-frame clip -> 161 frames (80 new), at 832x480 and 1280x720.

Native: RIFEInterpolater.interpolate end to end (PIL frames in, PIL frames out: the host conversions, both transfers
and the device work are inside the timed window).  Reference stand-in: the oracle's fp32 IFNet (the reference's
computation, on cuDNN, TF32 off) on the same GPU, batch 4, with the frames already on the device.  The two alternate;
each row is the median over the rounds.  Prints one JSON line per size with the card name, power limit and SM clock.

usage:  python tools/rife_bench.py [--rounds 3] [--frames 81] [--batch 4]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import rife_oracle as O  # noqa: E402
from tools import synth_rife as S  # noqa: E402
from tools.flops import rife_interp_flops  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    return [s.strip() for s in q.split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=81)
    ap.add_argument("--batch", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rife_bench needs a CUDA device")
    from diffsynth.extensions.RIFE import IFNet, RIFEInterpolater
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = S.make_state_dict(seed=0)
    model = IFNet().eval()
    model.load_state_dict(sd)
    model.to("cuda")
    sdd = {k: v.cuda() for k, v in sd.items()}
    interp = RIFEInterpolater(model, device="cuda")
    for H, W in ((480, 832), (720, 1280)):
        frames = S.make_frames(a.frames, H, W, seed=0)
        x = O.to_tensor(np.stack([np.asarray(f) for f in frames])).cuda()
        n_new = a.frames - 1

        def native():
            torch.cuda.synchronize()
            t = time.perf_counter()
            interp.interpolate(frames, batch_size=a.batch)
            torch.cuda.synchronize()
            return time.perf_counter() - t

        def reference():
            torch.cuda.synchronize()
            t = time.perf_counter()
            with torch.no_grad():
                for b in range(0, n_new, a.batch):
                    e = min(b + a.batch, n_new)
                    O.ifnet(sdd, torch.cat((x[b:e], x[b + 1:e + 1]), 1))[2][2].clip(0, 1)
            torch.cuda.synchronize()
            return time.perf_counter() - t

        native(), reference()
        tn, tr = [], []
        for _ in range(a.rounds):
            tn.append(native())
            tr.append(reference())
        name, plim, sm, smax = card()
        fl = rife_interp_flops(H, W)
        mn, mr = float(np.median(tn)), float(np.median(tr))
        print(json.dumps({"size": f"{W}x{H}", "new_frames": n_new, "batch": a.batch,
                          "native_ms_per_frame": round(1e3 * mn / n_new, 3), "native_tflops": round(fl * n_new / mn / 1e12, 2),
                          "fp32_torch_ms_per_frame": round(1e3 * mr / n_new, 3),
                          "fp32_torch_tflops": round(fl * n_new / mr / 1e12, 2), "speedup": round(mr / mn, 2),
                          "gflop_per_frame": round(fl / 1e9, 1), "native_s": [round(v, 4) for v in tn],
                          "fp32_torch_s": [round(v, 4) for v in tr], "card": name, "power_limit": plim, "sm_clock": sm,
                          "sm_clock_max": smax}), flush=True)


if __name__ == "__main__":
    main()
