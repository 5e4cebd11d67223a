"""Time ESRGAN x4 upscaling of 16 frames at batch 4, at 832x480 and 1280x720.

Native: ESRGAN.upscale end to end (PIL frames in, PIL frames out: the host conversions, both transfers and the device
work are inside the timed window), and the device work alone: CUDA events around the engine's calls (staging and the
convolutions) on frames already on the device, so the host's share is the difference.  Reference stand-in: the oracle's
fp32 RRDBNet (the reference's computation, on cuDNN, TF32 off) on the same GPU with the frames already on the device, at
--ref-batch frames per call (default 1: at 1280x720 one fp32 activation at 4x size is 3.8 GB per frame, and the
engine's own buffers stay allocated next to it).  The two alternate; each row is the median over the rounds.  Prints one
JSON line per size with the card name, power limit and SM clock.

usage:  python tools/esrgan_bench.py [--rounds 3] [--frames 16] [--batch 4] [--ref-batch 1]
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

from oracle import esrgan_oracle as O  # noqa: E402
from tools import synth_esrgan as S  # noqa: E402
from tools.flops import esrgan_flops  # noqa: E402
from tools.synth_rife import make_frames  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    return [s.strip() for s in q.split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--ref-batch", type=int, default=1)
    ap.add_argument("--sizes", default="480x832,720x1280")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("esrgan_bench needs a CUDA device")
    from diffsynth.extensions.ESRGAN import ESRGAN, RRDBNet
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = S.make_state_dict(23, seed=0)
    model = RRDBNet().eval()
    model.load_state_dict(sd)
    model.to("cuda")
    sdd = {k: v.cuda() for k, v in sd.items()}
    esr = ESRGAN(model)
    eng = model.engine("cuda")
    n = a.frames
    for size in a.sizes.split(","):
        H, W = (int(v) for v in size.split("x"))
        frames = make_frames(n, H, W, seed=0)
        u8 = torch.from_numpy(np.stack([np.asarray(f) for f in frames])).cuda()
        x = O.to_tensor(u8.cpu().numpy()).cuda()
        rgb = torch.empty(n, 4 * H, 4 * W, 3, dtype=torch.uint8, device="cuda")

        def native():
            torch.cuda.synchronize()
            t = time.perf_counter()
            esr.upscale(frames, batch_size=a.batch)
            torch.cuda.synchronize()
            return time.perf_counter() - t

        def device():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for b in range(0, n, a.batch):
                eng.upscale_u8(u8[b:b + a.batch], rgb[b:b + a.batch])
            e1.record()
            e1.synchronize()
            return e0.elapsed_time(e1) / 1e3

        def reference():
            torch.cuda.synchronize()
            t = time.perf_counter()
            with torch.no_grad():
                for b in range(0, n, a.ref_batch):
                    O.rrdbnet(sdd, x[b:b + a.ref_batch])
            torch.cuda.synchronize()
            return time.perf_counter() - t

        native(), device(), reference()
        tn, td, tr = [], [], []
        for _ in range(a.rounds):
            tn.append(native())
            td.append(device())
            tr.append(reference())
        name, plim, sm, smax = card()
        fl = esrgan_flops(H, W)
        mn, md, mr = float(np.median(tn)), float(np.median(td)), float(np.median(tr))
        print(json.dumps({"size": f"{W}x{H}", "frames": n, "batch": a.batch, "ref_batch": a.ref_batch,
                          "native_ms_per_frame": round(1e3 * mn / n, 2), "native_tflops": round(fl * n / mn / 1e12, 1),
                          "device_ms_per_frame": round(1e3 * md / n, 2), "device_tflops": round(fl * n / md / 1e12, 1),
                          "host_ms_per_frame": round(1e3 * (mn - md) / n, 2),
                          "fp32_torch_ms_per_frame": round(1e3 * mr / n, 2), "fp32_torch_tflops": round(fl * n / mr / 1e12, 1),
                          "speedup": round(mr / mn, 2), "tflop_per_frame": round(fl / 1e12, 2),
                          "native_s": [round(v, 4) for v in tn], "device_s": [round(v, 4) for v in td],
                          "fp32_torch_s": [round(v, 4) for v in tr], "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 1e9, 1),
                          "card": name, "power_limit": plim, "sm_clock": sm, "sm_clock_max": smax}), flush=True)


if __name__ == "__main__":
    main()
