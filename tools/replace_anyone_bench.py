"""UniAnimate-DiT Replace-Anyone on one GPU: the per-call preparation of WanRepalceAnyoneVideoPipeline at a full clip.

    python tools/replace_anyone_bench.py [--height 480 --width 832 --frames 81 --reps 3]

Times, with CUDA events around each part (one warm-up call each, then the mean of --reps calls):
  * svi_replace_mask_stage alone (masked video + the learn-in stem's first ring);
  * the learn-in stem, including its mask stage;
  * the untiled VAE encode of the masked video (synthetic VAE weights, tools/synth_vae.py);
  * the inpaint stem on those latents;
  * x_c = latents + offset (svi_axpby), the only extra work of a denoising step.
Prints one JSON object with the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-video-infinity_b200")):
    sys.path.insert(0, p)
from tools import synth_replace_anyone as SR, synth_vae  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0]
    return [s.strip() for s in q.split(",")]


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=832)
    ap.add_argument("--frames", type=int, default=81)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("replace_anyone_bench.py measures on a GPU; none found")
    from diffsynth import _native as nv
    from diffsynth.models.dwpose_embedding import (InpaintEmbeddingEngine, LearnInEmbeddingEngine, make_inpaint_embedding,
                                                   make_learn_in_embedding)
    from diffsynth.models.wan_video_vae import WanVideoVAE
    H, W, T = a.height, a.width, a.frames
    learn_in, inpaint = make_learn_in_embedding(), make_inpaint_embedding()
    learn_in.load_state_dict(SR.learn_in_sd(seed=1))
    inpaint.load_state_dict(SR.inpaint_sd(seed=2))
    li, ip = LearnInEmbeddingEngine(learn_in, "cuda"), InpaintEmbeddingEngine(inpaint, "cuda")
    vae = WanVideoVAE().eval()
    vae.load_state_dict({k: v.to(torch.bfloat16).float() for k, v in synth_vae.make_vae_state_dict(seed=0).items()})
    vae.to("cuda")
    video = SR.video(T, H, W, seed=3).cuda()
    seg = SR.segmentation(T, H, W, seed=4)[0].cuda()
    masked = torch.empty_like(video)
    ring = torch.zeros(T, H, W, li.full[0].c_in, device="cuda", dtype=torch.bfloat16)

    ms_mask, _ = timed(lambda: nv.replace_mask_stage(video, seg, masked, ring), a.reps)
    del ring
    ms_learn_in, out_li = timed(lambda: li.forward(video, seg, masked), a.reps)
    ms_vae, lat = timed(lambda: vae.encode([masked], device="cuda"), a.reps)
    ms_inpaint, out_ip = timed(lambda: ip.forward(lat), a.reps)
    x = torch.randn_like(out_ip)
    x_c = torch.empty_like(x)
    ms_axpby, _ = timed(lambda: nv.axpby(x, 1.0, out_li, 1.0, x_c), 20)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    mask_bytes = T * H * W * (3 * 4 + seg.element_size() + 3 * 4 + 4 * 2)
    name, power = card()
    print(json.dumps({
        "workload": f"{W}x{H}, {T} frames ({tuple(lat.shape[2:])} latents)", "reps": a.reps,
        "ms_mask_stage": round(ms_mask, 3), "mask_stage_GBps": round(mask_bytes / ms_mask / 1e6, 1),
        "ms_learn_in_stem": round(ms_learn_in, 2), "ms_vae_encode": round(ms_vae, 2),
        "ms_inpaint_stem": round(ms_inpaint, 2), "ms_axpby_per_step": round(ms_axpby, 4),
        "ms_preparation_total": round(ms_learn_in + ms_vae + ms_inpaint, 2), "peak_gib": round(peak, 2),
        "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
