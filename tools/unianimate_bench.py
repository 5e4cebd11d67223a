"""UniAnimate-DiT long video on one GPU: WanUniAnimateLongVideoPipeline.__call__ with synthetic Wan2.1-I2V-14B weights
(created on the device, as tools/dit14b_bench.py does) and 5120-wide pose stems.

    python tools/unianimate_bench.py [--height 480 --width 832 --frames 161 --context-size 21 --context-overlap 4]
                                     [--steps 2 --warmup 1]

The default workload is 161 frames (41 latent frames) at 832x480 in windows of 21 overlapping by 4: three windows, the
last one realigned.  The prompt and image encoders and the VAE are replaced by fixed tensors; everything from the pose
stems to the last window step runs.  Device events give, per timed denoising step: the whole step, the DiT forwards
(two per window), the window kernels (svi_window_accumulate / svi_window_normalize) and, as the step minus the
forwards, everything else of the loop (window gather and carry copies, the CFG + Euler kernel, launch gaps).  Once per
call: both stems.  Prints one JSON object with the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-video-infinity_b200")):
    sys.path.insert(0, p)
from tools import synth, synth_unianimate as SU  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0]
    return [s.strip() for s in q.split(",")]


def dit_14b():
    from diffsynth.models.wan_video_dit import WanModel, precompute_freqs_cis_3d
    cfg = synth.CFG_I2V_14B
    with torch.device("meta"):
        m = WanModel(**cfg).to(torch.bfloat16)
    m.to_empty(device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if p.dim() >= 2 and "modulation" not in name:
                p.copy_((torch.randn(p.shape, generator=g, device="cuda") * (1.0 / p[0].numel() ** 0.5)).to(p.dtype))
            elif name.endswith("bias"):
                p.zero_()
            elif "modulation" in name:
                p.copy_((torch.randn(p.shape, generator=g, device="cuda") * 0.02).to(p.dtype))
            else:
                p.fill_(1.0)
    m.freqs = precompute_freqs_cis_3d(cfg["dim"] // cfg["num_heads"])
    return m.eval(), cfg


class Timer:
    """Pairs of CUDA events by label; the sum of a label's intervals in ms once synchronised."""

    def __init__(self):
        self.spans = {}

    def wrap(self, label, fn):
        def run(*a, **k):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = fn(*a, **k)
            e.record()
            self.spans.setdefault(label, []).append((s, e))
            return out
        return run

    def total(self, label, lo=0, hi=None):
        return sum(s.elapsed_time(e) for s, e in self.spans.get(label, [])[lo:hi])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=832)
    ap.add_argument("--frames", type=int, default=161)
    ap.add_argument("--context-size", type=int, default=21)
    ap.add_argument("--context-overlap", type=int, default=4)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unianimate_bench.py measures on a GPU; none found")
    from diffsynth import ModelManager, WanUniAnimateLongVideoPipeline
    from diffsynth import _native as nv
    from diffsynth.pipelines.wan_video import context_windows
    H, W, nf, cs = a.height, a.width, a.frames, a.context_size
    h, w, n_lat = H // 8, W // 8, (nf - 1) // 4 + 1
    wins = context_windows(n_lat, cs, a.context_overlap)
    dit, cfg = dit_14b()
    mm = ModelManager(torch_dtype=torch.bfloat16, device="cuda")
    mm.add_model("wan_video_dit", dit)
    mm.state_dict_new_module = {"dwpose_embedding." + k: v for k, v in SU.pose_stem_sd(cfg["dim"], seed=1).items()}
    mm.state_dict_new_module.update({"randomref_embedding_pose." + k: v for k, v in SU.ref_stem_sd(seed=2).items()})
    pipe = WanUniAnimateLongVideoPipeline.from_model_manager(mm, torch_dtype=torch.bfloat16, device="cuda")
    g = torch.Generator().manual_seed(3)
    ctx = {True: torch.randn(1, 512, cfg["text_dim"], generator=g).cuda(),
           False: torch.randn(1, 512, cfg["text_dim"], generator=g).cuda()}
    clip = torch.randn(1, 257, 1280, generator=g).cuda()
    y = (torch.randn(1, 20, cs, h, w, generator=g) * 0.5).to(torch.bfloat16).cuda()
    pipe.image_encoder = object()
    pipe.encode_prompt = lambda prompt, positive=True: {"context": ctx[positive]}
    pipe.encode_image = lambda image, num_frames, height, width: {"clip_feature": clip, "y": y}
    pipe.decode_video = lambda latents, **kw: torch.zeros(1, 3, 1, 8, 8, device="cuda")
    pose = SU.pose_video(nf, H, W, seed=4).cuda()
    ref = SU.ref_pose(H, W, seed=5).cuda()

    t = Timer()
    eng = dit.engine("cuda")
    eng.forward = t.wrap("forward", eng.forward)
    pipe.encode_pose = t.wrap("pose_stem", pipe.encode_pose)
    pipe.encode_ref_pose = t.wrap("ref_stem", pipe.encode_ref_pose)
    acc, norm = nv.window_accumulate, nv.window_normalize
    nv.window_accumulate, nv.window_normalize = t.wrap("window", acc), t.wrap("window", norm)
    marks = []

    def bar(it):
        for i in it:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            marks.append(e)
            yield i
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        marks.append(e)

    n_steps = a.warmup + a.steps
    try:
        pipe(prompt="p", negative_prompt="n", input_image=SU.dummy_image(H, W), seed=0, height=H, width=W, num_frames=nf,
             num_inference_steps=n_steps, tiled=False, progress_bar_cmd=bar, dwpose_data=pose, random_ref_dwpose=ref,
             context_size=cs, context_overlap=a.context_overlap)
        torch.cuda.synchronize()
    finally:
        nv.window_accumulate, nv.window_normalize = acc, norm
    fw_per_step, win_per_step = 2 * len(wins), len(wins) + 1
    step = sum(marks[i].elapsed_time(marks[i + 1]) for i in range(a.warmup, n_steps)) / a.steps
    fwd = t.total("forward", a.warmup * fw_per_step) / a.steps
    kern = t.total("window", a.warmup * win_per_step) / a.steps
    name, power = card()
    print(json.dumps({
        "workload": f"{W}x{H}, {nf} frames ({n_lat} latent), context {cs} overlap {a.context_overlap}",
        "windows": [w_[0] for w_ in wins], "timed_steps": a.steps,
        "ms_per_step": round(step, 2), "ms_dit_forwards_per_step": round(fwd, 2),
        "ms_outside_forwards_per_step": round(step - fwd, 2),
        "outside_forwards_share": round((step - fwd) / step, 5),
        "ms_window_kernels_per_step": round(kern, 3),
        "ms_pose_stem_per_call": round(t.total("pose_stem"), 2), "ms_ref_stem_per_call": round(t.total("ref_stem"), 2),
        "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
