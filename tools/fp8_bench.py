"""e4m3 weights (the reference's weight-only FP8 mode, torch_dtype=torch.float8_e4m3fn) against bf16 weights on one GPU.

    python tools/fp8_bench.py [--gemm-only] [--frames 81 --height 480 --width 832] [--steps 2]

1. svi_gemm_bf16 with an e4m3 W against the same GEMM with W.to(bf16): M = 32760 at the 1.3B and 14B N/K (the bench
   shapes), M = 512 at the umT5-XXL shapes, M = 1 (time projection).  Both variants of a shape are warmed up, then timed
   in alternating rounds with CUDA events; the median per call is reported.
2. The 14B-I2V CFG step (two forwards + the fused CFG/Euler step) at 480p in both formats, random-init weights created on the
   device, with the peak device memory of each run.  The two models do not fit on one 80 GB card together, so these two
   runs are sequential (e4m3 first).

Prints one JSON object with the card's name and power limit, read in the same run."""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-video-infinity_b200")):
    sys.path.insert(0, p)
from tools import synth  # noqa: E402

GEMMS = [  # (label, M, N, K)
    ("1.3B qkv", 32760, 3 * 1536, 1536), ("1.3B o", 32760, 1536, 1536), ("1.3B ffn0", 32760, 8960, 1536),
    ("1.3B ffn2", 32760, 1536, 8960),
    ("14B qkv", 32760, 3 * 5120, 5120), ("14B o", 32760, 5120, 5120), ("14B ffn0", 32760, 13824, 5120),
    ("14B ffn2", 32760, 5120, 13824),
    ("umT5 qkv", 512, 3 * 4096, 4096), ("umT5 ffn in", 512, 10240, 4096), ("umT5 ffn out", 512, 4096, 10240),
    ("time proj 1.3B", 1, 6 * 1536, 1536), ("time proj 14B", 1, 6 * 5120, 5120),
]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def time_gemms(rounds=7, iters=20):
    from diffsynth import _native as nv
    res = []
    for label, M, N, K in GEMMS:
        g = torch.Generator(device="cuda").manual_seed(0)
        a = torch.randn(M, K, generator=g, device="cuda").to(torch.bfloat16)
        w8 = (torch.randn(N, K, generator=g, device="cuda") * 0.05).to(torch.float8_e4m3fn)
        wb = w8.to(torch.bfloat16)
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        times = {"e4m3": [], "bf16": []}
        for w in (w8, wb):                      # warm-up of both variants
            for _ in range(3):
                nv.gemm(a, w, out)
        torch.cuda.synchronize()
        for r in range(rounds):                 # alternating A/B rounds, the order flipped every round
            for name in (("e4m3", "bf16") if r % 2 == 0 else ("bf16", "e4m3")):
                w = w8 if name == "e4m3" else wb
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    nv.gemm(a, w, out)
                e1.record()
                e1.synchronize()
                times[name].append(e0.elapsed_time(e1) / iters)
        t8, tb = statistics.median(times["e4m3"]), statistics.median(times["bf16"])
        res.append({"gemm": label, "M": M, "N": N, "K": K, "e4m3_ms": round(t8, 4), "bf16_ms": round(tb, 4),
                    "e4m3_over_bf16": round(t8 / tb, 3), "bf16_tflops": round(2.0 * M * N * K / tb / 1e9, 1),
                    "spread_bf16_ms": round(max(times["bf16"]) - min(times["bf16"]), 4)})
        del a, w8, wb, out
    torch.cuda.empty_cache()
    return res


def step_14b(dtype, frames, height, width, steps):
    from diffsynth.models.wan_video_dit import WanModel, precompute_freqs_cis_3d
    cfg = synth.CFG_I2V_14B
    gc.collect()                     # a model and its engine reference each other: free the previous run's pair first
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.device("meta"):
        m = WanModel(**cfg)
    m = m.to(dtype)
    m.to_empty(device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if p.dim() >= 2 and "modulation" not in name:
                p.copy_((torch.randn(p.shape, generator=g, device="cuda") * (1.0 / p[0].numel() ** 0.5)).to(dtype))
            elif name.endswith("bias"):
                p.zero_()
            elif "modulation" in name:
                p.copy_((torch.randn(p.shape, generator=g, device="cuda") * 0.02).to(dtype))
            else:
                p.fill_(1.0)
    m.freqs = precompute_freqs_cis_3d(cfg["dim"] // cfg["num_heads"])
    m.eval()
    eng = m.engine("cuda")
    torch.cuda.synchronize()
    weights_gb = (torch.cuda.memory_allocated() - base) / 2 ** 30
    f, h, w = (frames - 1) // 4 + 1, height // 8, width // 8
    inp = synth.make_dit_inputs(cfg, f, h, w, seed=0, ctx_len=512)
    x = inp["x"].cuda().float()
    y, clip = inp["y"].cuda(), inp["clip_feature"].cuda()
    cp = eng.context_state(inp["context"].cuda(), clip)
    cn = eng.context_state(torch.randn(inp["context"].shape, generator=torch.Generator().manual_seed(2)).cuda(), clip)
    v_c, v_u = torch.empty_like(x), torch.empty_like(x)

    def step(t):
        eng.forward(x, t, cp, y=y, out=v_c)
        eng.forward(x, t, cn, y=y, out=v_u)
        eng.k.cfg_euler_step(x, v_c, v_u, 5.0, 0.9, 0.88)

    step(900.0)
    step(880.0)                      # second call of the geometry: captured into a CUDA graph
    torch.cuda.synchronize()
    ms = []
    for i in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step(860.0 - 20.0 * i)
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    out = {"weights": str(dtype).replace("torch.", ""), "tokens": f * (h // 2) * (w // 2), "ms_per_cfg_step": [round(v, 1) for v in ms],
           "model_and_engine_gb": round(weights_gb, 2), "peak_mem_gb": round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2)}
    del eng, m, cp, cn, x, y, clip, v_c, v_u
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gemm-only", action="store_true")
    ap.add_argument("--frames", type=int, default=81)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=832)
    ap.add_argument("--steps", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_bench.py measures on a CUDA device; none is visible")
    res = {"card": card(), "gemm": time_gemms()}
    if not a.gemm_only:
        res["dit_14b_i2v"] = [step_14b(d, a.frames, a.height, a.width, a.steps) for d in (torch.float8_e4m3fn, torch.bfloat16)]
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
