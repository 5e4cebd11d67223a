"""VAE throughput on one GPU (BASELINE configs[4] style sweep, reduced): decode / encode wall time (CUDA events),
algorithmic TFLOP/s from the per-position formulas of BASELINE.md §3, and per-kernel launch counts.

    python tools/vae_bench.py [--frames 81] [--height 480] [--width 832]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-video-infinity_b200")):
    sys.path.insert(0, p)
from tools import synth_vae  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=81)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=832)
    ap.add_argument("--iters", type=int, default=2)
    a = ap.parse_args()
    from diffsynth.models.wan_video_vae import WanVideoVAE
    vae = WanVideoVAE().eval()
    vae.load_state_dict(synth_vae.make_vae_state_dict(seed=0))
    vae.to("cuda")
    eng = vae.engine("cuda")
    T, H, W = a.frames, a.height, a.width
    tl, h, w = (T - 1) // 4 + 1, H // 8, W // 8
    g = torch.Generator().manual_seed(0)
    z = torch.randn(16, tl, h, w, generator=g).cuda()
    video = (torch.rand(3, T, H, W, generator=g) * 2 - 1).cuda()
    res = {}
    for name, fn, flops in (("decode", lambda: eng.decode(z), (0.688 + 2.162 * (tl - 1)) * 1e9 * h * w),
                            ("encode", lambda: eng.encode(video), (6.66 + 5.00 * (tl - 1)) * 1e6 * H * W)):
        fn()
        torch.cuda.synchronize()
        l0 = eng.launches
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.iters
        res[name] = {"ms": ms, "tflops": flops / ms / 1e9, "algorithmic_tflop": flops / 1e12,
                     "launches": (eng.launches - l0) // a.iters, "frames_per_s": T / ms * 1e3}
    print(json.dumps({"workload": f"vae {T}f x {H}x{W}", "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30, **res}))


def sweep_from_bench(args):
    """bench.py --workload cfg5 (BASELINE configs[4]): VAE encode / decode at 17..161 frames x 720 x 1280 on one GPU.  Per point:
    CUDA-event time (1 warm-up + 1 timed call through WanVideoVAE.encode / .decode, the public API), algorithmic TFLOP/s
    (BASELINE.md section 3 formulas) against the measured bf16 peak and minimal-traffic GB/s (conv in + out, bf16: SURVEY
    section 8d) against the measured HBM peak.  One JSON line; `value` = decoded pixel frames per second at 81 frames."""
    from diffsynth.models.wan_video_vae import WanVideoVAE
    from tools import flops
    world, rank, local = (int(os.environ.get(k, d)) for k, d in (("WORLD_SIZE", "1"), ("RANK", "0"), ("LOCAL_RANK", "0")))
    torch.cuda.set_device(local)
    if world > 1:      # N GPUs: every encode / decode is split into row bands (SpatialShard), times are the max over ranks
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    peaks = {}
    pp = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pp):
        peaks = json.load(open(pp))
    # without a measured file: NVIDIA's data-sheet figures for the H100 SXM (dense bf16, HBM3), not reached by a power-capped card
    tf_peak = peaks.get("bf16_tflops_sustained", 989.0)
    bw_peak = peaks.get("hbm_gbs", peaks.get("hbm_gbps", 3350.0))
    vae = WanVideoVAE().eval()
    vae.load_state_dict(synth_vae.make_vae_state_dict(seed=0))
    vae.to("cuda")
    if world > 1:
        vae.enable_spatial_sharding()
    H, W = 720, 1280
    h, w = H // 8, W // 8
    pts = []
    frames_list = [int(v) for v in os.environ.get("SVI_VAE_SWEEP", "17,33,49,81,113,161").split(",")]
    for T in frames_list:
        tl = (T - 1) // 4 + 1
        g = torch.Generator().manual_seed(T)
        z = torch.randn(1, 16, tl, h, w, generator=g).cuda()
        video = (torch.rand(3, T, H, W, generator=g) * 2 - 1).cuda()
        row = {"frames": T, "latent_frames": tl}
        for name, fn, fl in (("decode", lambda: vae.decode(z, device="cuda"), flops.vae_decode_flops(tl, h, w)),
                             ("encode", lambda: vae.encode([video], device="cuda"), flops.vae_encode_flops(tl, H, W))):
            fn()
            if world > 1:
                dist.barrier()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
            if world > 1:
                tt = torch.tensor([ms], device="cuda")
                dist.all_reduce(tt, op=dist.ReduceOp.MAX)
                ms = tt.item()
            row[name] = {"ms": ms, "tflops": fl / ms / 1e9, "frac_of_bf16_peak": fl / ms / 1e9 / tf_peak, "frames_per_s": T / ms * 1e3}
            if name == "decode":
                nb = flops.vae_min_bytes(tl, h, w)
                row[name].update(min_traffic_gbs=nb / ms / 1e6, frac_of_hbm_peak=nb / ms / 1e6 / bw_peak)
        pts.append(row)
        del z, video
        torch.cuda.empty_cache()
    if world > 1:
        dist.destroy_process_group()
        if rank != 0:
            return
    ref = next((p for p in pts if p["frames"] == 81), pts[-1])
    print(json.dumps({"metric": "VAE decoded pixel frames/sec (720p)", "value": ref["decode"]["frames_per_s"], "unit": "frames/s",
                      "n_gpus": world, "higher_is_better": True, "scaling": "strong",
                      "parallelism": "single" if world == 1 else f"row bands over {world} ranks, 1-row halo exchange per conv input", "dtype": "bf16 conv operands, fp32 activations", "data": "synthetic",
                      "config": {"workload": "cfg5", "description": "3D-VAE encode/decode sweep 17..161 frames x 720x1280 (BASELINE configs[4])"},
                      "peaks": {"bf16_tflops_sustained": tf_peak, "hbm_gbs": bw_peak, "note": "per-GPU peaks; fractions below are of ONE GPU's peak"},
                      "points": pts,
                      "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30}), flush=True)


if __name__ == "__main__":
    main()
