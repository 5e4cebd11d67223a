"""End-to-end time of the quality scorers (PIL frames in, floats out): 81 frames at 832x480 against one prompt, per
metric, at the real tower sizes with seeded weights (tools/synth_quality).  The native scorer scores the 81 frames in one
call; the reference-equivalent fp32 oracle scores them one image per call (prompt re-encoded each time), as the
reference's score() does.  The two alternate; each is timed with CUDA events around work that ends in a synchronise.

    python tools/quality_bench.py [--frames 81] [--reps 3] [--metrics CLIP,PickScore,Aesthetic]

HPSv2 / v2.1 run the same ViT-H-14 towers as CLIP and are not timed separately.  Prints the card, power limit and SM
clock with the numbers, and one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stable-video-infinity_b200")]

from tools import synth_quality as S  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else torch.cuda.get_device_name()


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), out


def full_checkpoints(d, metrics):
    """the real-size checkpoints, written once (the tokenizer files are the tiny synthetic ones)"""
    import safetensors.torch as st
    paths, ref = S.write_tiny_checkpoints(os.path.join(d, "tiny"))
    if "CLIP" in metrics:
        cfg = dict(S.OPENCLIP_FULL, text_cfg=dict(S.OPENCLIP_FULL["text_cfg"], vocab_size=ref["oc_config"]["text_cfg"]["vocab_size"]))
        sd = S.openclip_state_dict(cfg, seed=31)
        paths["open_clip"] = os.path.join(d, "open_clip.safetensors")
        st.save_file(sd, paths["open_clip"])
        ref["open_clip"] = (cfg, sd)
    for key, conf, m in (("pickscore", S.HF_FULL_PICK, "PickScore"), ("clip-large", S.HF_FULL_LARGE, "Aesthetic")):
        if m in metrics:
            V = ref["pickscore"][0]["text_config"]["vocab_size"]
            conf = dict(conf, text_config=dict(conf["text_config"], vocab_size=V))
            sd = S.hf_state_dict(conf, seed=32)
            paths[key] = S.write_hf_model(os.path.join(d, key), conf, sd)
            if key == "clip-large":
                S.write_hf_dir(paths[key], S.learn_merges(), image_size=224)
            ref[key] = (conf, sd)
    S.write_hf_dir(paths["clip"], S.learn_merges(), image_size=224)
    return paths, ref


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=81)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--metrics", default="CLIP,PickScore,Aesthetic")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "quality_bench measures on a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    from diffsynth.extensions.ImageQualityMetric import load_preference_model
    metrics = a.metrics.split(",")
    frames = S.frames(a.frames, 480, 832, seed=7)
    prompt = "a cinematic video frame of a city street at night, neon lights reflecting in the rain"
    result = {"card": card(), "frames": a.frames}
    print("card:", result["card"])
    with tempfile.TemporaryDirectory() as d:
        paths, ref = full_checkpoints(d, metrics)
        for name in metrics:
            model = load_preference_model(name, device="cuda", path=paths)
            key = {"CLIP": "open_clip", "PickScore": "pickscore", "Aesthetic": "clip-large"}[name]
            gpu_ref = {key: (ref[key][0], {k: v.cuda() for k, v in ref[key][1].items()}),
                       "aesthetic_predictor": (None, {k: v.cuda() for k, v in ref["aesthetic_predictor"][1].items()})}

            def oracle_one_by_one():
                with torch.no_grad():
                    return [v for f in frames for v in S.oracle_scores(name, paths, gpu_ref, [f], prompt, device="cuda")]
            model.score(frames[:2], prompt)                          # warm-up of both paths
            S.oracle_scores(name, paths, gpu_ref, frames[:1], prompt, device="cuda")
            nat, ora = [], []
            for _ in range(a.reps):
                t, got = timed(lambda: model.score(frames, prompt))
                nat.append(t)
                t, want = timed(oracle_one_by_one)
                ora.append(t)
            err = max(abs(x - y) for x, y in zip(got, want))
            result[name] = {"native_ms": min(nat), "oracle_fp32_ms": min(ora), "max_abs_score_diff": err}
            print(f"{name}: native {min(nat):.1f} ms for {a.frames} frames ({min(nat) / a.frames:.2f} ms/frame), "
                  f"fp32 one-by-one {min(ora):.1f} ms, speed-up {min(ora) / min(nat):.1f}x, |score diff| max {err:.2e}")
            del model
            torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
