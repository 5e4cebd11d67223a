"""End-to-end time of the cross-attention scorers (PIL frames in, floats out): 81 frames at 832x480 against one prompt,
ImageReward (BLIP ViT-L/16 + BERT-base) and MPS (CLIP ViT-H/14 + 4-layer cross model), real sizes, seeded weights
(tools/synth_reward).  The native scorer scores the 81 frames in one call; the fp32 oracle (oracle/reward_oracle.py)
scores them one image per call, re-encoding the prompt each time, as the reference's score() does.  The two alternate;
each is timed with CUDA events around work that ends in a synchronise.  A second native pass reports the time split
between the towers (vision and text) and the heads (BERT stack / cross model and the score).

    python tools/reward_bench.py [--frames 81] [--reps 3] [--metrics ImageReward,MPS]

Prints the card, power limit and SM clock with the numbers, and one JSON line.
"""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stable-video-infinity_b200")]

from tools import synth_quality as SQ  # noqa: E402
from tools import synth_reward as R  # noqa: E402
from tools.quality_bench import card, timed  # noqa: E402


def full_checkpoints(d):
    """real-size ImageReward and MPS files (the tokenizer files are the tiny synthetic ones)"""
    from safetensors.torch import save_file
    paths, _ = R.write_reward_checkpoints(os.path.join(d, "tiny"))
    V = json.load(open(paths["med_config"]))["vocab_size"]
    med = dict(R.FULL_MED, vocab_size=V)
    with open(paths["med_config"], "w") as f:
        json.dump(med, f)
    ir = R.imagereward_state_dict(med, R.FULL_VISION, seed=71)
    save_file({k: v.contiguous() for k, v in ir.items()}, paths["imagereward"])
    conf = json.load(open(os.path.join(paths["clip"], "config.json")))
    conf = dict(SQ.HF_FULL_PICK, text_config=dict(SQ.HF_FULL_PICK["text_config"], vocab_size=conf["text_config"]["vocab_size"]))
    R.write_clip_dir(paths["clip"], SQ.learn_merges(), conf)
    mps = R.mps_state_dict(conf, layers=4, seed=72)
    save_file({k: v.contiguous() for k, v in mps.items()}, paths["mps"])
    return paths, {"imagereward": (med, ir), "mps": (conf, mps)}


def split(name, model, frames, prompt):
    """(tower ms, head ms) of one native call: the vision tower and the text tower, then the rest"""
    from diffsynth.extensions.ImageQualityMetric import towers as T
    eng = model.engine()
    if name == "ImageReward":
        px = torch.stack([T.blip_pixels(f, 224) for f in frames]).cuda()
        ids, mask = model.tokenize(prompt)
        t_tower, _ = timed(lambda: (eng.vision.image_states(px), eng.prompt_states(ids, mask)))
        t_all, _ = timed(lambda: eng.score(px, ids, mask))
    else:
        px = torch.stack([T.hf_pixels(model.image_processor, f) for f in frames]).cuda()
        ids, cids = model.tokenize(prompt), model.tokenize(model.condition_prompt())
        t_tower, _ = timed(lambda: (eng.vision.image_states(px), eng.text.encode_text_rows(torch.cat([ids, cids]))))
        t_all, _ = timed(lambda: eng.score(px, ids, cids))
    return t_tower, t_all - t_tower


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=81)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--metrics", default="ImageReward,MPS")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "reward_bench measures on a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    from diffsynth.extensions.ImageQualityMetric import load_preference_model
    from diffsynth.extensions.ImageQualityMetric import towers as T
    from oracle import reward_oracle as O
    frames = SQ.frames(a.frames, 480, 832, seed=7)
    prompt = "a cinematic video frame of a city street at night, neon lights reflecting in the rain"
    result = {"card": card(), "frames": a.frames}
    print("card:", result["card"])
    with tempfile.TemporaryDirectory() as d:
        paths, ref = full_checkpoints(d)
        for name in a.metrics.split(","):
            model = load_preference_model(name, device="cuda", path=paths)
            conf, sd = ref["imagereward" if name == "ImageReward" else "mps"]
            sd = {k: v.cuda() for k, v in sd.items()}

            def oracle_one(f):
                if name == "ImageReward":
                    ids, mask = model.tokenize(prompt)
                    px = O.Q.normalize(T.blip_pixels(f, 224)[None].cuda())
                    return O.imagereward(sd, conf, 24, px, ids.cuda(), mask.cuda())[2].tolist()
                px = O.Q.normalize(T.hf_pixels(model.image_processor, f)[None].cuda(), *T.hf_mean_std(model.image_processor))
                ids, cids = model.tokenize(prompt).cuda(), model.tokenize(model.condition_prompt()).cuda()
                return O.mps(sd, conf, 16, 4, px, ids, cids)["scores"].tolist()

            def oracle_one_by_one():
                with torch.no_grad():
                    return [v for f in frames for v in oracle_one(f)]
            model.score(frames[:2], prompt)                          # warm-up of both paths
            oracle_one(frames[0])
            nat, ora = [], []
            for _ in range(a.reps):
                t, got = timed(lambda: model.score(frames, prompt))
                nat.append(t)
                t, want = timed(oracle_one_by_one)
                ora.append(t)
            with torch.no_grad():
                towers, heads = split(name, model, frames, prompt)
            err = max(abs(x - y) for x, y in zip(got, want))
            result[name] = {"native_ms": min(nat), "oracle_fp32_ms": min(ora), "towers_ms": towers, "heads_ms": heads,
                            "max_abs_score_diff": err}
            print(f"{name}: native {min(nat):.1f} ms for {a.frames} frames ({min(nat) / a.frames:.2f} ms/frame; towers "
                  f"{towers:.1f} ms, heads {heads:.1f} ms, host preprocessing the rest), fp32 one-by-one {min(ora):.1f} ms, "
                  f"speed-up {min(ora) / min(nat):.1f}x, |score diff| max {err:.2e}")
            del model
            torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
