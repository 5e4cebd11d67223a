"""Golden vectors of the UniAnimate-DiT Replace-Anyone pipeline from the REAL reference module
(pipelines/wan_video.py, ``WanRepalceAnyoneVideoPipeline``) on the CPU.

Runs only where the reference tree exists; its output, ``tests/golden/replace_anyone_tiny.npz``, is committed and pins
``oracle/replace_anyone_oracle.py``.  The reference module is loaded with make_golden_unianimate.py's loader and
``_FakeManager``.  The text and image encoders are replaced by fixed tensors; ``encode_video`` records its input (the
masked video) and returns seeded latents; ``decode_video`` records the latents it is given.

The reference's ``__call__`` runs only at the pipeline dtype bf16: at f32 it feeds the f32 VAE latents into the inpaint
stem it has just cast to bf16, and the convolution rejects the mixed dtypes.  At bf16 that input is the latents rounded
to bf16.  To pin the loop tightly the fixture runs at f32 and gives the inpaint stem that bf16 input (``_Bf16Input``);
everything else is the reference's own code.

The fixture holds, for a 9-frame 64x48 call (tools/synth_replace_anyone.py) on a one-layer 5120-wide DiT:
  * ``vae_input``: what ``encode_video`` received, f32 [1, 3, T, H, W];
  * ``learn_in_bf16`` / ``inpaint_bf16``: both stems' outputs as the reference ran them (bf16, stored as f32), and
    ``learn_in_f32`` / ``inpaint_f32``: the same reference-built modules in f32 on the same (bf16) inputs;
  * ``latents_cfg5`` / ``latents_cfg1``: the latents handed to ``decode_video`` at cfg_scale 5 and 1, two steps each,
    and ``noise``, the initial latents.

usage:  python tests/golden/make_golden_replace_anyone.py [--ref /root/reference]
"""
import argparse
import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from tools import synth, synth_unianimate as SU, synth_replace_anyone as SR  # noqa: E402


class _Bf16Input(torch.nn.Module):
    """The inpaint stem with the input it gets at the pipeline dtype bf16 (see the module docstring)."""

    def __init__(self, stem):
        super().__init__()
        self.stem = stem

    def forward(self, x):
        return self.stem(x.to(torch.bfloat16))


def run(wv, dit_mod, cfg_scale):
    from make_golden_unianimate import _FakeManager
    R = SR.REPLACE
    H, W, nf = R["H"], R["W"], R["num_frames"]
    h, w, f = H // 8, W // 8, (nf - 1) // 4 + 1
    cfg = SR.CFG_5120
    dit = dit_mod.WanModel(**cfg).eval()
    dit.load_state_dict(synth.make_dit_state_dict(cfg, seed=3), strict=True)
    new_module = {"pipe.dwpose_embedding." + k: v for k, v in SU.pose_stem_sd(cfg["dim"], seed=7).items()}
    new_module.update({"pipe.randomref_embedding_pose." + k: v for k, v in SU.ref_stem_sd(seed=8).items()})
    new_module.update({"pipe.learn_in_embedding." + k: v for k, v in SR.learn_in_sd(seed=20).items()})
    new_module.update({"pipe.inpaint_embedding." + k: v for k, v in SR.inpaint_sd(seed=21).items()})
    pipe = wv.WanRepalceAnyoneVideoPipeline(device="cpu", torch_dtype=torch.float32)
    pipe.fetch_models(_FakeManager({"wan_video_dit": dit, "wan_video_vae": object(), "wan_video_image_encoder": object()},
                                   new_module))
    f32_stems = copy.deepcopy(pipe.learn_in_embedding), copy.deepcopy(pipe.inpaint_embedding)
    pipe.inpaint_embedding = _Bf16Input(pipe.inpaint_embedding)
    pos, neg, clip, y = SU.conditioning(cfg, f, h, w, R["ctx_len"], seed=9)
    pipe.encode_prompt = lambda prompt, positive=True: {"context": pos if positive else neg}
    pipe.encode_image = lambda image, num_frames, height, width: {"clip_feature": clip, "y": y.clone()}
    rec = {}

    def encode_video(input_video, **kw):
        rec["vae_input"] = input_video.clone()
        return SR.masked_latents(f, h, w, seed=22)

    def decode(latents, **kw):
        rec["latents"] = latents.clone()
        return torch.zeros(1, 3, nf, H, W)
    pipe.encode_video, pipe.decode_video = encode_video, decode
    stems = {"learn_in": pipe.learn_in_embedding, "inpaint": pipe.inpaint_embedding.stem}
    for name, m in stems.items():
        m.register_forward_hook(lambda mod, inp, out, name=name: rec.update({name + "_in": inp[0].clone(),
                                                                            name + "_out": out.clone()}))
    batch = {"video": SR.video(nf, H, W, seed=30), "segmentation_data": SR.segmentation(nf, H, W, seed=31)}
    with torch.no_grad():
        pipe(prompt="p", negative_prompt="n", input_image=SU.dummy_image(H, W), seed=R["seed"], height=H, width=W,
             num_frames=nf, cfg_scale=cfg_scale, num_inference_steps=R["steps"], tiled=False,
             progress_bar_cmd=lambda x: x, dwpose_data=SU.pose_video(nf, H, W, seed=10),
             random_ref_dwpose=SU.ref_pose(H, W, seed=11), batch=batch)
        assert rec["learn_in_out"].dtype == rec["inpaint_out"].dtype == torch.bfloat16
        rec["learn_in_f32"] = f32_stems[0](rec["learn_in_in"].float())
        rec["inpaint_f32"] = f32_stems[1](rec["inpaint_in"].float())
    noise = pipe.generate_noise((1, 16, f, h, w), seed=R["seed"], device="cpu", dtype=torch.float32)
    print(f"cfg {cfg_scale}: latents {tuple(rec['latents'].shape)} std {rec['latents'].std().item():.4f}")
    return rec, noise


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    from make_golden_unianimate import load_reference_pipeline
    wv, dit_mod = load_reference_pipeline(a.ref)
    r5, noise = run(wv, dit_mod, 5.0)
    r1, _ = run(wv, dit_mod, 1.0)
    res = {"vae_input": r5["vae_input"], "learn_in_bf16": r5["learn_in_out"].float(),
           "inpaint_bf16": r5["inpaint_out"].float(), "learn_in_f32": r5["learn_in_f32"],
           "inpaint_f32": r5["inpaint_f32"], "latents_cfg5": r5["latents"], "latents_cfg1": r1["latents"], "noise": noise}
    np.savez_compressed(os.path.join(HERE, "replace_anyone_tiny.npz"), **{k: v.numpy() for k, v in res.items()})
    print("wrote replace_anyone_tiny.npz:", len(res), "arrays")
