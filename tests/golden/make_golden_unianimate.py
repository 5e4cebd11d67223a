"""Golden vectors of the UniAnimate-DiT pipelines from the REAL reference module (pipelines/wan_video.py) on the CPU.

Runs only where the reference tree exists; its output, ``tests/golden/unianimate_tiny.npz``, is committed and pins
``oracle/unianimate_oracle.py``.  The reference pipeline module is loaded by file path inside bare ``diffsynth``
packages that point into the reference tree (the recipe of make_golden.py); the modules it imports but this run does
not exercise (prompters, VRAM management, the model manager) are stubs.  Nothing is copied from it.

The fixture holds:
  * ``context_scheduler`` window lists over a grid of (frames, size, overlap), at context_stride 1 and 3;
  * the reference's own ``randomref_embedding_pose`` (built by its ``fetch_models``) on seeded weights;
  * the latents ``WanUniAnimateLongVideoPipeline.__call__`` hands to ``decode_video``, in fp32 on a one-layer
    5120-wide DiT (tools/synth_unianimate.py), with the text, image and VAE encoders replaced by fixed tensors, and the
    carries' initial noise it drew.

usage:  python tests/golden/make_golden_unianimate.py [--ref /root/reference]
"""
import argparse
import importlib
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from tools import synth, synth_unianimate as SU  # noqa: E402

SCHED_FRAMES = (5, 9, 13, 20, 21, 22, 30, 41, 60)
SCHED_SIZES = (5, 8, 21)
SCHED_OVERLAPS = (2, 3, 4)


def load_reference_pipeline(ref_root):
    import make_golden
    dit_mod, _, fm = make_golden.import_reference(ref_root)

    def stub(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    class _Any:
        def __init__(self, *a, **k):
            pass

    sys.modules["diffsynth.models"].ModelManager = _Any
    stub("diffsynth.prompters", WanPrompter=_Any)
    stub("diffsynth.vram_management", enable_vram_management=_Any, AutoWrappedModule=_Any, AutoWrappedLinear=_Any)
    pk = types.ModuleType("diffsynth.pipelines")
    pk.__path__ = [os.path.join(ref_root, "diffsynth", "pipelines")]
    sys.modules["diffsynth.pipelines"] = pk
    for name in ("wan_video_text_encoder", "wan_video_image_encoder"):
        importlib.import_module("diffsynth.models." + name)
    path = os.path.join(ref_root, "diffsynth", "pipelines", "wan_video.py")
    spec = importlib.util.spec_from_file_location("diffsynth.pipelines.wan_video", path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod, dit_mod


class _FakeManager:
    """What the reference fetch_models reads: fetch_model and state_dict_new_module."""

    def __init__(self, models, new_module):
        self.models, self.state_dict_new_module = models, new_module

    def fetch_model(self, name, require_model_path=False):
        return self.models.get(name)


def golden_schedule(wv):
    res = {}
    for stride in (1, 3):
        for n in SCHED_FRAMES:
            for size in SCHED_SIZES:
                for ov in SCHED_OVERLAPS:
                    q = list(wv.context_scheduler(0, 31, n, context_size=size, context_stride=stride, context_overlap=ov))
                    res[f"sched_{stride}_{n}_{size}_{ov}"] = np.array(q, dtype=np.int64)
    return res


def golden_long(wv, dit_mod):
    L = SU.LONG
    H, W, nf, cs = L["H"], L["W"], L["num_frames"], L["context_size"]
    h, w = H // 8, W // 8
    cfg = SU.CFG_5120
    dit = dit_mod.WanModel(**cfg).eval()
    dit.load_state_dict(synth.make_dit_state_dict(cfg, seed=3), strict=True)
    new_module = {"pipe.dwpose_embedding." + k: v for k, v in SU.pose_stem_sd(cfg["dim"], seed=7).items()}
    new_module.update({"pipe.randomref_embedding_pose." + k: v for k, v in SU.ref_stem_sd(seed=8).items()})
    pipe = wv.WanUniAnimateLongVideoPipeline(device="cpu", torch_dtype=torch.float32)
    pipe.fetch_models(_FakeManager({"wan_video_dit": dit, "wan_video_vae": object(), "wan_video_image_encoder": object()},
                                   new_module))
    pos, neg, clip, y = SU.conditioning(cfg, cs, h, w, L["ctx_len"], seed=9)
    pipe.encode_prompt = lambda prompt, positive=True: {"context": pos if positive else neg}
    pipe.encode_image = lambda image, num_frames, height, width: {"clip_feature": clip, "y": y.clone()}
    captured = {}

    def decode(latents, **kw):
        captured["latents"] = latents.clone()
        return torch.zeros(1, 3, nf, H, W)
    pipe.decode_video = decode
    draws = []
    randn_like = torch.randn_like

    def recording_randn_like(t, *a, **k):
        r = randn_like(t, *a, **k)
        draws.append(r.clone())
        return r
    pose = SU.pose_video(nf, H, W, seed=10)
    ref = SU.ref_pose(H, W, seed=11)
    torch.manual_seed(1234)
    torch.randn_like = recording_randn_like
    try:
        with torch.no_grad():
            pipe(prompt="p", negative_prompt="n", input_image=SU.dummy_image(H, W), seed=L["seed"], height=H, width=W,
                 num_frames=nf, cfg_scale=L["cfg_scale"], num_inference_steps=L["steps"], tiled=False,
                 progress_bar_cmd=lambda x: x, dwpose_data=pose, random_ref_dwpose=ref, context_size=cs,
                 context_overlap=L["context_overlap"])
    finally:
        torch.randn_like = randn_like
    with torch.no_grad():
        stem = pipe.randomref_embedding_pose((ref.unsqueeze(0) / 255.).permute(0, 3, 1, 2)).unsqueeze(2)
    noise = pipe.generate_noise((1, 16, (nf - 1) // 4 + 1, h, w), seed=L["seed"], device="cpu", dtype=torch.float32)
    print("long: latents", tuple(captured["latents"].shape), "std", captured["latents"].std().item(), "carries", len(draws))
    return {"long_latents": captured["latents"].numpy(), "long_carries": torch.cat(draws, dim=0).numpy(),
            "long_noise": noise.numpy(), "ref_stem_out": stem.numpy()}


def golden_ref_stem(wv):
    """The stem alone at a size whose sides are multiples of 16 but not of 32."""
    pipe = wv.WanUniAnimateLongVideoPipeline(device="cpu", torch_dtype=torch.float32)
    new_module = {"pipe.dwpose_embedding." + k: v for k, v in SU.pose_stem_sd(5120, seed=7).items()}
    new_module.update({"pipe.randomref_embedding_pose." + k: v for k, v in SU.ref_stem_sd(seed=12).items()})
    pipe.fetch_models(_FakeManager({}, new_module))
    img = SU.ref_pose(80, 112, seed=13)
    with torch.no_grad():
        out = pipe.randomref_embedding_pose((img.unsqueeze(0) / 255.).permute(0, 3, 1, 2)).unsqueeze(2)
    return {"stem_out_80x112": out.numpy()}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    wv, dit_mod = load_reference_pipeline(a.ref)
    res = golden_schedule(wv)
    res.update(golden_ref_stem(wv))
    res.update(golden_long(wv, dit_mod))
    np.savez_compressed(os.path.join(HERE, "unianimate_tiny.npz"), **res)
    print("wrote unianimate_tiny.npz:", len(res), "arrays")
