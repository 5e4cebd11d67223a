"""Regenerate tests/golden/quality_tiny.npz from the REAL reference modules (run on a machine with the reference tree):

    python tests/golden/make_golden_quality.py /path/to/reference

* the vendored open_clip (loaded by path, so the ImageQualityMetric package __init__, which imports modelscope, does not
  run; ftfy stubbed as the identity): SimpleTokenizer on the synthetic merges file, image_transform(resize_longest_max=
  True) as preprocess_val with light_augmentation, and a CLIP built from the tiny config with the seeded weights;
* transformers CLIPModel / AutoProcessor (as the reference's PickScore and AestheticScore use them) on tiny configs;
* the reference aesthetic MLP.
The reference classes' score() cannot be pointed at tiny weights (CLIPScore / HPScore_v2 hard-code "ViT-H-14"), and with
the installed transformers get_image_features returns an output object, so scores are computed as their score() does
from the features.  Records token ids, preprocessed pixels (odd aspect ratios), tower features and scores.
"""
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stable-video-infinity_b200")]
from tools import synth_quality as S  # noqa: E402

SIZES = [(40, 70), (71, 33), (56, 56), (97, 120)]


def load_open_clip(ref):
    sys.modules["ftfy"] = types.SimpleNamespace(fix_text=lambda s: s)
    root = os.path.join(ref, "diffsynth", "extensions", "ImageQualityMetric", "open_clip")
    spec = importlib.util.spec_from_file_location("ref_open_clip", os.path.join(root, "__init__.py"),
                                                  submodule_search_locations=[root])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["ref_open_clip"] = mod
    spec.loader.exec_module(mod)
    return mod


def load_aesthetic_mlp(ref):
    src = open(os.path.join(ref, "diffsynth", "extensions", "ImageQualityMetric", "aesthetic.py")).read()
    ns = {}
    exec(src.split("class AestheticScore")[0].replace("from .config import MODEL_PATHS", ""), ns)
    return ns["MLP"]


def main(ref):
    oc = load_open_clip(ref)
    from transformers import AutoProcessor, CLIPConfig, CLIPModel
    torch.manual_seed(0)
    out = {}
    d = tempfile.mkdtemp()
    merges = S.learn_merges()
    V = S.bpe_vocab_size(merges)
    tok = oc.SimpleTokenizer(S.write_bpe(os.path.join(d, "bpe.txt.gz"), merges))
    out["openclip_ids"] = tok(S.PROMPTS, context_length=77).numpy()
    frames = [S.frames(1, h, w, seed=i)[0] for i, (h, w) in enumerate(SIZES)]
    tf = oc.image_transform(56, is_train=False, mean=(0.0, 0.0, 0.0), std=(1.0, 1.0, 1.0), resize_longest_max=True)
    out["openclip_pixels"] = torch.stack([tf(f) for f in frames]).numpy()       # preprocess_val without the normalisation
    tf_norm = oc.image_transform(56, is_train=False, resize_longest_max=True)
    px = torch.stack([tf_norm(f) for f in frames])
    cfg = S.openclip_tiny(V)
    model = oc.CLIP(cfg["embed_dim"], oc.CLIPVisionCfg(**cfg["vision_cfg"]), oc.CLIPTextCfg(**cfg["text_cfg"]), output_dict=True)
    model.load_state_dict(S.openclip_state_dict(cfg, seed=1), strict=True)
    model.eval()
    with torch.no_grad():
        ids = torch.from_numpy(out["openclip_ids"])
        o = model(px, ids[:1])
        out["openclip_image_features"] = model.encode_image(px).numpy()
        out["openclip_text_features"] = model.encode_text(ids).numpy()
        out["openclip_scores"] = (o["image_features"] @ o["text_features"].T)[:, 0].numpy()

    hf_dir = S.write_hf_dir(os.path.join(d, "hf"), merges)
    proc = AutoProcessor.from_pretrained(hf_dir)
    for i, p in enumerate(S.PROMPTS):
        out[f"hf_ids_{i}"] = proc(text=p, padding=True, truncation=True, max_length=77, return_tensors="pt")["input_ids"].numpy()
    out["hf_pixels"] = torch.cat([proc(images=f, return_tensors="pt", do_normalize=False)["pixel_values"] for f in frames]).numpy()
    hpx = torch.cat([proc(images=f, return_tensors="pt")["pixel_values"] for f in frames])
    for name, conf, seed in (("pick", S.hf_tiny_pick(V), 2), ("large", S.hf_tiny_large(V), 3)):
        m = CLIPModel(CLIPConfig.from_dict(conf)).eval()
        sd = S.hf_state_dict(conf, seed=seed)
        m.load_state_dict(sd, strict=True)
        with torch.no_grad():
            img = m.get_image_features(pixel_values=hpx).pooler_output
            t_ids = torch.from_numpy(out["hf_ids_0"])
            txt = m.get_text_features(input_ids=t_ids).pooler_output
        out[f"{name}_image_features"], out[f"{name}_text_features"] = img.numpy(), txt.numpy()
        ie, te = img / img.norm(dim=-1, keepdim=True), txt / txt.norm(dim=-1, keepdim=True)
        out[f"{name}_scores"] = (te @ ie.T)[0].numpy()
    MLP = load_aesthetic_mlp(ref)
    mlp = MLP(768).eval()
    mlp.load_state_dict(S.aesthetic_state_dict(seed=4))
    img = torch.from_numpy(out["large_image_features"])
    with torch.no_grad():
        out["aesthetic_scores"] = mlp(img / img.norm(dim=-1, keepdim=True)).flatten().numpy()
    path = os.path.join(ROOT, "tests", "golden", "quality_tiny.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main(sys.argv[1])
