"""Seeded weights, tokenizer files and frames for the quality-metric scorers (diffsynth.extensions.ImageQualityMetric).

* state dicts of open_clip ``CLIP``, transformers ``CLIPModel`` and the aesthetic MLP, in the checkpoints' key names, at
  tiny size and at the real sizes (open_clip ViT-H-14; CLIPModel ViT-H/14 as PickScore, ViT-L/14 as the aesthetic CLIP).
  Tiny configs keep the real head widths (80 for the ViT-H vision tower, 64 elsewhere), so the real kernel
  instantiations run.  Weights are N(0, 1/fan_in) with small biases and LayerNorm gains near 1.
* a small byte-level BPE merges file (``bpe_simple_vocab``-format, gzip) learnt from a fixed word list, and the same
  vocabulary as a transformers CLIPTokenizer + CLIPImageProcessor directory.
"""
import gzip
import json
import os
from collections import Counter

import numpy as np
import torch



def openclip_tiny(vocab):
    return dict(embed_dim=64, vision_cfg=dict(image_size=56, patch_size=14, width=160, layers=2, head_width=80),
                text_cfg=dict(context_length=77, vocab_size=vocab, width=128, heads=2, layers=2))


OPENCLIP_FULL = dict(embed_dim=1024, vision_cfg=dict(image_size=224, layers=32, width=1280, head_width=80, patch_size=14),
                     text_cfg=dict(context_length=77, vocab_size=49408, width=1024, heads=16, layers=24))


def hf_config(vision, text, projection_dim, eos_token_id=2):
    return {"architectures": ["CLIPModel"], "model_type": "clip", "projection_dim": projection_dim,
            "logit_scale_init_value": 2.6592,
            "vision_config": dict(vision, model_type="clip_vision_model", num_channels=3, layer_norm_eps=1e-5),
            "text_config": dict(text, model_type="clip_text_model", layer_norm_eps=1e-5, eos_token_id=eos_token_id,
                                bos_token_id=0, pad_token_id=1)}


def _v(hidden, layers, heads, inter, image, patch, act):
    return dict(hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads, intermediate_size=inter,
                image_size=image, patch_size=patch, hidden_act=act)


def _t(hidden, layers, heads, inter, vocab, act):
    return dict(hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads, intermediate_size=inter,
                vocab_size=vocab, max_position_embeddings=77, hidden_act=act)


def hf_tiny_pick(vocab):
    return hf_config(_v(160, 2, 2, 320, 56, 14, "gelu"), _t(128, 2, 2, 256, vocab, "gelu"), 64)


def hf_tiny_large(vocab):
    """ViT-L/14-like: quick-GELU, head width 64; projection 768 as the aesthetic head needs"""
    return hf_config(_v(128, 2, 2, 256, 56, 14, "quick_gelu"), _t(128, 2, 2, 256, vocab, "quick_gelu"), 768)


HF_FULL_PICK = hf_config(_v(1280, 32, 16, 5120, 224, 14, "gelu"), _t(1024, 24, 16, 4096, 49408, "gelu"), 1024)
HF_FULL_LARGE = hf_config(_v(1024, 24, 16, 4096, 224, 14, "quick_gelu"), _t(768, 12, 12, 3072, 49408, "quick_gelu"), 768)


def _fill(shapes, seed):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in shapes.items():
        if name.endswith("logit_scale"):
            sd[name] = torch.tensor(4.6052)
        elif len(shape) == 1 and ("ln" in name or "norm" in name or "layrnorm" in name) and name.endswith("weight"):
            sd[name] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif len(shape) == 1:
            sd[name] = 0.02 * torch.randn(shape, generator=g)
        elif "embedding" in name or "positional" in name:
            sd[name] = 0.5 * torch.randn(shape, generator=g)
        else:
            fan_in = int(np.prod(shape[1:]))
            if name.endswith("proj") or name.endswith("projection"):     # open_clip stores [in, out]
                fan_in = shape[0]
            sd[name] = torch.randn(shape, generator=g) / fan_in ** 0.5
    return sd


def openclip_state_dict(cfg, seed=0):
    from diffsynth.extensions.ImageQualityMetric.towers import OpenCLIP
    m = OpenCLIP(**cfg)
    return _fill({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed)


def hf_state_dict(config, seed=0):
    from diffsynth.extensions.ImageQualityMetric.towers import HFCLIPModel
    m = HFCLIPModel(config)
    return _fill({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed)


def aesthetic_state_dict(seed=0):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i, (o, n) in zip((0, 2, 4, 6, 7), ((1024, 768), (128, 1024), (64, 128), (16, 64), (1, 16))):
        sd[f"layers.{i}.weight"] = torch.randn(o, n, generator=g) / n ** 0.5
        sd[f"layers.{i}.bias"] = 0.1 * torch.randn(o, generator=g)
    return sd


def weight_checksum(sd):
    """sum over tensors (sorted by name) of sum(w) + 1e-3 * sum(w^2), in fp64"""
    return float(sum(v.double().sum() + 1e-3 * (v.double() ** 2).sum() for _, v in sorted(sd.items())))


# ------------------------------------------------------------------------------------------------------ tokenizers
CORPUS = ("a photo of a cat sitting on the table next to the window the dog runs in the park at night "
          "beautiful landscape with mountains and rivers high quality cinematic lighting portrait of a woman "
          "smiling man walking through the city street rain reflections neon lights video frame").split()


def _byte_symbols():
    from diffsynth.extensions.ImageQualityMetric.tokenizer import byte_symbols
    return byte_symbols()


def learn_merges(n_merges=160):
    """BPE merges learnt greedily from CORPUS (most frequent adjacent pair first, ties by the pair)"""
    words = Counter(tuple(w[:-1]) + (w[-1] + "</w>",) for w in CORPUS)
    merges = []
    while len(merges) < n_merges:
        pairs = Counter()
        for w, c in words.items():
            for p in zip(w, w[1:]):
                pairs[p] += c
        if not pairs:
            break
        best = max(pairs.items(), key=lambda kv: (kv[1], kv[0]))[0]
        merges.append(best)
        new = Counter()
        for w, c in words.items():
            out, i = [], 0
            while i < len(w):
                if i + 1 < len(w) and (w[i], w[i + 1]) == best:
                    out.append(w[i] + w[i + 1])
                    i += 2
                else:
                    out.append(w[i])
                    i += 1
            new[tuple(out)] += c
        words = new
    return merges


def write_bpe(path, merges):
    with gzip.open(path, "wt", encoding="utf-8") as f:
        f.write("#version: synthetic\n" + "\n".join(f"{a} {b}" for a, b in merges))     # no trailing empty line
    return path


def bpe_vocab_size(merges):
    return 512 + len(merges) + 2


def write_hf_dir(path, merges, image_size=56):
    """CLIPTokenizer + CLIPImageProcessor files for the same vocabulary (HF names its specials <|startoftext|>,
    <|endoftext|>)"""
    from transformers import CLIPImageProcessor, CLIPProcessor, CLIPTokenizer
    os.makedirs(path, exist_ok=True)
    sym = list(_byte_symbols().values())
    vocab = sym + [s + "</w>" for s in sym] + ["".join(m) for m in merges] + ["<|startoftext|>", "<|endoftext|>"]
    with open(os.path.join(path, "vocab.json"), "w") as f:
        json.dump({s: i for i, s in enumerate(vocab)}, f)
    with open(os.path.join(path, "merges.txt"), "w", encoding="utf-8") as f:
        f.write("#version: 0.2\n" + "".join(f"{a} {b}\n" for a, b in merges))
    tok = CLIPTokenizer(vocab={s: i for i, s in enumerate(vocab)}, merges=[tuple(m) for m in merges])
    ip = CLIPImageProcessor(size={"shortest_edge": image_size}, crop_size={"height": image_size, "width": image_size})
    CLIPProcessor(image_processor=ip, tokenizer=tok).save_pretrained(path)
    return path


def write_hf_model(path, config, sd):
    from safetensors.torch import save_file
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(config, f)
    save_file({k: v.contiguous() for k, v in sd.items()}, os.path.join(path, "model.safetensors"))
    return path


PROMPTS = ["a photo of a cat", "A DOG, running... in the park!!", "café naïve — 東京 🙂 2024", "",
           " ".join(["beautiful landscape with mountains"] * 30), "it's   the dog's\tnight"]


def frames(n, h, w, seed=0):
    """n smooth RGB PIL frames"""
    from PIL import Image
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w] / max(h, w)
    out = []
    for _ in range(n):
        a = g.uniform(0, 6, size=(3, 3))
        img = np.stack([0.5 + 0.45 * np.sin(a[c, 0] * xx + a[c, 1] * yy + a[c, 2]) for c in range(3)], -1)
        img = img + 0.05 * g.standard_normal(img.shape)
        out.append(Image.fromarray((np.clip(img, 0, 1) * 255).astype(np.uint8)))
    return out


def write_tiny_checkpoints(d):
    """every tiny checkpoint the five load_preference_model names read, under d -> (path dict in the reference's keys,
    {name: (config, state dict)})"""
    import safetensors.torch as st
    os.makedirs(d, exist_ok=True)
    merges = learn_merges()
    V = bpe_vocab_size(merges)
    oc_cfg = openclip_tiny(V)
    ref = {"open_clip": (oc_cfg, openclip_state_dict(oc_cfg, seed=1)), "hpsv2": (oc_cfg, openclip_state_dict(oc_cfg, seed=5)),
           "hpsv2.1": (oc_cfg, openclip_state_dict(oc_cfg, seed=6)), "pickscore": (hf_tiny_pick(V), hf_state_dict(hf_tiny_pick(V), seed=2)),
           "clip-large": (hf_tiny_large(V), hf_state_dict(hf_tiny_large(V), seed=3)), "aesthetic_predictor": (None, aesthetic_state_dict(seed=4))}
    paths = {"open_clip_bpe": write_bpe(os.path.join(d, "bpe_simple_vocab_16e6.txt.gz"), merges)}
    paths["open_clip"] = os.path.join(d, "open_clip_pytorch_model.bin")
    torch.save(ref["open_clip"][1], paths["open_clip"])
    for k in ("hpsv2", "hpsv2.1"):
        paths[k] = os.path.join(d, f"{k}.safetensors")
        st.save_file(ref[k][1], paths[k])
    paths["aesthetic_predictor"] = os.path.join(d, "aesthetic.safetensors")
    st.save_file(ref["aesthetic_predictor"][1], paths["aesthetic_predictor"])
    paths["clip"] = write_hf_dir(os.path.join(d, "clip"), merges)
    paths["pickscore"] = write_hf_model(os.path.join(d, "pickscore"), *ref["pickscore"])
    paths["clip-large"] = write_hf_model(os.path.join(d, "clip-large"), *ref["clip-large"])
    write_hf_dir(paths["clip-large"], merges)
    return paths, {"oc_config": oc_cfg, **ref}


_LOADED = {}


def _once(key, make):
    if key not in _LOADED:
        _LOADED[key] = make()
    return _LOADED[key]


def oracle_scores(name, paths, ref, images, prompt, device="cpu"):
    """the fp32 oracle's scores of one load_preference_model name, preprocessing and tokenising as the scorers do
    (tokenizer and processor are loaded once per path)"""
    from transformers import AutoProcessor

    from diffsynth.extensions.ImageQualityMetric import SimpleTokenizer
    from diffsynth.extensions.ImageQualityMetric import towers as T
    from oracle import quality_oracle as O
    if name in ("CLIP", "HPSv2", "HPSv2.1"):
        cfg, sd = ref[{"CLIP": "open_clip", "HPSv2": "hpsv2", "HPSv2.1": "hpsv2.1"}[name]]
        px = O.normalize(torch.stack([T.openclip_pixels(im, cfg["vision_cfg"]["image_size"]) for im in images]).to(device))
        ids = _once(paths["open_clip_bpe"], lambda: SimpleTokenizer(paths["open_clip_bpe"]))([prompt]).to(device)
        return O.cosine(O.openclip_image(sd, cfg, px), O.openclip_text(sd, cfg, ids))[:, 0].tolist()
    key = "pickscore" if name == "PickScore" else "clip-large"
    pdir = paths["clip" if name == "PickScore" else "clip-large"]
    proc = _once(pdir, lambda: AutoProcessor.from_pretrained(pdir))
    conf, sd = ref[key]
    px = O.normalize(torch.stack([T.hf_pixels(proc, im) for im in images]).to(device), *T.hf_mean_std(proc))
    img = O.hf_image(sd, conf, px)
    if name == "Aesthetic":
        return O.aesthetic(ref["aesthetic_predictor"][1], img).tolist()
    ids = proc(text=prompt, padding=True, truncation=True, max_length=77, return_tensors="pt")["input_ids"].to(device)
    return O.cosine(img, O.hf_text(sd, conf, ids))[:, 0].tolist()
