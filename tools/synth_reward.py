"""Seeded weights, tokenizer files and configs for the cross-attention scorers (ImageReward, MPS) of
diffsynth.extensions.ImageQualityMetric.

* ImageReward: a BLIP ViT + BERT-with-cross-attention + reward MLP state dict in the checkpoint's key names (plus the
  ``blip.vision_proj`` / ``blip.text_proj`` / ``position_ids`` keys the scorer skips), BERT's ``med_config`` JSON and a
  BertTokenizer directory whose ``vocab.txt`` is built from a fixed word list.
* MPS: a transformers CLIPModel + cross model state dict (``model.*``, ``cross_model.*``) and the ``clip`` directory
  (config, processor, tokenizer with ``model_max_length`` 77).
Tiny sizes keep the real head widths (64; 80 in the CLIP vision tower) and the real sequence lengths (197 BLIP image
rows, 35 BERT tokens, 257 MPS image rows at full size).  Weights are N(0, 1/fan_in) with small biases and LayerNorm gains
near 1.
"""
import json
import os

import numpy as np
import torch

from tools import synth_quality as SQ

PROMPTS = ["a photo of a cat", " ".join(["beautiful landscape with mountains and rivers"] * 8),
           "The DOG runs in the park at night!", ""]
SIZES = [(240, 320), (300, 224), (224, 224), (97, 120)]


def med_config(vocab, hidden=768, layers=12, heads=12, inter=3072, max_pos=512):
    return {"architectures": ["BertModel"], "attention_probs_dropout_prob": 0.1, "hidden_act": "gelu",
            "hidden_dropout_prob": 0.1, "hidden_size": hidden, "initializer_range": 0.02, "intermediate_size": inter,
            "layer_norm_eps": 1e-12, "max_position_embeddings": max_pos, "model_type": "bert",
            "num_attention_heads": heads, "num_hidden_layers": layers, "pad_token_id": 0, "type_vocab_size": 2,
            "vocab_size": vocab, "encoder_width": 768, "add_cross_attention": True}


TINY_VISION = dict(image_size=224, patch=16, width=192, layers=2, mlp_width=384)
FULL_VISION = dict(image_size=224, patch=16, width=1024, layers=24, mlp_width=4096)
FULL_MED = med_config(30524)


def tiny_med(vocab):
    return med_config(vocab, hidden=128, layers=2, heads=2, inter=256, max_pos=40)


def _seeded(model, seed, skip=()):
    """N(0, 1/fan_in) matrices, LayerNorm gains 1 + 0.1 N, small biases, embeddings 0.5 N, in the model's key names"""
    g = torch.Generator().manual_seed(seed)
    norms = {n for n, m in model.named_modules() if isinstance(m, torch.nn.LayerNorm) or type(m).__name__ == "BiasFreeLayerNorm"}
    sd = {}
    for name, t in model.state_dict().items():
        owner, leaf = name.rsplit(".", 1) if "." in name else ("", name)
        shape = tuple(t.shape)
        if any(name.startswith(s) for s in skip):
            continue
        if owner in norms:
            sd[name] = 1.0 + 0.1 * torch.randn(shape, generator=g) if leaf == "weight" else 0.02 * torch.randn(shape, generator=g)
            if type(model.get_submodule(owner)).__name__ == "BiasFreeLayerNorm" and leaf == "bias":
                sd[name] = torch.zeros(shape)
        elif name.endswith("logit_scale"):
            sd[name] = torch.tensor(4.6052)
        elif len(shape) == 1:
            sd[name] = 0.02 * torch.randn(shape, generator=g)
        elif "embed" in name or "cls_token" in name:
            sd[name] = 0.5 * torch.randn(shape, generator=g)
        else:
            sd[name] = torch.randn(shape, generator=g) / int(np.prod(shape[1:])) ** 0.5
    return sd


def imagereward_state_dict(med, vision, seed=0, extra=True):
    """the ImageReward checkpoint's tensors; extra: also the keys the scorer skips by name"""
    from diffsynth.extensions.ImageQualityMetric.reward import ImageRewardModel
    with torch.device("meta"):
        shapes = ImageRewardModel(med, **vision)
    sd = _seeded(shapes, seed)
    if extra:
        g = torch.Generator().manual_seed(seed + 1000)
        d, w = med["hidden_size"], vision["width"]
        sd |= {"blip.vision_proj.weight": torch.randn(256, w, generator=g), "blip.vision_proj.bias": torch.zeros(256),
               "blip.text_proj.weight": torch.randn(256, d, generator=g), "blip.text_proj.bias": torch.zeros(256),
               "blip.text_encoder.embeddings.position_ids": torch.arange(med["max_position_embeddings"])[None]}
    return sd


def cross_state_dict(dim, heads, layers, seed=0, prefix="cross_model.", ff_mult=4):
    from diffsynth.extensions.ImageQualityMetric.reward import CrossModel
    m = CrossModel(dim, heads, 64, dim * ff_mult, layers)
    sd = {prefix + k: v for k, v in _seeded(m, seed).items()}
    inv_freq = 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))
    for i in range(layers):                     # the reference's persistent RotaryEmbedding buffer, skipped by the scorer
        sd[f"{prefix}layers.{i}.1.fn.rotary_emb.inv_freq"] = inv_freq.clone()
    return sd


def mps_state_dict(clip_conf, layers, seed=0):
    heads = max(clip_conf["projection_dim"] // 64, 2)           # the reference's 16 at dim 1024
    sd = {"model." + k: v for k, v in SQ.hf_state_dict(clip_conf, seed=seed).items()}
    return sd | cross_state_dict(clip_conf["projection_dim"], heads, layers, seed=seed + 1)


# ------------------------------------------------------------------------------------------------------ files
BERT_WORDS = sorted(set(SQ.CORPUS) | {"dog", "cat", "photo", "runs", "park", "night", "the", "a", "!", ",", ".", "'"})
BERT_PIECES = ["##s", "##ing", "##ed", "##y", "##er", "##ly", "##a", "##e", "##o", "##t"]


def write_bert_dir(path):
    """a BertTokenizer directory (uncased) whose vocab.txt holds BERT's specials, the corpus words and a few word
    pieces; returns the vocabulary size"""
    from transformers import BertTokenizer
    os.makedirs(path, exist_ok=True)
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + BERT_WORDS + BERT_PIECES + list("abcdefghijklmnopqrstuvwxyz")
    vocab = list(dict.fromkeys(vocab))
    with open(os.path.join(path, "vocab.txt"), "w") as f:
        f.write("\n".join(vocab) + "\n")
    BertTokenizer(os.path.join(path, "vocab.txt"), do_lower_case=True).save_pretrained(path)
    return len(vocab)


def write_clip_dir(path, merges, config):
    """the MPS ``clip`` directory: CLIPModel config.json, processor and tokenizer (model_max_length 77)"""
    from transformers import AutoTokenizer
    SQ.write_hf_dir(path, merges, image_size=config["vision_config"]["image_size"])
    tok = AutoTokenizer.from_pretrained(path)
    tok.model_max_length = 77
    tok.save_pretrained(path)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(config, f)
    return path


def mps_tiny_clip(vocab):
    return SQ.hf_tiny_pick(vocab)          # ViT-H-like head width 80, projection 64 = the cross model's width


def write_reward_checkpoints(d):
    """tiny ImageReward and MPS checkpoints under d -> (path dict in the reference's keys, {name: (config, state dict)});
    the keys are the ones tools.synth_quality.write_tiny_checkpoints does not write"""
    from safetensors.torch import save_file
    os.makedirs(d, exist_ok=True)
    paths = {"bert_model_path": os.path.join(d, "bert-base-uncased")}
    V = write_bert_dir(paths["bert_model_path"]) + 2          # + [DEC], [ENC]
    med = tiny_med(V)
    paths["med_config"] = os.path.join(d, "med_config.json")
    with open(paths["med_config"], "w") as f:
        json.dump(med, f)
    ir = imagereward_state_dict(med, TINY_VISION, seed=31)
    paths["imagereward"] = os.path.join(d, "ImageReward.safetensors")
    save_file({k: v.contiguous() for k, v in ir.items()}, paths["imagereward"])
    merges = SQ.learn_merges()
    conf = mps_tiny_clip(SQ.bpe_vocab_size(merges))
    paths["clip"] = write_clip_dir(os.path.join(d, "clip"), merges, conf)
    mps = mps_state_dict(conf, layers=2, seed=41)
    paths["mps"] = os.path.join(d, "mps.safetensors")
    save_file({k: v.contiguous() for k, v in mps.items()}, paths["mps"])
    return paths, {"imagereward": (med, ir), "mps": (conf, mps)}


def frames():
    return [SQ.frames(1, h, w, seed=10 + i)[0] for i, (h, w) in enumerate(SIZES)]
