"""CLIP towers of the quality scorers: parameter containers in both checkpoint formats, host preprocessing, and the
engines that run the towers on the kernel library.

Containers carry the checkpoints' own key names, so real files load with ``strict=True``:

* ``OpenCLIP``: open_clip's ``CLIP`` (``visual.*``, ``transformer.*``, ``token_embedding``, ``positional_embedding``,
  ``ln_final``, ``text_projection``, ``logit_scale``): CLIPScore and HPSv2 / v2.1, ViT-H-14.
* ``HFCLIPModel``: transformers' ``CLIPModel`` (``vision_model.*``, ``text_model.*``, ``visual_projection``,
  ``text_projection``, ``logit_scale``), read from ``config.json`` + ``model.safetensors`` / ``pytorch_model.bin``:
  PickScore (ViT-H/14) and the aesthetic score's CLIP (ViT-L/14, quick-GELU).

Both reduce to one ``TowerSpec`` per tower, which ``TowerEngine`` runs: every matrix product on ``svi_gemm_bf16`` (bias,
GELU(erf) and the f32 residual add in its epilogue), the block LayerNorms on ``svi_layernorm_modulate``, attention,
staging, pooling and quick-GELU on ``include/svi_b200_quality.h``.  A whole batch of images goes through the vision tower
together, in chunks of at most ``chunk`` images to bound device memory.  There is no torch compute fallback.
"""
import json
import math
import os
from dataclasses import dataclass

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from PIL import Image

from ... import _native as nv

OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)
# open_clip's model_configs/ViT-H-14.json
VIT_H_14 = dict(embed_dim=1024,
                vision_cfg=dict(image_size=224, layers=32, width=1280, head_width=80, patch_size=14),
                text_cfg=dict(context_length=77, vocab_size=49408, width=1024, heads=16, layers=24))
HEAD_WIDTHS = (64, 80)
ACTS = ("gelu", "quick_gelu")


def _reject(what, field_name, value, why):
    raise ValueError(f"ImageQualityMetric: unsupported {what} config {field_name}={value!r} ({why})")


def check_tower(what, width, heads, seq_len, mlp_width, act, fields):
    """the shapes the kernels implement; anything else raises ValueError naming the field (fields: the config's names of
    heads, width, sequence length and activation)"""
    if heads < 1 or width % heads or width // heads not in HEAD_WIDTHS:
        _reject(what, fields[0], heads, f"the head width width / heads must be one of {HEAD_WIDTHS}")
    if width % 8 or mlp_width % 8:
        _reject(what, fields[1], width, "the width and the MLP width must be multiples of 8")
    if not 1 <= seq_len <= nv.QUALITY_MAX_L:
        _reject(what, fields[2], seq_len, f"the attention kernel takes 1 .. {nv.QUALITY_MAX_L} tokens")
    if act not in ACTS:
        _reject(what, fields[3], act, f"one of {ACTS}")


# ================================================================================================ containers
class _Block(nn.Module):
    """open_clip ResidualAttentionBlock: ln_1, attn (nn.MultiheadAttention's in_proj / out_proj), ln_2, mlp.c_fc / c_proj."""

    def __init__(self, width, mlp_width, eps=1e-5):
        super().__init__()
        self.ln_1 = nn.LayerNorm(width, eps=eps)
        self.attn = nn.Module()
        self.attn.in_proj_weight = nn.Parameter(torch.empty(3 * width, width))
        self.attn.in_proj_bias = nn.Parameter(torch.empty(3 * width))
        self.attn.out_proj = nn.Linear(width, width)
        self.ln_2 = nn.LayerNorm(width, eps=eps)
        self.mlp = nn.Module()
        self.mlp.c_fc = nn.Linear(width, mlp_width)
        self.mlp.c_proj = nn.Linear(mlp_width, width)


class _Transformer(nn.Module):
    def __init__(self, width, layers, mlp_width):
        super().__init__()
        self.resblocks = nn.ModuleList([_Block(width, mlp_width) for _ in range(layers)])


class _OpenCLIPVisual(nn.Module):
    def __init__(self, image_size, patch_size, width, layers, mlp_width, embed_dim):
        super().__init__()
        grid = image_size // patch_size
        self.conv1 = nn.Conv2d(3, width, patch_size, patch_size, bias=False)
        self.class_embedding = nn.Parameter(torch.empty(width))
        self.positional_embedding = nn.Parameter(torch.empty(grid * grid + 1, width))
        self.ln_pre = nn.LayerNorm(width)
        self.transformer = _Transformer(width, layers, mlp_width)
        self.ln_post = nn.LayerNorm(width)
        self.proj = nn.Parameter(torch.empty(width, embed_dim))


class OpenCLIP(nn.Module):
    """open_clip ``CLIP`` parameters (model.py / transformer.py of open_clip): ViT vision tower with a CLS pool, causal text
    tower pooled at the end-of-text token (the largest id)."""

    def __init__(self, embed_dim=1024, vision_cfg=None, text_cfg=None, quick_gelu=False):
        super().__init__()
        v = dict(image_size=224, patch_size=16, width=768, layers=12, head_width=64, mlp_ratio=4.0) | dict(vision_cfg or {})
        t = dict(context_length=77, vocab_size=49408, width=512, heads=8, layers=12, mlp_ratio=4.0) | dict(text_cfg or {})
        for name, value in v.items():
            if name not in ("image_size", "patch_size", "width", "layers", "head_width", "mlp_ratio"):
                _reject("open_clip vision", f"vision_cfg.{name}", value, "not implemented")
        for name, value in t.items():
            if name not in ("context_length", "vocab_size", "width", "heads", "layers", "mlp_ratio"):
                _reject("open_clip text", f"text_cfg.{name}", value, "not implemented")
        if v["width"] % v["head_width"] or v["head_width"] not in HEAD_WIDTHS:
            _reject("open_clip vision", "vision_cfg.head_width", v["head_width"], f"one of {HEAD_WIDTHS} dividing the width")
        if v["image_size"] % v["patch_size"]:
            _reject("open_clip vision", "vision_cfg.patch_size", v["patch_size"], "must divide image_size")
        act = "quick_gelu" if quick_gelu else "gelu"
        v_mlp, t_mlp = int(v["width"] * v["mlp_ratio"]), int(t["width"] * t["mlp_ratio"])
        check_tower("open_clip vision", v["width"], v["width"] // v["head_width"], (v["image_size"] // v["patch_size"]) ** 2 + 1,
                    v_mlp, act, ("vision_cfg.head_width", "vision_cfg.width", "vision_cfg.image_size", "quick_gelu"))
        check_tower("open_clip text", t["width"], t["heads"], t["context_length"], t_mlp, act,
                    ("text_cfg.heads", "text_cfg.width", "text_cfg.context_length", "quick_gelu"))
        self.embed_dim, self.vision_cfg, self.text_cfg, self.act = embed_dim, v, t, act
        self.visual = _OpenCLIPVisual(v["image_size"], v["patch_size"], v["width"], v["layers"], v_mlp, embed_dim)
        self.transformer = _Transformer(t["width"], t["layers"], t_mlp)
        self.token_embedding = nn.Embedding(t["vocab_size"], t["width"])
        self.positional_embedding = nn.Parameter(torch.empty(t["context_length"], t["width"]))
        self.ln_final = nn.LayerNorm(t["width"])
        self.text_projection = nn.Parameter(torch.empty(t["width"], embed_dim))
        self.logit_scale = nn.Parameter(torch.ones([]) * math.log(1 / 0.07))
        self._engine = None

    def specs(self):
        v, t = self.vision_cfg, self.text_cfg

        def blocks(tr):
            return [dict(ln1=(b.ln_1.weight, b.ln_1.bias), qkv=(b.attn.in_proj_weight, b.attn.in_proj_bias),
                         out=(b.attn.out_proj.weight, b.attn.out_proj.bias), ln2=(b.ln_2.weight, b.ln_2.bias),
                         fc1=(b.mlp.c_fc.weight, b.mlp.c_fc.bias), fc2=(b.mlp.c_proj.weight, b.mlp.c_proj.bias))
                    for b in tr.resblocks]
        vis = self.visual
        vspec = TowerSpec(width=v["width"], heads=v["width"] // v["head_width"], act=self.act, eps=vis.ln_pre.eps,
                          blocks=blocks(vis.transformer), final_ln=(vis.ln_post.weight, vis.ln_post.bias),
                          proj=vis.proj.t(), pos=vis.positional_embedding, causal=False,
                          image_size=v["image_size"], patch=v["patch_size"], patch_weight=vis.conv1.weight,
                          cls=vis.class_embedding, pre_ln=(vis.ln_pre.weight, vis.ln_pre.bias))
        tspec = TowerSpec(width=t["width"], heads=t["heads"], act=self.act, eps=self.ln_final.eps,
                          blocks=blocks(self.transformer), final_ln=(self.ln_final.weight, self.ln_final.bias),
                          proj=self.text_projection.t(), pos=self.positional_embedding, causal=True,
                          token_embedding=self.token_embedding.weight, pool=nv.POOL_ARGMAX)
        return vspec, tspec

    def engine(self, device=None, mean=OPENAI_MEAN, std=OPENAI_STD):
        """the cached CLIPEngines of this model on `device` (the vision tower normalises with mean / std)"""
        return _cached_engine(self, self.visual.conv1.weight, self.transformer.resblocks[-1].mlp.c_proj.weight, device,
                              mean, std)


class _HFAttention(nn.Module):
    def __init__(self, width):
        super().__init__()
        self.k_proj, self.v_proj, self.q_proj, self.out_proj = (nn.Linear(width, width) for _ in range(4))


class _HFLayer(nn.Module):
    def __init__(self, width, mlp_width, eps):
        super().__init__()
        self.self_attn = _HFAttention(width)
        self.layer_norm1 = nn.LayerNorm(width, eps=eps)
        self.mlp = nn.Module()
        self.mlp.fc1 = nn.Linear(width, mlp_width)
        self.mlp.fc2 = nn.Linear(mlp_width, width)
        self.layer_norm2 = nn.LayerNorm(width, eps=eps)


class _HFEncoder(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.layers = nn.ModuleList([_HFLayer(c["hidden_size"], c["intermediate_size"], c["layer_norm_eps"])
                                     for _ in range(c["num_hidden_layers"])])


class HFCLIPModel(nn.Module):
    """transformers ``CLIPModel`` parameters (modeling_clip.py): vision tower with a CLS pool, causal text tower pooled
    at the end-of-sequence token by the rule of the installed transformers (argmax of the ids when eos_token_id == 2,
    else the first eos_token_id)."""

    TEXT_DEFAULTS = dict(vocab_size=49408, hidden_size=512, intermediate_size=2048, num_hidden_layers=12,
                         num_attention_heads=8, max_position_embeddings=77, hidden_act="quick_gelu", layer_norm_eps=1e-5,
                         eos_token_id=2)
    VISION_DEFAULTS = dict(hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                           num_channels=3, image_size=224, patch_size=32, hidden_act="quick_gelu", layer_norm_eps=1e-5)

    def __init__(self, config):
        super().__init__()
        t = {k: config.get("text_config", {}).get(k, d) for k, d in self.TEXT_DEFAULTS.items()}
        v = {k: config.get("vision_config", {}).get(k, d) for k, d in self.VISION_DEFAULTS.items()}
        proj = config.get("projection_dim", 512)
        if v["num_channels"] != 3:
            _reject("CLIPVisionConfig", "vision_config.num_channels", v["num_channels"], "RGB only")
        if v["image_size"] % v["patch_size"]:
            _reject("CLIPVisionConfig", "vision_config.patch_size", v["patch_size"], "must divide image_size")
        for name, c, seq, seq_field in (("vision_config", v, (v["image_size"] // v["patch_size"]) ** 2 + 1, "image_size"),
                                        ("text_config", t, t["max_position_embeddings"], "max_position_embeddings")):
            check_tower("CLIPModel", c["hidden_size"], c["num_attention_heads"], seq, c["intermediate_size"], c["hidden_act"],
                        tuple(f"{name}.{f}" for f in ("num_attention_heads", "hidden_size", seq_field, "hidden_act")))
        self.text_cfg, self.vision_cfg, self.projection_dim = t, v, proj
        grid = v["image_size"] // v["patch_size"]
        W = v["hidden_size"]
        self.vision_model = nn.Module()
        emb = self.vision_model.embeddings = nn.Module()
        emb.class_embedding = nn.Parameter(torch.empty(W))
        emb.patch_embedding = nn.Conv2d(3, W, v["patch_size"], v["patch_size"], bias=False)
        emb.position_embedding = nn.Embedding(grid * grid + 1, W)
        self.vision_model.pre_layrnorm = nn.LayerNorm(W, eps=v["layer_norm_eps"])
        self.vision_model.encoder = _HFEncoder(v)
        self.vision_model.post_layernorm = nn.LayerNorm(W, eps=v["layer_norm_eps"])
        Wt = t["hidden_size"]
        self.text_model = nn.Module()
        temb = self.text_model.embeddings = nn.Module()
        temb.token_embedding = nn.Embedding(t["vocab_size"], Wt)
        temb.position_embedding = nn.Embedding(t["max_position_embeddings"], Wt)
        self.text_model.encoder = _HFEncoder(t)
        self.text_model.final_layer_norm = nn.LayerNorm(Wt, eps=t["layer_norm_eps"])
        self.visual_projection = nn.Linear(W, proj, bias=False)
        self.text_projection = nn.Linear(Wt, proj, bias=False)
        self.logit_scale = nn.Parameter(torch.tensor(2.6592))
        self._engine = None

    @classmethod
    def from_pretrained(cls, path):
        """``config.json`` + ``model.safetensors`` (or ``pytorch_model.bin``) of a CLIPModel directory, loaded strictly.
        ``*.position_ids`` buffers that older checkpoints store are dropped first: they are index tables, not weights."""
        with open(os.path.join(path, "config.json")) as f:
            model = cls(json.load(f))
        st, pt = os.path.join(path, "model.safetensors"), os.path.join(path, "pytorch_model.bin")
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        elif os.path.exists(pt):
            sd = torch.load(pt, map_location="cpu", weights_only=True)
        else:
            raise FileNotFoundError(f"ImageQualityMetric: no model.safetensors or pytorch_model.bin in {path}")
        model.load_state_dict({k: v for k, v in sd.items() if not k.endswith("position_ids")}, strict=True)
        return model.eval()

    def specs(self):
        def blocks(enc):
            out = []
            for ly in enc.layers:
                a = ly.self_attn
                out.append(dict(ln1=(ly.layer_norm1.weight, ly.layer_norm1.bias),
                                qkv=(torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight]),
                                     torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias])),
                                out=(a.out_proj.weight, a.out_proj.bias), ln2=(ly.layer_norm2.weight, ly.layer_norm2.bias),
                                fc1=(ly.mlp.fc1.weight, ly.mlp.fc1.bias), fc2=(ly.mlp.fc2.weight, ly.mlp.fc2.bias)))
            return out
        v, t, vm, tm = self.vision_cfg, self.text_cfg, self.vision_model, self.text_model
        vspec = TowerSpec(width=v["hidden_size"], heads=v["num_attention_heads"], act=v["hidden_act"], eps=v["layer_norm_eps"],
                          blocks=blocks(vm.encoder), final_ln=(vm.post_layernorm.weight, vm.post_layernorm.bias),
                          proj=self.visual_projection.weight, pos=vm.embeddings.position_embedding.weight, causal=False,
                          image_size=v["image_size"], patch=v["patch_size"], patch_weight=vm.embeddings.patch_embedding.weight,
                          cls=vm.embeddings.class_embedding, pre_ln=(vm.pre_layrnorm.weight, vm.pre_layrnorm.bias))
        tspec = TowerSpec(width=t["hidden_size"], heads=t["num_attention_heads"], act=t["hidden_act"], eps=t["layer_norm_eps"],
                          blocks=blocks(tm.encoder), final_ln=(tm.final_layer_norm.weight, tm.final_layer_norm.bias),
                          proj=self.text_projection.weight, pos=tm.embeddings.position_embedding.weight, causal=True,
                          token_embedding=tm.embeddings.token_embedding.weight,
                          pool=nv.POOL_ARGMAX if t["eos_token_id"] == 2 else nv.POOL_EOS, eos_id=t["eos_token_id"])
        return vspec, tspec

    def engine(self, device=None, mean=OPENAI_MEAN, std=OPENAI_STD):
        """the cached CLIPEngines of this model on `device` (the vision tower normalises with mean / std)"""
        return _cached_engine(self, self.vision_model.embeddings.patch_embedding.weight,
                              self.text_model.encoder.layers[-1].mlp.fc2.weight, device, mean, std)


class AestheticMLP(nn.Module):
    """The aesthetic predictor's head (reference aesthetic.py ``MLP``): five Linear layers at ``layers.{0,2,4,6,7}``; the
    ReLUs are commented out in the reference and Dropout is the identity in eval, so the head is one affine map."""

    def __init__(self, input_size=768):
        super().__init__()
        self.layers = nn.Sequential(nn.Linear(input_size, 1024), nn.Dropout(0.2), nn.Linear(1024, 128), nn.Dropout(0.2),
                                    nn.Linear(128, 64), nn.Dropout(0.1), nn.Linear(64, 16), nn.Linear(16, 1))

    def folded(self, shift=0.0, scale=1.0):
        """(w [input_size], b) of (layers(x) - shift) / scale: the five layers and the standardisation composed on the host
        in fp64, rounded once to f32."""
        w = torch.eye(self.layers[0].in_features, dtype=torch.float64)
        b = torch.zeros(self.layers[0].in_features, dtype=torch.float64)
        for i in (0, 2, 4, 6, 7):
            lin = self.layers[i]
            W = lin.weight.detach().double().cpu()
            w, b = W @ w, W @ b + lin.bias.detach().double().cpu()
        return (w[0] / scale).float(), float((b[0] - shift) / scale)


# ================================================================================================ engines
@dataclass
class TowerSpec:
    """one tower in the engine's terms; matrices in nn.Linear's [out, in] layout"""
    width: int
    heads: int
    act: str
    eps: float
    blocks: list
    final_ln: tuple
    proj: torch.Tensor
    pos: torch.Tensor
    causal: bool
    image_size: int = 0
    patch: int = 0
    patch_weight: torch.Tensor = None
    cls: torch.Tensor = None
    pre_ln: tuple = None            # None: no LayerNorm after the position embedding (BLIP's ViT)
    patch_bias: torch.Tensor = None
    token_embedding: torch.Tensor = None
    pool: int = nv.POOL_FIRST
    eos_id: int = 0


class TowerEngine:
    """One CLIP tower on the device.  ``encode_images(px)`` takes preprocessed (un-normalised) f32 [B, 3, S, S] pixels,
    ``encode_text(ids)`` int64 [T, L] token ids; both return the projected f32 features [n, embed_dim], not normalised.
    ``image_states(px)`` is the residual stream after the last block, every row of every image; ``encode_text_rows(ids)``
    projects every row after the final LayerNorm and pools afterwards (the cross-attention scorers use both).  A tower
    without a projection (``proj`` None) has only ``image_states``."""

    def __init__(self, spec, device, mean=OPENAI_MEAN, std=OPENAI_STD, chunk=128):
        nv.require_cuda(device, "the quality-metric towers")
        self.device = torch.device(device)
        bf = lambda t: t.detach().to(device=self.device, dtype=torch.bfloat16).contiguous()
        f32 = lambda t: t.detach().to(device=self.device, dtype=torch.float32).contiguous()
        self.width, self.heads, self.act, self.eps = spec.width, spec.heads, spec.act, spec.eps
        self.hd = spec.width // spec.heads
        self.causal, self.pool, self.eos_id, self.chunk = spec.causal, spec.pool, spec.eos_id, chunk
        self.layers = [dict(n1w=f32(b["ln1"][0]), n1b=f32(b["ln1"][1]), w_qkv=bf(b["qkv"][0]), b_qkv=f32(b["qkv"][1]),
                            w_o=bf(b["out"][0]), b_o=f32(b["out"][1]), n2w=f32(b["ln2"][0]), n2b=f32(b["ln2"][1]),
                            w_1=bf(b["fc1"][0]), b_1=f32(b["fc1"][1]), w_2=bf(b["fc2"][0]), b_2=f32(b["fc2"][1]))
                       for b in spec.blocks]
        self.mlp_width = self.layers[0]["w_1"].shape[0]
        self.fw, self.fb = f32(spec.final_ln[0]), f32(spec.final_ln[1])
        self.w_proj = bf(spec.proj) if spec.proj is not None else None
        self.embed_dim = self.w_proj.shape[0] if spec.proj is not None else None
        self.pos = f32(spec.pos)
        if spec.patch_weight is not None:                  # vision tower
            P = self.patch = spec.patch
            self.image_size = spec.image_size
            k = 3 * P * P
            self.kpad = (k + 7) // 8 * 8
            wp = torch.zeros(spec.width, self.kpad)
            wp[:, :k] = spec.patch_weight.detach().float().reshape(spec.width, k).cpu()
            self.w_patch = bf(wp)
            self.b_patch = f32(spec.patch_bias) if spec.patch_bias is not None else None
            self.cls = f32(spec.cls)
            self.pre_ln = (f32(spec.pre_ln[0]), f32(spec.pre_ln[1])) if spec.pre_ln is not None else None
            self.mean_std = torch.tensor([*mean, *std], dtype=torch.float32, device=self.device)
        else:
            self.tok = bf(spec.token_embedding)
        self.launches = 0

    def _blocks(self, x, n_seq):
        """the residual stream x f32 [n_seq * L, width] through every block, in place"""
        dev, d, rows = self.device, self.width, x.shape[0]
        h = torch.empty(rows, d, device=dev, dtype=torch.bfloat16)
        qkv = torch.empty(rows, 3 * d, device=dev, dtype=torch.bfloat16)
        att = torch.empty(rows, d, device=dev, dtype=torch.bfloat16)
        m = torch.empty(rows, self.mlp_width, device=dev, dtype=torch.bfloat16)
        mf = torch.empty(rows, self.mlp_width, device=dev, dtype=torch.float32) if self.act == "quick_gelu" else None
        scale = self.hd ** -0.5
        for ly in self.layers:
            nv.layernorm_modulate(x, h, self.eps, gamma=ly["n1w"], beta=ly["n1b"])
            nv.gemm(h, ly["w_qkv"], qkv, bias=ly["b_qkv"])
            nv.quality_attn(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], att, n_seq, self.heads, self.hd, scale, self.causal)
            nv.gemm(att, ly["w_o"], x, bias=ly["b_o"], residual=x)
            nv.layernorm_modulate(x, h, self.eps, gamma=ly["n2w"], beta=ly["n2b"])
            if mf is None:
                nv.gemm(h, ly["w_1"], m, bias=ly["b_1"], act=nv.ACT_GELU_ERF)
            else:
                nv.gemm(h, ly["w_1"], mf, bias=ly["b_1"])
                nv.quality_quick_gelu(mf, m)
                self.launches += 1
            nv.gemm(m, ly["w_2"], x, bias=ly["b_2"], residual=x)
            self.launches += 7

    def _head(self, x, n_seq, ids=None):
        """pool one row per sequence -> final LayerNorm -> projection: f32 [n_seq, embed_dim]"""
        dev = self.device
        pooled = torch.empty(n_seq, self.width, device=dev, dtype=torch.float32)
        nv.quality_pool(x, n_seq, pooled, self.pool, ids, self.eos_id)
        hn = torch.empty(n_seq, self.width, device=dev, dtype=torch.bfloat16)
        nv.layernorm_modulate(pooled, hn, self.eps, gamma=self.fw, beta=self.fb)
        feats = torch.empty(n_seq, self.embed_dim, device=dev, dtype=torch.float32)
        nv.gemm(hn, self.w_proj, feats)
        self.launches += 3
        return feats

    def check_pixels(self, px):
        if tuple(px.shape[1:]) != (3, self.image_size, self.image_size):
            raise ValueError(f"ImageQualityMetric: pixels must be [B, 3, {self.image_size}, {self.image_size}], got {tuple(px.shape)}")

    def encode_images(self, px):
        B = px.shape[0]
        self.check_pixels(px)
        out = torch.empty(B, self.embed_dim, device=self.device, dtype=torch.float32)
        for s in range(0, B, self.chunk):
            chunk = px[s:s + self.chunk].to(self.device, torch.float32).contiguous()
            out[s:s + self.chunk] = self._head(self.image_states(chunk), chunk.shape[0])
        return out

    def image_states(self, px):
        """preprocessed pixels f32 [B, 3, S, S] on the device (one chunk) -> residual stream f32 [B * (1 + np), width]"""
        dev, B, d = self.device, px.shape[0], self.width
        n = (self.image_size // self.patch) ** 2
        a = torch.empty(B * n, self.kpad, device=dev, dtype=torch.bfloat16)
        nv.quality_stage_pixels(px, self.mean_std, a, self.patch)
        patch = torch.empty(B * n, d, device=dev, dtype=torch.float32)
        nv.gemm(a, self.w_patch, patch, bias=self.b_patch)
        x = torch.empty(B * (n + 1), d, device=dev, dtype=torch.float32)
        if self.pre_ln is not None:
            nv.quality_embed_ln(patch, self.cls, self.pos, *self.pre_ln, self.eps, x)
        else:
            nv.reward_embed(patch, self.cls, self.pos, x)
        self.launches += 3
        self._blocks(x, B)
        return x

    def encode_text(self, ids):
        dev, (T, L) = self.device, ids.shape
        if L > self.pos.shape[0]:
            raise ValueError(f"ImageQualityMetric: {L} tokens exceed the text tower's {self.pos.shape[0]} positions")
        ids = ids.to(device=dev, dtype=torch.int64).contiguous()
        g = torch.empty(T * L, self.width, device=dev, dtype=torch.float32)
        nv.embedding_gather(ids.view(-1), self.tok, g)
        x = torch.empty_like(g)
        nv.add_rows(g, self.pos[:L].contiguous(), x)
        self.launches += 2
        self._blocks(x, T)
        return self._head(x, T, ids)

    def encode_text_rows(self, ids):
        """(every row after the final LayerNorm, projected: f32 [T * L, embed_dim]; the pooled rows of those, f32
        [T, embed_dim]).  LayerNorm and projection act per row, so the pooled rows are the bytes encode_text returns."""
        dev, (T, L) = self.device, ids.shape
        if L > self.pos.shape[0]:
            raise ValueError(f"ImageQualityMetric: {L} tokens exceed the text tower's {self.pos.shape[0]} positions")
        ids = ids.to(device=dev, dtype=torch.int64).contiguous()
        g = torch.empty(T * L, self.width, device=dev, dtype=torch.float32)
        nv.embedding_gather(ids.view(-1), self.tok, g)
        x = torch.empty_like(g)
        nv.add_rows(g, self.pos[:L].contiguous(), x)
        self._blocks(x, T)
        hn = torch.empty(T * L, self.width, device=dev, dtype=torch.bfloat16)
        nv.layernorm_modulate(x, hn, self.eps, gamma=self.fw, beta=self.fb)
        rows = torch.empty(T * L, self.embed_dim, device=dev, dtype=torch.float32)
        nv.gemm(hn, self.w_proj, rows)
        pooled = torch.empty(T, self.embed_dim, device=dev, dtype=torch.float32)
        nv.quality_pool(rows, T, pooled, self.pool, ids, self.eos_id)
        self.launches += 6
        return rows, pooled


class CLIPEngines:
    """the vision and text engines of one container"""

    def __init__(self, model, device, mean, std):
        vspec, tspec = model.specs()
        self.vision = TowerEngine(vspec, device, mean, std)
        self.text = TowerEngine(tspec, device)


def _cached_engine(model, first, last, device, mean, std):
    """one engine per container, rebuilt when the device or the weights change (as WanImageEncoder.engine)"""
    dev = torch.device(device) if device is not None else first.device
    if dev.type == "cuda" and dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    sig = (str(dev), first.data_ptr(), first._version, last.data_ptr(), last._version, tuple(mean), tuple(std))
    if model._engine is None or model._engine[0] != sig:
        model._engine = None
        model._engine = (sig, CLIPEngines(model, dev, mean, std))
    return model._engine[1]


# ================================================================================================ preprocessing
def to_rgb(image):
    """open_clip's _convert_to_rgb_or_rgba keeps RGBA, which its 3-channel patch conv then rejects; say so up front"""
    if image.mode == "RGBA":
        raise ValueError("ImageQualityMetric: RGBA images are not supported (the towers take 3 channels)")
    return image.convert("RGB")


def openclip_pixels(image, size):
    """open_clip's preprocess_val with light_augmentation=True (image_transform(resize_longest_max=True)) up to, not
    including, Normalize: ToTensor -> ResizeMaxSize(size) (bicubic, antialiased, on the float tensor; the longer side
    becomes `size`) -> zero padding to size x size, centred.  f32 [3, size, size] in [0, 1] (plus bicubic overshoot)."""
    x = torch.from_numpy(np.asarray(to_rgb(image), dtype=np.uint8).copy()).permute(2, 0, 1).float().div(255)
    h, w = x.shape[1:]
    scale = size / float(max(h, w))
    if scale != 1.0:
        nh, nw = round(h * scale), round(w * scale)
        x = F.interpolate(x[None], size=(nh, nw), mode="bicubic", align_corners=False, antialias=True)[0]
        ph, pw = size - nh, size - nw
        x = F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=0.0)
    return x


def blip_pixels(image, size):
    """torchvision's Resize(size, BICUBIC) on the PIL image (the shorter side becomes `size`, the longer one
    int(size * long / short); no resampling when the shorter side is already `size`), CenterCrop(size) (offsets
    int(round((side - size) / 2))), conversion to RGB, ToTensor: f32 [3, size, size] in [0, 1].  Normalisation runs on the
    device."""
    if image.mode == "RGBA":
        to_rgb(image)
    w, h = image.size
    short, long = (w, h) if w <= h else (h, w)
    nw, nh = (size, int(size * long / short)) if w <= h else (int(size * long / short), size)
    if (nw, nh) != (w, h):
        image = image.resize((nw, nh), Image.BICUBIC)
    top, left = int(round((nh - size) / 2.0)), int(round((nw - size) / 2.0))
    image = image.crop((left, top, left + size, top + size)).convert("RGB")
    return torch.from_numpy(np.asarray(image, dtype=np.uint8).copy()).permute(2, 0, 1).float().div(255)


def hf_pixels(processor, image):
    """the CLIPImageProcessor of the model directory (resize, centre crop, rescale) without its normalisation, which runs
    on the device: f32 [3, S, S]."""
    return processor(images=image, return_tensors="pt", do_normalize=False)["pixel_values"][0].float()


def hf_mean_std(processor):
    ip = getattr(processor, "image_processor", processor)
    return tuple(float(v) for v in ip.image_mean), tuple(float(v) for v in ip.image_std)
