"""The two cross-attention scorers with the reference's names, arguments and return values (reference ``imagereward.py``
with ``BLIP/vit.py`` and ``BLIP/med.py``; ``mps.py`` with ``trainer/models/clip_model.py`` and ``cross_modeling.py``).

* ``ImageRewardScore``: a BLIP ViT-L/16 encodes each image (all 197 rows, final LayerNorm); a BERT reads the prompt and,
  in every layer, cross-attends from its tokens to that image's rows; the ``[CLS]`` row goes through the reward head.
* ``MPScore``: a CLIP ViT-H/14 gives 257 projected rows per image (before ``post_layernorm``, as the reference's
  ``XCLIPModel.get_image_features``), the text tower gives the prompt's and a condition prompt's 77 projected rows; a
  4-layer cross model lets the image rows attend to the prompt rows whose similarity to the condition is high enough,
  then to each other; the first row's cosine with the prompt's EOS feature, times ``exp(logit_scale)``, is the score.

Containers carry the checkpoints' key names and load strictly over every key the kernels use; a few keys the scorers do
not use are skipped by name (``IGNORED``).  All images of a ``score()`` call go through the towers together, in chunks of
``chunk`` images; the prompt is encoded once per call.  Every matrix product is ``svi_gemm_bf16``, the rest is
``include/svi_b200_quality.h`` and ``include/svi_b200_reward.h``; there is no torch compute fallback.
"""
import json
import os
from typing import List, Union

import torch
import torch.nn as nn
from PIL import Image

from .config import MODEL_PATHS
from .scorers import _as_list, _device, _open
from .towers import (OPENAI_MEAN, OPENAI_STD, AestheticMLP, HFCLIPModel, TowerEngine, TowerSpec, _reject, blip_pixels,
                     check_tower, hf_mean_std, hf_pixels)
from ... import _native as nv

# ImageReward's reward standardisation (reference ImageReward.__init__)
REWARD_MEAN, REWARD_STD = 0.16717362830052426, 1.0333394966054072
BERT_MAX_LENGTH = 35
MPS_THRESHOLD = 0.3
MPS_CONDITIONS = {
    "overall": "light, color, clarity, tone, style, ambiance, artistry, shape, face, hair, hands, limbs, structure, "
               "instance, texture, quantity, attributes, position, number, location, word, things",
    "aesthetics": "light, color, clarity, tone, style, ambiance, artistry",
    "quality": "shape, face, hair, hands, limbs, structure, instance, texture",
    "semantic": "quantity, attributes, position, number, location",
}
IGNORED = ("blip.vision_proj.", "blip.text_proj.", "position_ids", "rotary_emb.inv_freq")


def _ignored(key):
    return key.startswith(IGNORED[:2]) or key.endswith(IGNORED[2:])


def _required_paths(model, path, keys):
    """the path entries a scorer reads; a missing or unreadable one raises ValueError naming the model and the key"""
    out = []
    for key in keys:
        p = path.get(key)
        if p is None or not os.path.exists(p):
            raise ValueError(f"ImageQualityMetric: {model} needs path[{key!r}], which is missing or unreadable ({p!r})")
        out.append(p)
    return out


def _load_safetensors(p):
    from safetensors.torch import load_file
    return {k: v for k, v in load_file(p).items() if not _ignored(k)}


def _lin(i, o, bias=True):
    return nn.Linear(i, o, bias=bias)


def _ln(d, eps):
    return nn.LayerNorm(d, eps=eps)


# ================================================================================================ ImageReward containers
class _BLIPBlock(nn.Module):
    def __init__(self, d, mlp):
        super().__init__()
        self.norm1, self.norm2 = _ln(d, 1e-6), _ln(d, 1e-6)
        self.attn = nn.Module()
        self.attn.qkv, self.attn.proj = _lin(d, 3 * d), _lin(d, d)
        self.mlp = nn.Module()
        self.mlp.fc1, self.mlp.fc2 = _lin(d, mlp), _lin(mlp, d)


class BLIPVisionTransformer(nn.Module):
    """BLIP/vit.py ``VisionTransformer`` (timm key names): patch_embed.proj (Conv2d with bias), cls_token, pos_embed,
    pre-LN blocks (eps 1e-6, qkv bias, GELU), final norm; no LayerNorm before the blocks."""

    def __init__(self, image_size, patch, width, layers, mlp_width):
        super().__init__()
        check_tower("BLIP vision", width, width // 64, (image_size // patch) ** 2 + 1, mlp_width, "gelu",
                    ("visual_encoder.width", "visual_encoder.width", "visual_encoder.pos_embed", "hidden_act"))
        self.image_size, self.patch, self.width = image_size, patch, width
        self.patch_embed = nn.Module()
        self.patch_embed.proj = nn.Conv2d(3, width, patch, patch)
        self.cls_token = nn.Parameter(torch.empty(1, 1, width))
        self.pos_embed = nn.Parameter(torch.empty(1, (image_size // patch) ** 2 + 1, width))
        self.blocks = nn.ModuleList([_BLIPBlock(width, mlp_width) for _ in range(layers)])
        self.norm = _ln(width, 1e-6)

    def spec(self):
        blocks = [dict(ln1=(b.norm1.weight, b.norm1.bias), qkv=(b.attn.qkv.weight, b.attn.qkv.bias),
                       out=(b.attn.proj.weight, b.attn.proj.bias), ln2=(b.norm2.weight, b.norm2.bias),
                       fc1=(b.mlp.fc1.weight, b.mlp.fc1.bias), fc2=(b.mlp.fc2.weight, b.mlp.fc2.bias)) for b in self.blocks]
        return TowerSpec(width=self.width, heads=self.width // 64, act="gelu", eps=1e-6, blocks=blocks,
                         final_ln=(self.norm.weight, self.norm.bias), proj=None, pos=self.pos_embed[0], causal=False,
                         image_size=self.image_size, patch=self.patch, patch_weight=self.patch_embed.proj.weight,
                         patch_bias=self.patch_embed.proj.bias, cls=self.cls_token.view(-1), pre_ln=None)


def _bert_attention(d, kv_width, eps):
    a = nn.Module()
    a.self = nn.Module()
    a.self.query, a.self.key, a.self.value = _lin(d, d), _lin(kv_width, d), _lin(kv_width, d)
    a.output = nn.Module()
    a.output.dense, a.output.LayerNorm = _lin(d, d), _ln(d, eps)
    return a


class _BertLayer(nn.Module):
    def __init__(self, d, inter, kv_width, eps):
        super().__init__()
        self.attention = _bert_attention(d, d, eps)
        self.crossattention = _bert_attention(d, kv_width, eps)
        self.intermediate = nn.Module()
        self.intermediate.dense = _lin(d, inter)
        self.output = nn.Module()
        self.output.dense, self.output.LayerNorm = _lin(inter, d), _ln(d, eps)


BERT_DEFAULTS = dict(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                     intermediate_size=3072, hidden_act="gelu", max_position_embeddings=512, layer_norm_eps=1e-12,
                     position_embedding_type="absolute", add_cross_attention=False)


def check_bert_config(c):
    """the BERT the kernels implement (BertConfig defaults for absent fields); anything else raises ValueError naming the
    field"""
    c = dict(BERT_DEFAULTS) | dict(c)
    if c["hidden_act"] != "gelu":
        _reject("med_config", "hidden_act", c["hidden_act"], "the FFN runs GELU(erf)")
    if c["position_embedding_type"] != "absolute":
        _reject("med_config", "position_embedding_type", c["position_embedding_type"], "absolute positions only")
    if not c["add_cross_attention"]:
        _reject("med_config", "add_cross_attention", c["add_cross_attention"], "ImageReward cross-attends in every layer")
    heads, d = c["num_attention_heads"], c["hidden_size"]
    if heads < 1 or d % heads or d // heads != 64:
        _reject("med_config", "num_attention_heads", heads, "the head width hidden_size / heads must be 64")
    if d % 8 or c["intermediate_size"] % 8:
        _reject("med_config", "hidden_size", d, "the width and the intermediate size must be multiples of 8")
    if c["max_position_embeddings"] < BERT_MAX_LENGTH:
        _reject("med_config", "max_position_embeddings", c["max_position_embeddings"], f"the prompt takes {BERT_MAX_LENGTH}")
    return c


class BertCrossModel(nn.Module):
    """BLIP/med.py ``BertModel`` without the pooler: word + absolute position embeddings, LayerNorm, then per layer
    post-LN self-attention, cross-attention to the image rows (K/V input width ``encoder_width``) and a GELU FFN."""

    def __init__(self, config, encoder_width):
        super().__init__()
        c = self.config = check_bert_config(config)
        d, eps = c["hidden_size"], c["layer_norm_eps"]
        self.embeddings = nn.Module()
        self.embeddings.word_embeddings = nn.Embedding(c["vocab_size"], d)
        self.embeddings.position_embeddings = nn.Embedding(c["max_position_embeddings"], d)
        self.embeddings.LayerNorm = _ln(d, eps)
        self.encoder = nn.Module()
        self.encoder.layer = nn.ModuleList([_BertLayer(d, c["intermediate_size"], encoder_width, eps)
                                            for _ in range(c["num_hidden_layers"])])


class ImageRewardModel(nn.Module):
    """The ImageReward checkpoint's modules: ``blip.visual_encoder``, ``blip.text_encoder``, ``mlp`` (the reference MLP:
    five Linear layers at ``layers.{0,2,4,6,7}``, no activations)."""

    def __init__(self, med_config, image_size=224, patch=16, width=1024, layers=24, mlp_width=4096):
        super().__init__()
        self.blip = nn.Module()
        self.blip.visual_encoder = BLIPVisionTransformer(image_size, patch, width, layers, mlp_width)
        self.blip.text_encoder = BertCrossModel(med_config, width)
        self.mlp = AestheticMLP(self.blip.text_encoder.config["hidden_size"])

    @staticmethod
    def vision_sizes(sd):
        """(image_size, patch, width, layers, mlp_width) of the checkpoint's visual encoder"""
        p = "blip.visual_encoder."
        w = sd[p + "patch_embed.proj.weight"]
        grid = int(round((sd[p + "pos_embed"].shape[1] - 1) ** 0.5))
        layers = len({k.split(".")[3] for k in sd if k.startswith(p + "blocks.")})
        return grid * w.shape[-1], w.shape[-1], w.shape[0], layers, sd[p + "blocks.0.mlp.fc1.weight"].shape[0]

    @classmethod
    def from_files(cls, weights, med_config):
        with open(med_config) as f:
            conf = json.load(f)
        sd = _load_safetensors(weights)
        model = cls(conf, *cls.vision_sizes(sd))
        model.load_state_dict(sd, strict=True)
        return model.eval()


def bert_tokenizer(bert_model_path):
    """transformers' BertTokenizer of the directory plus the two special tokens BLIP's init_tokenizer adds"""
    from transformers import BertTokenizer
    tok = BertTokenizer.from_pretrained(bert_model_path)
    tok.add_special_tokens({"bos_token": "[DEC]"})
    tok.add_special_tokens({"additional_special_tokens": ["[ENC]"]})
    return tok


class ImageRewardEngine:
    """ImageReward on the device: the BLIP vision tower on TowerEngine, the BERT stack and the folded head here."""

    def __init__(self, model, device, chunk=128):
        self.device = torch.device(device)
        self.chunk = chunk
        self.vision = TowerEngine(model.blip.visual_encoder.spec(), device, OPENAI_MEAN, OPENAI_STD, chunk=chunk)
        ve = model.blip.visual_encoder
        bf = lambda t: t.detach().to(device=self.device, dtype=torch.bfloat16).contiguous()
        f32 = lambda t: t.detach().to(device=self.device, dtype=torch.float32).contiguous()
        self.vnorm = (f32(ve.norm.weight), f32(ve.norm.bias))
        te = model.blip.text_encoder
        c = te.config
        self.width, self.heads, self.eps = c["hidden_size"], c["num_attention_heads"], c["layer_norm_eps"]
        emb = te.embeddings
        self.tok, self.pos = bf(emb.word_embeddings.weight), f32(emb.position_embeddings.weight)
        self.emb_ln = (f32(emb.LayerNorm.weight), f32(emb.LayerNorm.bias))

        def att(a, fused_kv):
            s = a.self
            w = dict(o=bf(a.output.dense.weight), bo=f32(a.output.dense.bias),
                     ln=(f32(a.output.LayerNorm.weight), f32(a.output.LayerNorm.bias)))
            if fused_kv:
                w.update(q=bf(s.query.weight), bq=f32(s.query.bias), kv=bf(torch.cat([s.key.weight, s.value.weight])),
                         bkv=f32(torch.cat([s.key.bias, s.value.bias])))
            else:
                w.update(qkv=bf(torch.cat([s.query.weight, s.key.weight, s.value.weight])),
                         bqkv=f32(torch.cat([s.query.bias, s.key.bias, s.value.bias])))
            return w
        self.layers = [dict(self_=att(ly.attention, False), cross=att(ly.crossattention, True),
                            w_i=bf(ly.intermediate.dense.weight), b_i=f32(ly.intermediate.dense.bias),
                            w_o=bf(ly.output.dense.weight), b_o=f32(ly.output.dense.bias),
                            ln=(f32(ly.output.LayerNorm.weight), f32(ly.output.LayerNorm.bias)))
                       for ly in te.encoder.layer]
        self.mlp_width = self.layers[0]["w_i"].shape[0]
        w, b = model.mlp.folded(REWARD_MEAN, REWARD_STD)
        self.head_w, self.head_b = w.to(self.device), b
        self.launches = 0

    # -------------------------------------------------------------------------------------------- BERT sub-blocks
    def _post_ln(self, x, xb, ln):
        nv.reward_layernorm(x, *ln, self.eps, x, xb)

    def _self_attn(self, x, xb, n, a, key_mask):
        d, rows = self.width, x.shape[0]
        qkv = torch.empty(rows, 3 * d, device=self.device, dtype=torch.bfloat16)
        att = torch.empty(rows, d, device=self.device, dtype=torch.bfloat16)
        nv.gemm(xb, a["qkv"], qkv, bias=a["bqkv"])
        nv.reward_attn(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], att, n, self.heads, 64 ** -0.5, key_mask=key_mask)
        nv.gemm(att, a["o"], x, bias=a["bo"], residual=x)
        self._post_ln(x, xb, a["ln"])
        self.launches += 4

    def _cross_attn(self, x, xb, n, a, ctx):
        d, rows = self.width, x.shape[0]
        q = torch.empty(rows, d, device=self.device, dtype=torch.bfloat16)
        kv = torch.empty(ctx.shape[0], 2 * d, device=self.device, dtype=torch.bfloat16)
        att = torch.empty(rows, d, device=self.device, dtype=torch.bfloat16)
        nv.gemm(xb, a["q"], q, bias=a["bq"])
        nv.gemm(ctx, a["kv"], kv, bias=a["bkv"])
        nv.reward_attn(q, kv[:, :d], kv[:, d:], att, n, self.heads, 64 ** -0.5)
        nv.gemm(att, a["o"], x, bias=a["bo"], residual=x)
        self._post_ln(x, xb, a["ln"])
        self.launches += 5

    def _ffn(self, x, xb, ly):
        m = torch.empty(x.shape[0], self.mlp_width, device=self.device, dtype=torch.bfloat16)
        nv.gemm(xb, ly["w_i"], m, bias=ly["b_i"], act=nv.ACT_GELU_ERF)
        nv.gemm(m, ly["w_o"], x, bias=ly["b_o"], residual=x)
        self._post_ln(x, xb, ly["ln"])
        self.launches += 3

    def prompt_states(self, ids, attention_mask):
        """the prompt through the embeddings and layer 0's self-attention, which do not depend on the image:
        (x f32 [L, width], its bf16 copy, the key mask uint8 [L])"""
        L = ids.shape[-1]
        ids = ids.reshape(-1).to(device=self.device, dtype=torch.int64).contiguous()
        key_mask = attention_mask.reshape(-1).to(device=self.device, dtype=torch.uint8).contiguous()
        g = torch.empty(L, self.width, device=self.device, dtype=torch.float32)
        nv.embedding_gather(ids, self.tok, g)
        x = torch.empty_like(g)
        nv.add_rows(g, self.pos[:L].contiguous(), x)
        xb = torch.empty(L, self.width, device=self.device, dtype=torch.bfloat16)
        self._post_ln(x, xb, self.emb_ln)
        self.launches += 3
        self._self_attn(x, xb, 1, self.layers[0]["self_"], key_mask)
        return x, xb, key_mask

    def score(self, px, ids, attention_mask):
        """preprocessed pixels f32 [B, 3, S, S] and one prompt's ids / attention mask [1, L] -> rewards f32 [B]"""
        self.vision.check_pixels(px)
        x0, xb0, key_mask = self.prompt_states(ids, attention_mask)
        out = torch.empty(px.shape[0], device=self.device, dtype=torch.float32)
        for s in range(0, px.shape[0], self.chunk):
            chunk = px[s:s + self.chunk].to(self.device, torch.float32).contiguous()
            n = chunk.shape[0]
            img = self.vision.image_states(chunk)
            ctx = torch.empty(img.shape, device=self.device, dtype=torch.bfloat16)
            nv.layernorm_modulate(img, ctx, 1e-6, gamma=self.vnorm[0], beta=self.vnorm[1])
            x, xb = x0.repeat(n, 1), xb0.repeat(n, 1)
            for i, ly in enumerate(self.layers):
                if i > 0:
                    self._self_attn(x, xb, n, ly["self_"], key_mask)
                self._cross_attn(x, xb, n, ly["cross"], ctx)
                self._ffn(x, xb, ly)
            nv.reward_head(x, n, self.head_w, self.head_b, out[s:s + n])
            self.launches += 2
        return out


class ImageRewardScore(torch.nn.Module):
    """ImageReward (BLIP ViT-L/16 + BERT-base with cross-attention + reward head).  ``path`` needs ``imagereward`` (the
    safetensors weights), ``med_config`` (BERT's JSON config) and ``bert_model_path`` (the bert-base-uncased tokenizer
    directory).  Like the reference, errors are not wrapped."""

    def __init__(self, device: Union[str, torch.device], path: dict = MODEL_PATHS):
        super().__init__()
        weights, med_config, bert_path = _required_paths("ImageReward", path, ("imagereward", "med_config", "bert_model_path"))
        self.device = _device(device)
        self.model = ImageRewardModel.from_files(weights, med_config)
        self.tokenizer = bert_tokenizer(bert_path)
        self._engine = None

    def engine(self):
        if self._engine is None:
            self._engine = ImageRewardEngine(self.model, self.device)
        return self._engine

    def tokenize(self, prompt):
        t = self.tokenizer(prompt, padding="max_length", truncation=True, max_length=BERT_MAX_LENGTH, return_tensors="pt")
        return t.input_ids, t.attention_mask

    @torch.no_grad()
    def score(self, images: Union[str, List[str], Image.Image, List[Image.Image]], prompt: str) -> List[float]:
        ims = [_open(im) for im in _as_list(images)]
        if not ims:
            return []
        size = self.model.blip.visual_encoder.image_size
        px = torch.stack([blip_pixels(im, size) for im in ims])
        ids, mask = self.tokenize(prompt)
        return self.engine().score(px, ids, mask).tolist()


# ================================================================================================ MPS containers
class BiasFreeLayerNorm(nn.Module):
    """cross_modeling.py's LayerNorm: a weight and a persistent all-zero ``bias`` buffer (loaded like any tensor)"""

    def __init__(self, d):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(d))
        self.register_buffer("bias", torch.zeros(d))


class _CrossAttention(nn.Module):
    def __init__(self, dim, heads, dim_head, ff_inner):
        super().__init__()
        self.norm = BiasFreeLayerNorm(dim)
        self.to_q = _lin(dim, heads * dim_head, False)
        self.to_kv = _lin(dim, 2 * dim_head, False)
        self.to_out = _lin(heads * dim_head, dim, False)
        self.ff = nn.Sequential(_lin(dim, 2 * ff_inner, False), nn.Identity(), _lin(ff_inner, dim, False))


class _ParallelBlock(nn.Module):
    def __init__(self, dim, heads, dim_head, ff_inner):
        super().__init__()
        self.norm = BiasFreeLayerNorm(dim)
        self.fused_attn_ff_proj = _lin(dim, heads * dim_head + 2 * dim_head + 2 * ff_inner, False)
        self.attn_out = _lin(heads * dim_head, dim, False)
        self.ff_out = nn.Sequential(nn.Identity(), _lin(ff_inner, dim, False))


def _residual(fn):
    r = nn.Module()
    r.fn = fn
    return r


class CrossModel(nn.Module):
    """cross_modeling.py ``Cross_model``: per layer Residual(CrossAttention(parallel_ff=True)) then
    Residual(ParallelTransformerBlock) (``layers.{i}.{0,1}.fn.*``)."""

    def __init__(self, dim, heads, dim_head, ff_inner, layers):
        super().__init__()
        self.dim, self.heads, self.dim_head, self.ff_inner = dim, heads, dim_head, ff_inner
        self.layers = nn.ModuleList([nn.ModuleList([_residual(_CrossAttention(dim, heads, dim_head, ff_inner)),
                                                    _residual(_ParallelBlock(dim, heads, dim_head, ff_inner))])
                                     for _ in range(layers)])

    @staticmethod
    def sizes(sd, prefix="cross_model."):
        """(dim, heads, dim_head, ff_inner, layers) read from the weights; unsupported sizes raise ValueError"""
        p = prefix + "layers.0.0.fn."
        dim = sd[p + "to_q.weight"].shape[1]
        dim_head = sd[p + "to_kv.weight"].shape[0] // 2
        if dim_head != 64:
            _reject("MPS cross_model", "to_kv dim_head", dim_head, "the attention kernel takes head width 64")
        inner = sd[p + "to_q.weight"].shape[0]
        if inner % dim_head:
            _reject("MPS cross_model", "to_q heads", inner / dim_head, "to_q's width must be a multiple of dim_head")
        ff_inner = sd[p + "ff.0.weight"].shape[0] // 2
        if dim % 8 or ff_inner % 8:
            _reject("MPS cross_model", "dim", dim, "the width and the feed-forward width must be multiples of 8")
        layers = len({k[len(prefix):].split(".")[1] for k in sd if k.startswith(prefix + "layers.")})
        return dim, inner // dim_head, dim_head, ff_inner, layers


class MPSModel(nn.Module):
    """The MPS checkpoint's modules: ``model`` (transformers CLIPModel keys) and ``cross_model``."""

    def __init__(self, clip_config, cross_sizes):
        super().__init__()
        self.model = HFCLIPModel(clip_config)
        self.cross_model = CrossModel(*cross_sizes)
        if cross_sizes[0] != self.model.projection_dim:
            _reject("MPS cross_model", "dim", cross_sizes[0], f"must equal projection_dim = {self.model.projection_dim}")

    @classmethod
    def from_files(cls, weights, clip_dir):
        with open(os.path.join(clip_dir, "config.json")) as f:
            conf = json.load(f)
        sd = _load_safetensors(weights)
        model = cls(conf, CrossModel.sizes(sd))
        model.load_state_dict(sd, strict=True)
        return model.eval()


def rope_tables(n, dim_head=64):
    """cos, sin f32 [n, dim_head / 2] of cross_modeling.py's RotaryEmbedding, computed as it does (fp32, on the host)"""
    inv_freq = 1.0 / (10000 ** (torch.arange(0, dim_head, 2).float() / dim_head))
    freqs = torch.einsum("i , j -> i j", torch.arange(n, dtype=torch.float32), inv_freq)
    return freqs.cos().contiguous(), freqs.sin().contiguous()


class MPSEngine:
    """MPS on the device: the CLIP towers on TowerEngine, the condition mask and the cross model here."""

    def __init__(self, model, device, mean, std, chunk=128):
        self.device = torch.device(device)
        self.chunk = chunk
        vspec, tspec = model.model.specs()
        self.vision = TowerEngine(vspec, device, mean, std, chunk=chunk)
        self.text = TowerEngine(tspec, device)
        bf = lambda t: t.detach().to(device=self.device, dtype=torch.bfloat16).contiguous()
        f32 = lambda t: t.detach().to(device=self.device, dtype=torch.float32).contiguous()
        self.w_vproj = bf(model.model.visual_projection.weight)
        self.logit_scale = model.model.logit_scale.detach().float()
        cm = model.cross_model
        self.dim, self.heads, self.dh, self.ff = cm.dim, cm.heads, cm.dim_head, cm.ff_inner
        inner = self.heads * self.dh
        self.layers = []
        for ca, sa in ((pair[0].fn, pair[1].fn) for pair in cm.layers):
            fused = sa.fused_attn_ff_proj.weight
            self.layers.append(dict(
                c_norm=(f32(ca.norm.weight), f32(ca.norm.bias)), c_q=bf(ca.to_q.weight), c_kv=bf(ca.to_kv.weight),
                c_ff1=bf(ca.ff[0].weight), c_out=bf(torch.cat([ca.to_out.weight, ca.ff[2].weight], 1)),
                s_norm=(f32(sa.norm.weight), f32(sa.norm.bias)), s_qkv=bf(fused[:inner + 2 * self.dh]),
                s_ff1=bf(fused[inner + 2 * self.dh:]), s_out=bf(torch.cat([sa.attn_out.weight, sa.ff_out[1].weight], 1))))
        self.tokens = (self.vision.image_size // self.vision.patch) ** 2 + 1
        self.cos, self.sin = (t.to(self.device) for t in rope_tables(self.tokens, self.dh))
        self.launches = 0

    def prompt(self, ids, cond_ids):
        """(text rows f32 [L, E] as bf16, text_EOS f32 [1, E], key mask uint8 [L], ratio f32 [L]) of one prompt and its
        condition prompt, one text-tower batch"""
        rows, pooled = self.text.encode_text_rows(torch.cat([ids, cond_ids]))
        L = ids.shape[1]
        text_f, cond_f = rows[:L], rows[L:]
        ratio = torch.empty(L, device=self.device, dtype=torch.float32)
        keep = torch.empty(L, device=self.device, dtype=torch.uint8)
        nv.reward_cond_mask(text_f, cond_f, MPS_THRESHOLD, ratio, keep)
        tb = torch.empty(L, self.dim, device=self.device, dtype=torch.bfloat16)
        nv.cast_f32_to_bf16(text_f, tb)
        self.launches += 2
        return tb, pooled[:1].contiguous(), keep, ratio

    def cross(self, x, n, tb, keep):
        """the cross model on the residual stream x f32 [n * tokens, dim], in place"""
        dev, rows, inner, dh = self.device, x.shape[0], self.heads * self.dh, self.dh
        h = torch.empty(rows, self.dim, device=dev, dtype=torch.bfloat16)
        cat = torch.empty(rows, inner + self.ff, device=dev, dtype=torch.bfloat16)
        ff1 = torch.empty(rows, 2 * self.ff, device=dev, dtype=torch.float32)
        q = torch.empty(rows, inner, device=dev, dtype=torch.bfloat16)
        qkv = torch.empty(rows, inner + 2 * dh, device=dev, dtype=torch.bfloat16)
        kv = torch.empty(tb.shape[0], 2 * dh, device=dev, dtype=torch.bfloat16)
        scale = dh ** -0.5
        for ly in self.layers:
            nv.layernorm_modulate(x, h, 1e-5, gamma=ly["c_norm"][0], beta=ly["c_norm"][1])
            nv.gemm(h, ly["c_q"], q)
            nv.gemm(tb, ly["c_kv"], kv)
            nv.reward_attn(q, kv[:, :dh], kv[:, dh:], cat[:, :inner], n, self.heads, scale, kv_heads=1, kv_shared=True,
                           key_mask=keep)
            nv.gemm(h, ly["c_ff1"], ff1)
            nv.reward_swiglu(ff1, cat[:, inner:])
            nv.gemm(cat, ly["c_out"], x, residual=x)
            nv.layernorm_modulate(x, h, 1e-5, gamma=ly["s_norm"][0], beta=ly["s_norm"][1])
            nv.gemm(h, ly["s_qkv"], qkv)
            nv.reward_rope(qkv[:, :inner + dh], self.tokens, self.cos, self.sin)
            nv.reward_attn(qkv[:, :inner], qkv[:, inner:inner + dh], qkv[:, inner + dh:], cat[:, :inner], n, self.heads,
                           scale, kv_heads=1)
            nv.gemm(h, ly["s_ff1"], ff1)
            nv.reward_swiglu(ff1, cat[:, inner:])
            nv.gemm(cat, ly["s_out"], x, residual=x)
            self.launches += 14

    def score(self, px, ids, cond_ids):
        """preprocessed pixels f32 [B, 3, S, S], the prompt's and the condition's ids [1, L] -> scores f32 [B] (host)"""
        self.vision.check_pixels(px)
        tb, eos, keep, _ = self.prompt(ids, cond_ids)
        B, dev = px.shape[0], self.device
        first = torch.empty(B, self.dim, device=dev, dtype=torch.float32)
        for s in range(0, B, self.chunk):
            chunk = px[s:s + self.chunk].to(dev, torch.float32).contiguous()
            n = chunk.shape[0]
            states = self.vision.image_states(chunk)
            sb = torch.empty(states.shape, device=dev, dtype=torch.bfloat16)
            nv.cast_f32_to_bf16(states, sb)
            x = torch.empty(states.shape[0], self.dim, device=dev, dtype=torch.float32)
            nv.gemm(sb, self.w_vproj, x)
            self.cross(x, n, tb, keep)
            nv.quality_pool(x, n, first[s:s + n])
            self.launches += 3
        cos = torch.empty(B, 1, device=dev, dtype=torch.float32)
        nv.quality_score(first, eos, cos)
        return cos[:, 0].cpu() * self.logit_scale.exp()


class MPScore(torch.nn.Module):
    """MPS (multi-dimensional preference score): a CLIP ViT-H/14 (``clip`` directory: config, processor, tokenizer) and
    a condition-aware cross model (``mps`` safetensors).  ``condition`` is one of ``MPS_CONDITIONS``; an unknown one
    raises ``ValueError`` when ``score`` is called, as in the reference.  Like the reference, errors are not wrapped."""

    def __init__(self, device: Union[str, torch.device], path: dict = MODEL_PATHS, condition: str = "overall"):
        super().__init__()
        clip_dir, weights = _required_paths("MPS", path, ("clip", "mps"))
        from transformers import AutoTokenizer, CLIPImageProcessor
        self.device = _device(device)
        self.image_processor = CLIPImageProcessor.from_pretrained(clip_dir)
        self.tokenizer = AutoTokenizer.from_pretrained(clip_dir)
        self.model = MPSModel.from_files(weights, clip_dir)
        self.mean, self.std = hf_mean_std(self.image_processor)
        self.condition = condition
        self._engine = None

    def engine(self):
        if self._engine is None:
            self._engine = MPSEngine(self.model, self.device, self.mean, self.std)
        return self._engine

    def tokenize(self, caption):
        return self.tokenizer(caption, max_length=self.tokenizer.model_max_length, padding="max_length", truncation=True,
                              return_tensors="pt").input_ids

    def condition_prompt(self):
        if self.condition not in MPS_CONDITIONS:
            raise ValueError(f"Unsupported condition: {self.condition}. Choose 'overall', 'aesthetics', 'quality', or "
                             f"'semantic'.")
        return MPS_CONDITIONS[self.condition]

    @torch.no_grad()
    def score(self, images: Union[str, List[str], Image.Image, List[Image.Image]], prompt: str) -> List[float]:
        ims = [_open(im) for im in _as_list(images)]
        if not ims:
            return []
        cond = self.condition_prompt()
        px = torch.stack([hf_pixels(self.image_processor, im) for im in ims])
        return self.engine().score(px, self.tokenize(prompt), self.tokenize(cond)).tolist()
