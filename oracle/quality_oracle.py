"""fp32 torch restatement of the quality-metric towers (open_clip CLIP and transformers CLIPModel key names), their
pooling, the cosine scores and the aesthetic head — TEST INFRASTRUCTURE ONLY.

Pinned to the real reference modules by tests/golden/quality_tiny.npz (tests/golden/make_golden_quality.py)."""
import torch
import torch.nn.functional as F

OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)


def normalize(px, mean=OPENAI_MEAN, std=OPENAI_STD):
    """torchvision Normalize: (x - mean) / std per channel of [B, 3, H, W]"""
    return (px - torch.tensor(mean, device=px.device).view(1, 3, 1, 1)) / torch.tensor(std, device=px.device).view(1, 3, 1, 1)


def _act(x, act):
    return x * torch.sigmoid(1.702 * x) if act == "quick_gelu" else F.gelu(x)


def _attn(x, w_qkv, b_qkv, w_o, b_o, heads, causal):
    B, L, D = x.shape
    q, k, v = F.linear(x, w_qkv, b_qkv).view(B, L, 3, heads, D // heads).permute(2, 0, 3, 1, 4)
    s = (q @ k.transpose(-1, -2)) * (D // heads) ** -0.5
    if causal:
        s = s.masked_fill(torch.ones(L, L, dtype=torch.bool, device=s.device).triu(1), float("-inf"))
    o = (s.softmax(-1) @ v).transpose(1, 2).reshape(B, L, D)
    return F.linear(o, w_o, b_o)


def _block(x, p, heads, act, eps, causal):
    """pre-LN block; p: ln1, qkv, out, ln2, fc1, fc2 as (weight, bias)"""
    D = x.shape[-1]
    x = x + _attn(F.layer_norm(x, (D,), *p["ln1"], eps), *p["qkv"], *p["out"], heads, causal)
    h = F.layer_norm(x, (D,), *p["ln2"], eps)
    return x + F.linear(_act(F.linear(h, *p["fc1"]), act), *p["fc2"])


def _openclip_blocks(sd, prefix, n):
    out = []
    for i in range(n):
        b = f"{prefix}resblocks.{i}."
        g = lambda k: (sd[b + k + ".weight"], sd[b + k + ".bias"])
        out.append(dict(ln1=g("ln_1"), qkv=(sd[b + "attn.in_proj_weight"], sd[b + "attn.in_proj_bias"]), out=g("attn.out_proj"),
                        ln2=g("ln_2"), fc1=g("mlp.c_fc"), fc2=g("mlp.c_proj")))
    return out


def _hf_blocks(sd, prefix, n):
    out = []
    for i in range(n):
        b = f"{prefix}encoder.layers.{i}."
        g = lambda k: (sd[b + k + ".weight"], sd[b + k + ".bias"])
        qkv = (torch.cat([sd[b + f"self_attn.{n}_proj.weight"] for n in "qkv"]),
               torch.cat([sd[b + f"self_attn.{n}_proj.bias"] for n in "qkv"]))
        out.append(dict(ln1=g("layer_norm1"), qkv=qkv, out=g("self_attn.out_proj"), ln2=g("layer_norm2"), fc1=g("mlp.fc1"),
                        fc2=g("mlp.fc2")))
    return out


def _vit(px, conv_w, cls, pos, pre, blocks, post, proj_t, heads, act, eps):
    """px normalised [B, 3, S, S] -> [B, E]; proj_t [E, W] (Linear layout)"""
    P = conv_w.shape[-1]
    x = F.conv2d(px, conv_w, stride=P).flatten(2).transpose(1, 2)
    x = torch.cat([cls.view(1, 1, -1).expand(x.shape[0], 1, -1), x], 1) + pos
    D = x.shape[-1]
    x = F.layer_norm(x, (D,), *pre, eps)
    for p in blocks:
        x = _block(x, p, heads, act, eps, False)
    return F.linear(F.layer_norm(x[:, 0], (D,), *post, eps), proj_t)


def _text(ids, tok, pos, blocks, final, proj_t, heads, act, eps, rows):
    x = tok[ids] + pos[:ids.shape[1]]
    for p in blocks:
        x = _block(x, p, heads, act, eps, True)
    x = F.layer_norm(x[torch.arange(ids.shape[0], device=x.device), rows], (x.shape[-1],), *final, eps)
    return F.linear(x, proj_t)


def openclip_image(sd, cfg, px):
    v = cfg["vision_cfg"]
    return _vit(px, sd["visual.conv1.weight"], sd["visual.class_embedding"], sd["visual.positional_embedding"],
                (sd["visual.ln_pre.weight"], sd["visual.ln_pre.bias"]), _openclip_blocks(sd, "visual.transformer.", v["layers"]),
                (sd["visual.ln_post.weight"], sd["visual.ln_post.bias"]), sd["visual.proj"].t(), v["width"] // v["head_width"],
                "gelu", 1e-5)


def openclip_text(sd, cfg, ids):
    t = cfg["text_cfg"]
    return _text(ids, sd["token_embedding.weight"], sd["positional_embedding"], _openclip_blocks(sd, "transformer.", t["layers"]),
                 (sd["ln_final.weight"], sd["ln_final.bias"]), sd["text_projection"].t(), t["heads"], "gelu", 1e-5,
                 ids.argmax(-1))


def hf_image(sd, config, px):
    v = config["vision_config"]
    p = "vision_model."
    return _vit(px, sd[p + "embeddings.patch_embedding.weight"], sd[p + "embeddings.class_embedding"],
                sd[p + "embeddings.position_embedding.weight"], (sd[p + "pre_layrnorm.weight"], sd[p + "pre_layrnorm.bias"]),
                _hf_blocks(sd, p, v["num_hidden_layers"]), (sd[p + "post_layernorm.weight"], sd[p + "post_layernorm.bias"]),
                sd["visual_projection.weight"], v["num_attention_heads"], v["hidden_act"], v.get("layer_norm_eps", 1e-5))


def hf_text(sd, config, ids):
    t = config["text_config"]
    p = "text_model."
    eos = t.get("eos_token_id", 2)
    rows = ids.argmax(-1) if eos == 2 else (ids == eos).int().argmax(-1)
    return _text(ids, sd[p + "embeddings.token_embedding.weight"], sd[p + "embeddings.position_embedding.weight"],
                 _hf_blocks(sd, p, t["num_hidden_layers"]), (sd[p + "final_layer_norm.weight"], sd[p + "final_layer_norm.bias"]),
                 sd["text_projection.weight"], t["num_attention_heads"], t["hidden_act"], t.get("layer_norm_eps", 1e-5), rows)


def cosine(img, txt):
    """[B, T] cosines of L2-normalised features"""
    return F.normalize(img, dim=-1) @ F.normalize(txt, dim=-1).T


def aesthetic(sd, img):
    """the reference MLP (five Linear layers, no nonlinearity) on L2-normalised image features -> [B]"""
    x = img / img.norm(dim=-1, keepdim=True)
    for i in (0, 2, 4, 6, 7):
        x = F.linear(x, sd[f"layers.{i}.weight"], sd[f"layers.{i}.bias"])
    return x[:, 0]
