"""fp32 torch restatement of the cross-attention scorers — TEST INFRASTRUCTURE ONLY:

* ImageReward: the BLIP ViT (all rows, final LayerNorm), the BERT with cross-attention in every layer (its [CLS] row)
  and the reward head (five Linear layers, then (r - mean) / std);
* MPS: the CLIP towers' projected rows (text after the final LayerNorm, image before ``post_layernorm``), the condition
  mask, the 4-layer cross model and the score.

State dicts carry the checkpoints' key names (tools/synth_reward.py).  Pinned to the real reference modules by
tests/golden/reward_tiny.npz (tests/golden/make_golden_reward.py)."""
import torch
import torch.nn.functional as F

from oracle import quality_oracle as Q

REWARD_MEAN, REWARD_STD = 0.16717362830052426, 1.0333394966054072


# ------------------------------------------------------------------------------------------------ ImageReward
def blip_image_states(sd, px, layers):
    """normalised px [B, 3, S, S] -> the visual encoder's output, every row [B, 1 + np, W]"""
    p = "blip.visual_encoder."
    w = sd[p + "patch_embed.proj.weight"]
    x = F.conv2d(px, w, sd[p + "patch_embed.proj.bias"], stride=w.shape[-1]).flatten(2).transpose(1, 2)
    x = torch.cat([sd[p + "cls_token"].expand(x.shape[0], 1, -1), x], 1) + sd[p + "pos_embed"]
    heads = x.shape[-1] // 64
    for i in range(layers):
        b = f"{p}blocks.{i}."
        g = lambda k: (sd[b + k + ".weight"], sd[b + k + ".bias"])
        x = Q._block(x, dict(ln1=g("norm1"), qkv=g("attn.qkv"), out=g("attn.proj"), ln2=g("norm2"), fc1=g("mlp.fc1"),
                             fc2=g("mlp.fc2")), heads, "gelu", 1e-6, False)
    return F.layer_norm(x, (x.shape[-1],), sd[p + "norm.weight"], sd[p + "norm.bias"], 1e-6)


def _bert_attention(sd, p, x, ctx, add_mask, heads, eps):
    g = lambda k: (sd[p + k + ".weight"], sd[p + k + ".bias"])
    B, L, D = x.shape
    split = lambda t: t.view(t.shape[0], t.shape[1], heads, -1).transpose(1, 2)
    q, k, v = split(F.linear(x, *g("self.query"))), split(F.linear(ctx, *g("self.key"))), split(F.linear(ctx, *g("self.value")))
    s = (q @ k.transpose(-1, -2)) / (D // heads) ** 0.5
    if add_mask is not None:
        s = s + add_mask
    o = (s.softmax(-1) @ v).transpose(1, 2).reshape(B, L, D)
    return F.layer_norm(F.linear(o, *g("output.dense")) + x, (D,), *g("output.LayerNorm"), eps)


def bert_cls(sd, med, ids, attention_mask, image_states):
    """ids, attention_mask [B, L] (or [1, L], broadcast), image_states [B, N, W] -> the last layer's [CLS] rows [B, D]"""
    p = "blip.text_encoder."
    eps, heads, D = med["layer_norm_eps"], med["num_attention_heads"], med["hidden_size"]
    B, L = image_states.shape[0], ids.shape[1]
    x = sd[p + "embeddings.word_embeddings.weight"][ids] + sd[p + "embeddings.position_embeddings.weight"][:L]
    x = F.layer_norm(x, (D,), sd[p + "embeddings.LayerNorm.weight"], sd[p + "embeddings.LayerNorm.bias"], eps)
    x = x.expand(B, L, D)
    add_mask = ((1.0 - attention_mask.float()) * -10000.0)[:, None, None, :]      # BertModel.get_extended_attention_mask
    for i in range(med["num_hidden_layers"]):
        b = f"{p}encoder.layer.{i}."
        x = _bert_attention(sd, b + "attention.", x, x, add_mask, heads, eps)
        x = _bert_attention(sd, b + "crossattention.", x, image_states, None, heads, eps)
        h = F.gelu(F.linear(x, sd[b + "intermediate.dense.weight"], sd[b + "intermediate.dense.bias"]))
        x = F.layer_norm(F.linear(h, sd[b + "output.dense.weight"], sd[b + "output.dense.bias"]) + x, (D,),
                         sd[b + "output.LayerNorm.weight"], sd[b + "output.LayerNorm.bias"], eps)
    return x[:, 0]


def reward_head(sd, cls):
    """the reference MLP on the [CLS] rows, standardised -> [B]"""
    x = cls
    for i in (0, 2, 4, 6, 7):
        x = F.linear(x, sd[f"mlp.layers.{i}.weight"], sd[f"mlp.layers.{i}.bias"])
    return ((x - REWARD_MEAN) / REWARD_STD)[:, 0]


def imagereward(sd, med, vision_layers, px, ids, attention_mask):
    """normalised px [B, 3, S, S], one prompt's ids / mask [1, L] -> (image states, [CLS] rows, rewards [B])"""
    img = blip_image_states(sd, px, vision_layers)
    cls = bert_cls(sd, med, ids, attention_mask, img)
    return img, cls, reward_head(sd, cls)


# ------------------------------------------------------------------------------------------------ MPS
def _strip(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def mps_text_rows(sd, conf, ids):
    """ids [T, L] -> (every row after the final LayerNorm, projected [T, L, E]; the EOS rows [T, E])"""
    m, t = _strip(sd, "model."), conf["text_config"]
    x = m["text_model.embeddings.token_embedding.weight"][ids] + m["text_model.embeddings.position_embedding.weight"][:ids.shape[1]]
    for p in Q._hf_blocks(m, "text_model.", t["num_hidden_layers"]):
        x = Q._block(x, p, t["num_attention_heads"], t["hidden_act"], t.get("layer_norm_eps", 1e-5), True)
    x = F.layer_norm(x, (x.shape[-1],), m["text_model.final_layer_norm.weight"], m["text_model.final_layer_norm.bias"],
                     t.get("layer_norm_eps", 1e-5))
    rows = F.linear(x, m["text_projection.weight"])
    eos = t.get("eos_token_id", 2)
    r = ids.argmax(-1) if eos == 2 else (ids == eos).int().argmax(-1)
    return rows, rows[torch.arange(ids.shape[0]), r]


def mps_image_rows(sd, conf, px):
    """normalised px [B, 3, S, S] -> the vision encoder's last hidden state (before post_layernorm), projected
    [B, 1 + np, E]"""
    m, v = _strip(sd, "model."), conf["vision_config"]
    p = "vision_model."
    w = m[p + "embeddings.patch_embedding.weight"]
    x = F.conv2d(px, w, stride=w.shape[-1]).flatten(2).transpose(1, 2)
    x = torch.cat([m[p + "embeddings.class_embedding"].view(1, 1, -1).expand(x.shape[0], 1, -1), x], 1)
    x = x + m[p + "embeddings.position_embedding.weight"]
    eps = v.get("layer_norm_eps", 1e-5)
    x = F.layer_norm(x, (x.shape[-1],), m[p + "pre_layrnorm.weight"], m[p + "pre_layrnorm.bias"], eps)
    for blk in Q._hf_blocks(m, p, v["num_hidden_layers"]):
        x = Q._block(x, blk, v["num_attention_heads"], v["hidden_act"], eps, False)
    return F.linear(x, m["visual_projection.weight"])


def mps_mask(text_f, cond_f, threshold=0.3):
    """MPScore._calculate_score's condition mask: (ratio [L], keep bool [L])"""
    sim = (text_f @ cond_f.T).max(-1).values
    ratio = sim / sim.max()
    return ratio, ratio > threshold


def _rotate_half(t):
    t1, t2 = t.chunk(2, -1)
    return torch.cat([-t2, t1], -1)


def cross_model(sd, x, ctx, keep, heads, layers, dim_head=64):
    """x [B, N, dim] image rows, ctx [L, dim] text rows, keep bool [L] -> [B, N, dim]"""
    c = _strip(sd, "cross_model.")
    n = x.shape[1]
    inv_freq = 1.0 / (10000 ** (torch.arange(0, dim_head, 2, device=x.device).float() / dim_head))
    freqs = torch.einsum("i , j -> i j", torch.arange(n, device=x.device, dtype=torch.float32), inv_freq)
    pos = torch.cat([freqs, freqs], -1)
    rope = lambda t: t * pos.cos() + _rotate_half(t) * pos.sin()
    swiglu = lambda t: (lambda a, g: F.silu(g) * a)(*t.chunk(2, -1))
    split = lambda t: t.view(t.shape[0], t.shape[1], heads, dim_head).transpose(1, 2)
    merge = lambda t: t.transpose(1, 2).reshape(t.shape[0], t.shape[2], -1)
    neg = torch.where(keep, 0.0, float("-inf")).to(x.device)
    for i in range(layers):
        a = f"layers.{i}.0.fn."
        h = F.layer_norm(x, (x.shape[-1],), c[a + "norm.weight"], c[a + "norm.bias"])
        q = split(F.linear(h, c[a + "to_q.weight"])) * dim_head ** -0.5
        k, v = F.linear(ctx, c[a + "to_kv.weight"]).chunk(2, -1)
        att = (q @ k.T + neg).softmax(-1) @ v
        x = x + F.linear(merge(att), c[a + "to_out.weight"]) + F.linear(swiglu(F.linear(h, c[a + "ff.0.weight"])),
                                                                         c[a + "ff.2.weight"])
        s = f"layers.{i}.1.fn."
        h = F.layer_norm(x, (x.shape[-1],), c[s + "norm.weight"], c[s + "norm.bias"])
        inner = c[s + "attn_out.weight"].shape[1]
        q, k, v, ff = F.linear(h, c[s + "fused_attn_ff_proj.weight"]).split([inner, dim_head, dim_head,
                                                                              c[s + "fused_attn_ff_proj.weight"].shape[0] - inner - 2 * dim_head], -1)
        q, k = rope(split(q)) * dim_head ** -0.5, rope(k)
        att = (q @ k.unsqueeze(1).transpose(-1, -2)).softmax(-1) @ v.unsqueeze(1)
        x = x + F.linear(merge(att), c[s + "attn_out.weight"]) + F.linear(swiglu(ff), c[s + "ff_out.1.weight"])
    return x


def mps(sd, conf, heads, layers, px, ids, cond_ids):
    """normalised px [B, 3, S, S], the prompt's and the condition's ids [1, L] -> dict of the intermediate tensors and
    the scores [B]"""
    rows, eos = mps_text_rows(sd, conf, torch.cat([ids, cond_ids]))
    text_f, cond_f, text_eos = rows[0], rows[1], eos[:1]
    ratio, keep = mps_mask(text_f, cond_f)
    img = mps_image_rows(sd, conf, px)
    first = cross_model(sd, img, text_f, keep, heads, layers)[:, 0]
    score = sd["model.logit_scale"].exp() * Q.cosine(first, text_eos)[:, 0]
    return dict(text_f=text_f, cond_f=cond_f, text_eos=text_eos, ratio=ratio, keep=keep, image_rows=img, cross=first,
                scores=score)
