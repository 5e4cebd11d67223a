"""Torch stand-ins for the quality-metric entry points (include/svi_b200_quality.h) — TEST INFRASTRUCTURE ONLY.

Each function restates what its kernel computes, rounding to bf16 where the kernel stores bf16.  `install(monkeypatch)`
adds them (and the embedding gather the text tower uses) to the DiT stand-ins of tests/nv_emulation.py, so the scorers'
engines run end to end on the CPU.
"""
import torch
import torch.nn.functional as F

import nv_emulation


def _heads(t, batch, heads, hd):
    return t.double().reshape(batch, -1, heads, hd).transpose(1, 2)


def quality_attn(q, k, v, out, batch, num_heads, head_dim, scale, causal=False):
    Q, K, V = (_heads(t[:, :num_heads * head_dim], batch, num_heads, head_dim) for t in (q, k, v))
    s = (Q @ K.transpose(-1, -2)) * scale
    L = s.shape[-1]
    if causal:
        s = s.masked_fill(torch.ones(L, L, dtype=torch.bool, device=s.device).triu(1), float("-inf"))
    o = (s.softmax(-1) @ V).transpose(1, 2).reshape(batch * L, num_heads * head_dim)
    out[:, :num_heads * head_dim] = o.to(out.dtype)
    return out


def quality_stage_pixels(px, mean_std, out, patch):
    B, _, S, _ = px.shape
    G = S // patch
    x = (px - mean_std[:3].view(1, 3, 1, 1)) / mean_std[3:].view(1, 3, 1, 1)
    cols = x.reshape(B, 3, G, patch, G, patch).permute(0, 2, 4, 1, 3, 5).reshape(B * G * G, 3 * patch * patch)
    out.zero_()
    out[:, :cols.shape[1]] = cols.to(out.dtype)
    return out


def quality_embed_ln(patch, cls, pos, gamma, beta, eps, out):
    n, D = pos.shape[0] - 1, pos.shape[1]
    B = patch.shape[0] // n
    tok = torch.cat([cls.view(1, 1, D).expand(B, 1, D), patch.view(B, n, D)], 1) + pos
    out.copy_(F.layer_norm(tok, (D,), gamma, beta, eps).reshape(-1, D))
    return out


def quality_quick_gelu(x, out):
    out.copy_((x * torch.sigmoid(1.702 * x)).to(out.dtype))
    return out


def quality_pool(x, n_seq, out, mode=0, ids=None, eos_id=0):
    L = x.shape[0] // n_seq
    if mode == 0:
        rows = torch.zeros(n_seq, dtype=torch.long)
    elif mode == 1:
        rows = ids.argmax(-1).cpu()
    else:
        rows = (ids == eos_id).int().argmax(-1).cpu()
    out.copy_(x[torch.arange(n_seq) * L + rows])
    return out


def quality_score(img, txt=None, cos=None, w=None, bias=0.0, aes=None):
    xi = img / img.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    if txt is not None:
        cos.copy_(xi @ (txt / txt.norm(dim=-1, keepdim=True).clamp_min(1e-12)).T)
    if w is not None:
        aes.copy_(xi @ w + bias)
    return cos, aes


def embedding_gather(ids, table, out):
    out.copy_(table[ids.long()].float())
    return out


NAMES = ("quality_attn", "quality_stage_pixels", "quality_embed_ln", "quality_quick_gelu", "quality_pool", "quality_score")


def install(monkeypatch=None):
    from diffsynth import _native as nv
    nv_emulation.install(monkeypatch)
    put = (lambda n, v: monkeypatch.setattr(nv, n, v)) if monkeypatch is not None else (lambda n, v: setattr(nv, n, v))
    for name in NAMES + ("embedding_gather",):
        put(name, globals()[name])
