"""umT5 text encoder — host side (SURVEY.md §8f.1, the first "next" row after the denoising path).

Same module / parameter names as the reference (``diffsynth/models/wan_video_text_encoder.py``: ``WanTextEncoder``
:209-255, ``T5SelfAttention`` :113-144, ``T5Attention`` :38-89, ``T5FeedForward`` :92-110, ``T5LayerNorm`` :22-35,
``T5RelativeEmbedding`` :147-190) so the umT5-XXL checkpoint (`models_t5_umt5-xxl-enc-bf16.pth`, key hash
9c8818c2…) loads unchanged.  The nn.Modules are parameter containers; ``WanTextEncoderEngine`` runs the arithmetic on
the kernel library: every projection / MLP matrix product on ``svi_gemm_bf16`` (wgmma), RMS norms, the gated-GELU
product and the 512-token attention with its bucketed relative-position bias and key mask on the encoder kernels
(``csrc/encoder_kernels.cu``).  No torch compute fallback.

Numerics: bf16 weights / GEMM operands (the reference runs the encoder in bf16), fp32 accumulation, fp32 residual
stream, norms and softmax.
"""
import math

import torch
import torch.nn as nn

from .. import _native as nv


class T5LayerNorm(nn.Module):
    def __init__(self, dim, eps=1e-6):
        super().__init__()
        self.dim, self.eps = dim, eps
        self.weight = nn.Parameter(torch.ones(dim))


class T5Attention(nn.Module):
    def __init__(self, dim, dim_attn, num_heads, dropout=0.1):
        assert dim_attn % num_heads == 0
        super().__init__()
        self.dim, self.dim_attn, self.num_heads, self.head_dim = dim, dim_attn, num_heads, dim_attn // num_heads
        self.q = nn.Linear(dim, dim_attn, bias=False)
        self.k = nn.Linear(dim, dim_attn, bias=False)
        self.v = nn.Linear(dim, dim_attn, bias=False)
        self.o = nn.Linear(dim_attn, dim, bias=False)


class T5FeedForward(nn.Module):
    def __init__(self, dim, dim_ffn, dropout=0.1):
        super().__init__()
        self.dim, self.dim_ffn = dim, dim_ffn
        self.gate = nn.Sequential(nn.Linear(dim, dim_ffn, bias=False), nn.GELU(approximate="tanh"))
        self.fc1 = nn.Linear(dim, dim_ffn, bias=False)
        self.fc2 = nn.Linear(dim_ffn, dim, bias=False)


class T5RelativeEmbedding(nn.Module):
    def __init__(self, num_buckets, num_heads, bidirectional, max_dist=128):
        super().__init__()
        self.num_buckets, self.num_heads, self.bidirectional, self.max_dist = num_buckets, num_heads, bidirectional, max_dist
        self.embedding = nn.Embedding(num_buckets, num_heads)


class T5SelfAttention(nn.Module):
    def __init__(self, dim, dim_attn, dim_ffn, num_heads, num_buckets, shared_pos=True, dropout=0.1):
        super().__init__()
        self.shared_pos = shared_pos
        self.norm1 = T5LayerNorm(dim)
        self.attn = T5Attention(dim, dim_attn, num_heads, dropout)
        self.norm2 = T5LayerNorm(dim)
        self.ffn = T5FeedForward(dim, dim_ffn, dropout)
        self.pos_embedding = None if shared_pos else T5RelativeEmbedding(num_buckets, num_heads, bidirectional=True)


def relative_position_buckets(lq, lk, num_buckets=32, max_dist=128):
    """Bucket index int32 [lq, lk] of (key - query), bidirectional T5 scheme (reference :171-190): half of the buckets
    per direction; distances below num_buckets/4 get their own bucket, larger ones share logarithmic bins up to
    max_dist.  Position-only, so one table serves every layer and head."""
    rel = torch.arange(lk).unsqueeze(0) - torch.arange(lq).unsqueeze(1)
    half = num_buckets // 2
    side = (rel > 0).long() * half
    dist = rel.abs()
    exact = half // 2
    log_bin = exact + (torch.log(dist.float() / exact) / math.log(max_dist / exact) * (half - exact)).long()
    log_bin = torch.clamp(log_bin, max=half - 1)
    return (side + torch.where(dist < exact, dist, log_bin)).to(torch.int32)


class WanTextEncoderEngine:
    """Kernel-ready weights of one WanTextEncoder on one device + the forward that drives the native kernels."""

    def __init__(self, model: "WanTextEncoder", device):
        nv.require_cuda(device, "the text encoder")
        self.device = torch.device(device)
        self.dim, self.dim_attn, self.H = model.dim, model.dim_attn, model.num_heads
        self.hd = model.dim_attn // model.num_heads
        self.num_buckets = model.num_buckets
        bf = lambda t: t.detach().to(device=self.device, dtype=torch.bfloat16).contiguous()
        f32 = lambda t: t.detach().to(device=self.device, dtype=torch.float32).contiguous()
        self.table = bf(model.token_embedding.weight)
        self.norm_w, self.eps = f32(model.norm.weight), model.norm.eps
        if model.shared_pos:
            raise NotImplementedError("shared_pos=True (T5 v1.0 style single bias table) is not used by umT5 / Wan")
        self.layers = []
        for b in model.blocks:
            self.layers.append(dict(
                n1=f32(b.norm1.weight), n2=f32(b.norm2.weight), eps=b.norm1.eps,
                w_qkv=bf(torch.cat([b.attn.q.weight, b.attn.k.weight, b.attn.v.weight], 0)), w_o=bf(b.attn.o.weight),
                w_gate=bf(b.ffn.gate[0].weight), w_fc1=bf(b.ffn.fc1.weight), w_fc2=bf(b.ffn.fc2.weight),
                bias=f32(b.pos_embedding.embedding.weight)))          # [num_buckets, H]
        self._buckets = {}
        self.launches = 0

    def buckets(self, L):
        t = self._buckets.get(L)
        if t is None:
            t = relative_position_buckets(L, L, self.num_buckets).contiguous().to(self.device)
            self._buckets[L] = t
        return t

    def forward(self, ids, mask=None):
        """ids int64 [1, L], mask [1, L] (0 = padding) -> f32 [1, L, dim] (reference WanTextEncoder.forward :245-255)."""
        if ids.dim() != 2 or ids.shape[0] != 1:
            raise RuntimeError(f"svi_b200: text encoder expects ids of shape [1, L], got {tuple(ids.shape)}")
        dev, d, da, L = self.device, self.dim, self.dim_attn, ids.shape[1]
        ids_d = ids[0].to(device=dev, dtype=torch.int64).contiguous()
        if int(ids_d.min()) < 0 or int(ids_d.max()) >= self.table.shape[0]:
            raise RuntimeError("svi_b200: token id outside the embedding table")
        km = None if mask is None else mask[0].to(device=dev).ne(0).to(torch.int32).contiguous()
        bucket = self.buckets(L)
        x = torch.empty(L, d, device=dev, dtype=torch.float32)
        h = torch.empty(L, d, device=dev, dtype=torch.bfloat16)
        qkv = torch.empty(L, 3 * da, device=dev, dtype=torch.bfloat16)
        att = torch.empty(L, da, device=dev, dtype=torch.bfloat16)
        f = self.layers[0]["w_gate"].shape[0]
        g = torch.empty(L, f, device=dev, dtype=torch.bfloat16)
        u = torch.empty(L, f, device=dev, dtype=torch.bfloat16)
        nv.embedding_gather(ids_d, self.table, x)
        for ly in self.layers:
            nv.rmsnorm_affine(x, ly["n1"], ly["eps"], h)
            nv.gemm(h, ly["w_qkv"], qkv)
            # T5 attention: unscaled scores + per-layer bucketed position bias, padding keys masked (:70-82)
            nv.attention_small(qkv[:, :da], qkv[:, da:2 * da], qkv[:, 2 * da:], att, self.H, self.hd, 1.0,
                               bias_table=ly["bias"], bucket=bucket, key_mask=km)
            nv.gemm(att, ly["w_o"], x, residual=x)
            nv.rmsnorm_affine(x, ly["n2"], ly["eps"], h)
            nv.gemm(h, ly["w_gate"], g, act=nv.ACT_GELU_TANH)
            nv.gemm(h, ly["w_fc1"], u)
            nv.mul_bf16(g, u, g)
            nv.gemm(g, ly["w_fc2"], x, residual=x)
            self.launches += 9
        nv.rmsnorm_affine(x, self.norm_w, self.eps, h)
        self.launches += 2
        return h.to(torch.float32).unsqueeze(0)


class WanTextEncoder(nn.Module):
    def __init__(self, vocab=256384, dim=4096, dim_attn=4096, dim_ffn=10240, num_heads=64, num_layers=24, num_buckets=32,
                 shared_pos=False, dropout=0.1):
        super().__init__()
        self.dim, self.dim_attn, self.dim_ffn = dim, dim_attn, dim_ffn
        self.num_heads, self.num_layers, self.num_buckets, self.shared_pos = num_heads, num_layers, num_buckets, shared_pos
        self.token_embedding = vocab if isinstance(vocab, nn.Embedding) else nn.Embedding(vocab, dim)
        self.pos_embedding = T5RelativeEmbedding(num_buckets, num_heads, bidirectional=True) if shared_pos else None
        self.blocks = nn.ModuleList([T5SelfAttention(dim, dim_attn, dim_ffn, num_heads, num_buckets, shared_pos, dropout)
                                     for _ in range(num_layers)])
        self.norm = T5LayerNorm(dim)
        self._engine = None

    def engine(self, device=None):
        p = self.token_embedding.weight
        dev = torch.device(device) if device is not None else p.device
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        sig = (str(dev), p.data_ptr(), p._version, self.blocks[-1].ffn.fc2.weight.data_ptr())
        if self._engine is None or self._engine[0] != sig:
            self._engine = (sig, WanTextEncoderEngine(self, dev))
        return self._engine[1]

    def forward(self, ids, mask=None):
        """[1, L] token ids (+ padding mask) -> [1, L, dim] in the parameter dtype."""
        dev = ids.device if ids.is_cuda else self.token_embedding.weight.device
        out = self.engine(dev).forward(ids, mask)
        return out.to(self.token_embedding.weight.dtype)

    @staticmethod
    def state_dict_converter():
        return WanTextEncoderStateDictConverter()


class WanTextEncoderStateDictConverter:
    def from_diffusers(self, state_dict):
        return state_dict

    def from_civitai(self, state_dict):
        return state_dict
