"""Wan DiT — host side of the H100-native hot path.

Same module/parameter names as the reference (``diffsynth/models/wan_video_dit.py``: ``WanModel`` :407-567,
``DiTBlock`` :321-374, ``SelfAttention`` :210-242, ``CrossAttention`` :245-303, ``Head`` :392-404,
``RMSNorm`` :186-197) so that Wan checkpoints and SVI LoRA keys load unchanged, but the nn.Modules are only
PARAMETER CONTAINERS: all arithmetic runs in ``WanDiTEngine`` which drives the hand-written sm_90a kernels
of ``libsvi_b200.so`` through ``diffsynth._native`` (C ABI, ``include/svi_b200.h``).  There is no torch
compute fallback: without a CUDA device + the built library every forward raises.

Numerics policy (SURVEY.md §7 hard part 1): bf16 GEMM/attention operands, fp32 accumulation, fp32 residual
stream / norms / softmax / modulation; RoPE in fp32 with an fp64-built (cos, sin) table.
"""
import math
import types
import weakref
from collections import OrderedDict
from typing import Optional, Tuple

import torch
import torch.nn as nn

from .. import _native as nv

HEAD_DIM = 128


def sinusoidal_embedding_1d(dim, position):
    """Reference wan_video_dit.py:154-158 (fp64 on the host: `position` holds one scalar per batch row)."""
    pos = position.detach().to("cpu", torch.float64).reshape(-1)
    inv = torch.pow(10000.0, -torch.arange(dim // 2, dtype=torch.float64) / (dim // 2))
    ang = torch.outer(pos, inv)
    return torch.cat([ang.cos(), ang.sin()], dim=1).to(position.dtype if position.is_floating_point() else torch.float32)


def precompute_freqs_cis(dim: int, end: int = 1024, theta: float = 10000.0):
    """Reference wan_video_dit.py:169-175 (complex128 table)."""
    freqs = 1.0 / (theta ** (torch.arange(0, dim, 2)[: dim // 2].double() / dim))
    ang = torch.outer(torch.arange(end, dtype=torch.float64), freqs)
    return torch.polar(torch.ones_like(ang), ang)


def precompute_freqs_cis_3d(dim: int, end: int = 1024, theta: float = 10000.0):
    """Reference wan_video_dit.py:161-166: (frame | height | width) tables for head_dim `dim`."""
    return (precompute_freqs_cis(dim - 2 * (dim // 3), end, theta), precompute_freqs_cis(dim // 3, end, theta),
            precompute_freqs_cis(dim // 3, end, theta))


def rope_table(freqs, f, h, w, device):
    """(cos, sin) f32 [f*h*w, head_dim/2] from the complex tables (svi_video.py:106-110), built in fp64."""
    fr = torch.cat([freqs[0][:f].view(f, 1, 1, -1).expand(f, h, w, -1),
                    freqs[1][:h].view(1, h, 1, -1).expand(f, h, w, -1),
                    freqs[2][:w].view(1, 1, w, -1).expand(f, h, w, -1)], dim=-1).reshape(f * h * w, -1)
    return (fr.real.to(torch.float32).contiguous().to(device), fr.imag.to(torch.float32).contiguous().to(device))


class RMSNorm(nn.Module):
    """Parameter container for the full-width q/k RMSNorm (reference :186-197); applied by svi_rmsnorm_rope."""

    def __init__(self, dim, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(dim))


class SelfAttention(nn.Module):
    def __init__(self, dim: int, num_heads: int, eps: float = 1e-6):
        super().__init__()
        self.dim, self.num_heads, self.head_dim = dim, num_heads, dim // num_heads
        self.q, self.k, self.v, self.o = (nn.Linear(dim, dim) for _ in range(4))
        self.norm_q = RMSNorm(dim, eps=eps)
        self.norm_k = RMSNorm(dim, eps=eps)


class CrossAttention(nn.Module):
    def __init__(self, dim: int, num_heads: int, eps: float = 1e-6, has_image_input: bool = False):
        super().__init__()
        self.dim, self.num_heads, self.head_dim = dim, num_heads, dim // num_heads
        self.q, self.k, self.v, self.o = (nn.Linear(dim, dim) for _ in range(4))
        self.norm_q = RMSNorm(dim, eps=eps)
        self.norm_k = RMSNorm(dim, eps=eps)
        self.has_image_input = has_image_input
        if has_image_input:
            self.k_img = nn.Linear(dim, dim)
            self.v_img = nn.Linear(dim, dim)
            self.norm_k_img = RMSNorm(dim, eps=eps)


class SingleStreamMutiAttention(nn.Module):
    """Parameter container of the per-frame audio cross-attention of SVI-Talk (reference models/attention.py:282-411 with
    qk_norm=False, qkv_bias=True as instantiated at wan_video_dit.py:340-350; the rotary / multi-person branch is only
    taken for human_num > 1, which DiTBlock never passes)."""

    def __init__(self, dim, encoder_hidden_states_dim, num_heads):
        super().__init__()
        self.dim, self.encoder_hidden_states_dim, self.num_heads, self.head_dim = dim, encoder_hidden_states_dim, num_heads, dim // num_heads
        self.q_linear = nn.Linear(dim, dim, bias=True)
        self.proj = nn.Linear(dim, dim)
        self.kv_linear = nn.Linear(encoder_hidden_states_dim, dim * 2, bias=True)


class AudioProjModel(nn.Module):
    """Parameter container of the audio window projector (reference wan_video_dit.py:52-112)."""

    def __init__(self, seq_len=5, seq_len_vf=12, blocks=12, channels=768, intermediate_dim=512, output_dim=768,
                 context_tokens=32, norm_output_audio=False):
        super().__init__()
        self.seq_len, self.seq_len_vf, self.blocks, self.channels = seq_len, seq_len_vf, blocks, channels
        self.input_dim, self.input_dim_vf = seq_len * blocks * channels, seq_len_vf * blocks * channels
        self.intermediate_dim, self.context_tokens, self.output_dim = intermediate_dim, context_tokens, output_dim
        self.proj1 = nn.Linear(self.input_dim, intermediate_dim)
        self.proj1_vf = nn.Linear(self.input_dim_vf, intermediate_dim)
        self.proj2 = nn.Linear(intermediate_dim, intermediate_dim)
        self.proj3 = nn.Linear(intermediate_dim, context_tokens * output_dim)
        self.norm = nn.LayerNorm(output_dim) if norm_output_audio else nn.Identity()


class DiTBlock(nn.Module):
    def __init__(self, has_image_input: bool, dim: int, num_heads: int, ffn_dim: int, eps: float = 1e-6,
                 enable_multitalk: bool = False):
        super().__init__()
        self.enable_multitalk = enable_multitalk
        if enable_multitalk:                 # reference :339-352
            self.audio_cross_attn = SingleStreamMutiAttention(dim, 768, num_heads)
            self.norm_x = nn.LayerNorm(dim, eps=eps, elementwise_affine=True)
        self.dim, self.num_heads, self.ffn_dim = dim, num_heads, ffn_dim
        self.self_attn = SelfAttention(dim, num_heads, eps)
        self.cross_attn = CrossAttention(dim, num_heads, eps, has_image_input=has_image_input)
        self.norm1 = nn.LayerNorm(dim, eps=eps, elementwise_affine=False)
        self.norm2 = nn.LayerNorm(dim, eps=eps, elementwise_affine=False)
        self.norm3 = nn.LayerNorm(dim, eps=eps)
        self.ffn = nn.Sequential(nn.Linear(dim, ffn_dim), nn.GELU(approximate="tanh"), nn.Linear(ffn_dim, dim))
        self.modulation = nn.Parameter(torch.randn(1, 6, dim) / dim ** 0.5)


class MLP(nn.Module):
    """CLIP-feature projector (reference :377-389)."""

    def __init__(self, in_dim, out_dim):
        super().__init__()
        self.proj = nn.Sequential(nn.LayerNorm(in_dim), nn.Linear(in_dim, in_dim), nn.GELU(),
                                  nn.Linear(in_dim, out_dim), nn.LayerNorm(out_dim))


class Head(nn.Module):
    def __init__(self, dim: int, out_dim: int, patch_size: Tuple[int, int, int], eps: float):
        super().__init__()
        self.dim, self.patch_size = dim, patch_size
        self.norm = nn.LayerNorm(dim, eps=eps, elementwise_affine=False)
        self.head = nn.Linear(dim, out_dim * math.prod(patch_size))
        self.modulation = nn.Parameter(torch.randn(1, 2, dim) / dim ** 0.5)


def _f32(t, device):
    return t.detach().to(device=device, dtype=torch.float32).contiguous()


def _bf16(t, device):
    return t.detach().to(device=device, dtype=torch.bfloat16).contiguous()


def _mat(t, device):
    """Kernel-ready GEMM weight.  A model loaded as float8_e4m3fn (the reference's weight-only FP8 mode) keeps its matrices
    e4m3 on the device: svi_gemm_bf16 converts them exactly to bf16 in shared memory, so the result is the same as from the
    upcast copy at half the bytes.  A matrix whose K is not a multiple of 16 (the e4m3 TMA row pitch) is upcast to bf16."""
    if t.dtype == torch.float8_e4m3fn and t.shape[-1] % 16 == 0:
        return t.detach().to(device=device).contiguous()
    return _bf16(t, device)


class _BlockWeights:
    """Kernel-ready copies of one DiTBlock's parameters (fused QKV / KV weights, fp32 vectors)."""

    def __init__(self, blk: DiTBlock, device):
        sa, ca = blk.self_attn, blk.cross_attn
        self.w_qkv = _mat(torch.cat([sa.q.weight, sa.k.weight, sa.v.weight], 0), device)
        self.b_qkv = _f32(torch.cat([sa.q.bias, sa.k.bias, sa.v.bias], 0), device)
        self.w_q, self.b_q = self.w_qkv[: blk.dim], self.b_qkv[: blk.dim]          # views (sequence-parallel split)
        self.w_kv, self.b_kv = self.w_qkv[blk.dim:], self.b_qkv[blk.dim:]
        self.w_o, self.b_o = _mat(sa.o.weight, device), _f32(sa.o.bias, device)
        self.nq, self.nk = _f32(sa.norm_q.weight, device), _f32(sa.norm_k.weight, device)
        self.eps_qk = sa.norm_q.eps
        self.w_cq, self.b_cq = _mat(ca.q.weight, device), _f32(ca.q.bias, device)
        self.w_ckv = _mat(torch.cat([ca.k.weight, ca.v.weight], 0), device)
        self.b_ckv = _f32(torch.cat([ca.k.bias, ca.v.bias], 0), device)
        self.w_co, self.b_co = _mat(ca.o.weight, device), _f32(ca.o.bias, device)
        # cross-attention q is never normalised in memory: its RMS factor rides in the attention's softmax scale
        # (svi_attn_fwd_qscale) and norm_q's channel weight is folded into the (step-invariant) K:  q.w_q . k = q . (w_q k)
        self.cnk_q = _f32(ca.norm_k.weight.detach().float() * ca.norm_q.weight.detach().float(), device)
        if ca.has_image_input:
            self.w_ckv_img = _mat(torch.cat([ca.k_img.weight, ca.v_img.weight], 0), device)
            self.b_ckv_img = _f32(torch.cat([ca.k_img.bias, ca.v_img.bias], 0), device)
            self.cnk_img_q = _f32(ca.norm_k_img.weight.detach().float() * ca.norm_q.weight.detach().float(), device)
        self.n3w, self.n3b = _f32(blk.norm3.weight, device), _f32(blk.norm3.bias, device)
        self.eps = blk.norm1.eps
        self.w_f0, self.b_f0 = _mat(blk.ffn[0].weight, device), _f32(blk.ffn[0].bias, device)
        self.w_f2, self.b_f2 = _mat(blk.ffn[2].weight, device), _f32(blk.ffn[2].bias, device)
        if getattr(blk, "enable_multitalk", False):
            a = blk.audio_cross_attn
            self.w_aq, self.b_aq = _mat(a.q_linear.weight, device), _f32(a.q_linear.bias, device)
            self.w_akv, self.b_akv = _mat(a.kv_linear.weight, device), _f32(a.kv_linear.bias, device)
            self.w_ap, self.b_ap = _mat(a.proj.weight, device), _f32(a.proj.bias, device)
            self.nxw, self.nxb = _f32(blk.norm_x.weight, device), _f32(blk.norm_x.bias, device)


# The block GEMMs an unmerged LoRA adapter applies to, and the modules whose adapters each one stacks (one column group per
# module, group_cols = d for the fused ones).
_LORA_GEMMS = (("qkv", ("self_attn.q", "self_attn.k", "self_attn.v")), ("o", ("self_attn.o",)), ("cq", ("cross_attn.q",)),
               ("ckv", ("cross_attn.k", "cross_attn.v")), ("co", ("cross_attn.o",)), ("f0", ("ffn.0",)), ("f2", ("ffn.2",)))


class _LoRAStack:
    """The active adapters of one block GEMM, stacked for svi_gemm_lora_bf16: a bf16 [groups R, K] (the down-projections),
    b bf16 [N, R] (the up-projections), gate f32 [groups R] (each adapter's alpha on its columns).  Adapter j takes the
    columns [off_j, off_j + r_j) of every group, r_j its largest rank among the GEMM's modules (zero rows / columns where
    a module has a smaller rank or none); R = sum r_j rounded up to a multiple of 64 (the kernel's k-block)."""

    def __init__(self, adapters, block, modules, n_out, k_in, device):
        ranks = [max((ad[(block, m)][0].shape[0] for m in modules if (block, m) in ad), default=0) for _, ad, _ in adapters]
        groups = len(modules)
        self.R = (sum(ranks) + 63) // 64 * 64
        self.group_cols = n_out // groups if groups > 1 else 0
        gc = n_out // groups
        a = torch.zeros(groups * self.R, k_in, dtype=torch.bfloat16)
        b = torch.zeros(n_out, self.R, dtype=torch.bfloat16)
        self.spans = []                               # (adapter name, first column, rank) per group
        off = 0
        for (name, ad, _), r in zip(adapters, ranks):
            for g, m in enumerate(modules):
                self.spans.append((name, g * self.R + off, r))
                if (block, m) in ad:
                    am, bm = ad[(block, m)]
                    a[g * self.R + off: g * self.R + off + am.shape[0]] = am
                    b[g * gc:(g + 1) * gc, off:off + bm.shape[1]] = bm
            off += r
        self.a, self.b = a.to(device), b.to(device)
        self.gate = torch.zeros(groups * self.R, dtype=torch.float32, device=device)
        self.set_alphas({name: alpha for name, _, alpha in adapters})

    def set_alphas(self, alphas):
        g = torch.zeros(self.gate.shape[0], dtype=torch.float32)
        for name, c0, r in self.spans:
            g[c0:c0 + r] = float(alphas[name])
        self.gate.copy_(g)                            # in place: captured graphs read this buffer


class ContextState:
    """Step-invariant conditioning of one prompt: embedded context rows and every layer's cross-attention K/V
    (reference recomputes text_embedding + K/V projections on every forward, svi_video.py:92, wan_video_dit.py:273-274)."""

    def __init__(self, n_img, n_txt, n_layers=0, width=0, device=None):
        self.n_img, self.n_txt = n_img, n_txt
        # one allocation for all layers (a captured CUDA graph reads a fixed copy of it: one copy_ per forward)
        self.kv_txt_all = torch.empty(n_layers, n_txt, 2 * width, device=device, dtype=torch.bfloat16) if n_layers else None
        self.kv_img_all = torch.empty(n_layers, 257, 2 * width, device=device, dtype=torch.bfloat16) if n_layers and n_img else None
        self.kv_txt = [] if self.kv_txt_all is None else list(self.kv_txt_all.unbind(0))     # per layer bf16 [n_txt, 2d]  (k normalised | v)
        self.kv_img = [] if self.kv_img_all is None else list(self.kv_img_all.unbind(0))     # per layer bf16 [257, 2d]


class TimeState:
    """Timestep conditioning of one forward: t f32 [1,d], t_mod f32 [6,d] and `mods` f32 [6*layers + 2, d] = every block's
    modulation table + t_mod (rows 6i..6i+5: shift/scale/gate of self-attention, shift/scale/gate of the FFN;
    wan_video_dit.py:356-357) followed by the head's shift/scale rows (:402)."""

    def __init__(self, t, t_mod, mods, fold=None):
        self.t, self.t_mod, self.mods = t, t_mod, mods
        self.fold = fold          # FoldVectors (per-timestep part of the LayerNorm fold) or None


class FoldVectors:
    """Per-timestep vectors of the LayerNorm fold (include/svi_b200.h, svi_gemm_epilogue.ln_*): for block i
    u1[i], c1[i] ([3d]: W_qkv g, W_qkv t + b) and u3[i], c3[i] ([ffn]: W_ffn0 g, W_ffn0 t + b) live in one f32 `pack`
    [layers, 6d + 2 ffn] (a captured graph reads a fixed copy of it); g f32 [layers, 2, d] = 1 + scale of the self-attention /
    FFN LayerNorm is what the PRODUCER epilogues multiply into the next operand."""

    def __init__(self, layers, d, ffn, device):
        self.d, self.ffn = d, ffn
        self.pack = torch.empty(layers, 6 * d + 2 * ffn, device=device, dtype=torch.float32)
        self.g = torch.empty(layers, 2, d, device=device, dtype=torch.float32)
        self.u1, self.c1 = self.pack[:, :3 * d], self.pack[:, 3 * d:6 * d]
        self.u3, self.c3 = self.pack[:, 6 * d:6 * d + ffn], self.pack[:, 6 * d + ffn:]

    def copy_(self, other):
        self.pack.copy_(other.pack)
        self.g.copy_(other.g)


class _FoldRun:
    """One forward's view of the LayerNorm fold: per-timestep vectors `v` (FoldVectors), the constant norm3 vectors u2 / c2
    [layers, d] and the zeroed row statistics f32 [layers, 3, L, 2] ((sum x, sum x^2) of the token rows entering the
    self-attention / cross-attention / FFN LayerNorm of every block) that the producer epilogues accumulate."""

    def __init__(self, v, u2, c2, stats):
        self.v, self.u2, self.c2, self.stats = v, u2, c2, stats


class AudioState:
    """Step-invariant audio conditioning of SVI-Talk: every layer's per-frame audio K|V [n_frames * tokens, 2d]."""

    def __init__(self, n_frames, tokens):
        self.n_frames, self.tokens = n_frames, tokens
        self.kv = []          # per layer bf16 [n_frames * tokens, 2d]


def _gemm_epilogue_class(a, k):
    """What a gemm call's epilogue does, for the --breakdown tag: o, cross q and cross o share one shape."""
    out = k.get("out", a[2] if len(a) > 2 else None)
    parts = [name for name in ("gate", "residual", "sumsq", "ln", "emit") if k.get(name) is not None]
    if k.get("act", nv.ACT_NONE) != nv.ACT_NONE:
        parts.append("act")
    parts.append("f32" if out is not None and out.dtype == torch.float32 else "bf16")
    return "+".join(parts)


class _CountingNative:
    """Proxy over diffsynth._native that counts kernel launches (bench.py reports them as gpu_launches)."""

    def __init__(self):
        self.launches = 0
        self.events = None      # list -> every call is bracketed by CUDA events (bench.py --breakdown)

    def __getattr__(self, name):
        fn = getattr(nv, name)

        def call(*a, **k):
            self.launches += 1
            if self.events is None:
                return fn(*a, **k)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(*a, **k)
            e1.record()
            tag = name
            if name in ("gemm", "gemm_lora"):
                tag = f"{name} M={a[0].shape[0]} N={a[1].shape[0]} K={a[1].shape[1]} {_gemm_epilogue_class(a, k)}"
            elif name == "attention":
                tag = f"attention Lq={a[0].shape[0]} Lk={a[1].shape[0]}"
            self.events.append((tag, e0, e1))
            return r
        return call

    def breakdown(self):
        """Sum of the bracketed durations per call tag (ms), and clears the list."""
        torch.cuda.synchronize()
        out = {}
        for tag, e0, e1 in self.events:
            t = out.setdefault(tag, [0.0, 0])
            t[0] += e0.elapsed_time(e1)
            t[1] += 1
        self.events = None
        return out


class WanDiTEngine:
    """Runs WanModel's arithmetic on the native kernels.  One instance per (model, device)."""

    def __init__(self, model: "WanModel", device):
        nv.require_cuda(device, "the Wan DiT")
        self.device = torch.device(device)
        # what the engine reads from the model, held here rather than through the model: the model caches its engine
        # (WanModel._engine), so a reference back would be a cycle that keeps every weight copy on the device alive after
        # the model is dropped, until Python's cyclic garbage collector happens to run
        self.freq_dim = model.freq_dim
        self.has_image_input, self.enable_multitalk = model.has_image_input, getattr(model, "enable_multitalk", False)
        self._lora_state = model._lora_state
        self.dim, self.H = model.dim, model.num_heads
        self.sig = model._param_signature()
        d = self.dim
        self.blocks = [_BlockWeights(b, self.device) for b in model.blocks]
        pe = model.patch_embedding
        self.kpatch = pe.weight.shape[1] * 4
        self.w_patch = _mat(pe.weight.reshape(d, self.kpatch), self.device)
        self.b_patch = _f32(pe.bias, self.device)
        self.w_te0, self.b_te0 = _mat(model.text_embedding[0].weight, self.device), _f32(model.text_embedding[0].bias, self.device)
        self.w_te2, self.b_te2 = _mat(model.text_embedding[2].weight, self.device), _f32(model.text_embedding[2].bias, self.device)
        self.w_t0, self.b_t0 = _mat(model.time_embedding[0].weight, self.device), _f32(model.time_embedding[0].bias, self.device)
        self.w_t2, self.b_t2 = _mat(model.time_embedding[2].weight, self.device), _f32(model.time_embedding[2].bias, self.device)
        self.w_tp, self.b_tp = _mat(model.time_projection[1].weight, self.device), _f32(model.time_projection[1].bias, self.device)
        self.w_head, self.b_head = _mat(model.head.head.weight, self.device), _f32(model.head.head.bias, self.device)
        self.head_mod = _f32(model.head.modulation.reshape(2, d), self.device)
        self.mod_table = _f32(torch.cat([b.modulation.reshape(6, d) for b in model.blocks], 0), self.device)   # [6*layers, d]
        self.eps = model.head.norm.eps
        if model.has_image_input:
            p = model.img_emb.proj
            self.ie_ln0 = (_f32(p[0].weight, self.device), _f32(p[0].bias, self.device), p[0].eps)
            self.ie_w1, self.ie_b1 = _mat(p[1].weight, self.device), _f32(p[1].bias, self.device)
            self.ie_w3, self.ie_b3 = _mat(p[3].weight, self.device), _f32(p[3].bias, self.device)
            self.ie_ln4 = (_f32(p[4].weight, self.device), _f32(p[4].bias, self.device), p[4].eps)
        if getattr(model, "enable_multitalk", False):
            ap = model.audio_proj
            self.ap_w1, self.ap_b1 = _mat(ap.proj1.weight, self.device), _f32(ap.proj1.bias, self.device)
            self.ap_w1v, self.ap_b1v = _mat(ap.proj1_vf.weight, self.device), _f32(ap.proj1_vf.bias, self.device)
            self.ap_w2, self.ap_b2 = _mat(ap.proj2.weight, self.device), _f32(ap.proj2.bias, self.device)
            self.ap_w3, self.ap_b3 = _mat(ap.proj3.weight, self.device), _f32(ap.proj3.bias, self.device)
            self.ap_ln = (_f32(ap.norm.weight, self.device), _f32(ap.norm.bias, self.device), ap.norm.eps)
            self.ap_tokens, self.ap_dim = ap.context_tokens, ap.output_dim
        self._rope = {}
        self._ws = {}
        self._ctx_cache = OrderedDict()
        self._time_cache = OrderedDict()
        self._graphs = {}
        import os
        self.use_graphs = os.environ.get("SVI_CUDA_GRAPHS", "1") != "0"
        # SVI_LN_FOLD=1: LayerNorm + modulate folded into the GEMMs around it (no LayerNorm launch inside the block stack;
        # no audio branch).  The LayerNorm passes go away, but the consumer epilogues do more work and every producer writes
        # a further bf16 copy of its output.  On an H100 (400 W power limit, bench shape, two alternating runs each) the step
        # took 1733 / 1740 ms with the fold and 1734 / 1737 ms without: no measurable gain, so the plain path stays the
        # default and the fold stays selectable (and tested) as a design point.
        self.use_fold = os.environ.get("SVI_LN_FOLD", "0") == "1"
        self._fold_static = None
        self.attn_events = None  # bench.py: list collecting (start, end) events around self-attention launches
        self.k = _CountingNative()  # every native launch goes through this proxy (bench.py reads the count)
        self._lora = None           # per block {GEMM: _LoRAStack} of the model's active adapters, or None
        self._lora_version, self._lora_alphas = 0, {}

    # ------------------------------------------------------------------ unmerged LoRA adapters
    def _sync_lora(self):
        """Follow the model's active adapter set (WanModel.set_lora_adapters).  A new set rebuilds the LoRA stacks only
        (the base weight copies stay) and drops the captured graphs, whose launches name the old stacks; new alphas are
        written into the stacks' gate vectors in place, so the graphs stay valid.  Both drop the cached context K|V, which
        the cross-attention k|v adapters change."""
        m = self._lora_state
        if self._lora_version != m.version:
            adapters = [(name, m.adapters[name][0], alpha) for name, alpha in m.active.items()]
            self._lora = None
            if adapters:
                self._lora = []
                for i, bw in enumerate(self.blocks):
                    ws = {"qkv": bw.w_qkv, "o": bw.w_o, "cq": bw.w_cq, "ckv": bw.w_ckv, "co": bw.w_co, "f0": bw.w_f0,
                          "f2": bw.w_f2}
                    stacks = {}
                    for gname, modules in _LORA_GEMMS:
                        if any((i, md) in ad for _, ad, _ in adapters for md in modules):
                            w = ws[gname]
                            stacks[gname] = _LoRAStack(adapters, i, modules, w.shape[0], w.shape[1], self.device)
                    self._lora.append(stacks)
            self._lora_version, self._lora_alphas = m.version, dict(m.active)
            self._graphs.clear()
            self._ctx_cache.clear()
        elif self._lora_alphas != m.active:
            for stacks in self._lora or ():
                for st in stacks.values():
                    st.set_alphas(m.active)
            self._lora_alphas = dict(m.active)
            self._ctx_cache.clear()

    def _lora_down(self, st, a):
        """U = gate * (a @ st.a^T) in bf16: the scaled down-projection the LoRA segment of the GEMM consumes."""
        u = self._buf("lora_u", (a.shape[0], st.a.shape[0]), torch.bfloat16)
        self.k.gemm(a, st.a, u, gate=st.gate)
        return u

    def _proj(self, st, a, w, out, **kw):
        """self.k.gemm, plus the active adapters' term when the block GEMM has a _LoRAStack `st`."""
        if st is None:
            return self.k.gemm(a, w, out, **kw)
        return self.k.gemm_lora(a, w, out, self._lora_down(st, a), st.b, st.R, st.group_cols, **kw)

    def _lora_of(self, i):
        return {} if self._lora is None else self._lora[i]

    # ------------------------------------------------------------------ helpers
    def _buf(self, name, shape, dtype):
        key = (name, tuple(shape), dtype)
        t = self._ws.get(key)
        if t is None:
            t = torch.empty(shape, device=self.device, dtype=dtype)
            self._ws[key] = t
        return t

    def rope(self, f, h, w):
        key = (f, h, w)
        if key not in self._rope:
            self._rope[key] = rope_table(precompute_freqs_cis_3d(self.dim // self.H), f, h, w, self.device)
        return self._rope[key]

    # ------------------------------------------------------------------ conditioning
    def _gemm_split(self, a2, w, out, bias=None, residual=None, emit=None):
        """out(f32) = [a_hi | a_lo] @ w^T (+ bias) (+ residual) as two accumulating passes over the same weights: the A operand
        enters with ~16 mantissa bits instead of bf16's 8.  Used for the GEMMs whose bf16 A operand dominated the parity
        error at negligible cost (embedding MLPs, patch embedding, head; tools/rounding_study.py, DESIGN.md section 2)."""
        K = w.shape[1]
        self.k.gemm(a2[:, :K], w, out, bias=bias, residual=residual)
        self.k.gemm(a2[:, K:], w, out, residual=out, emit=emit)
        return out

    def _fold_vectors(self, mods) -> FoldVectors:
        """u = W g and c = W t + b of every block's QKV and FFN-in GEMM for this timestep's modulation (g = 1 + scale,
        t = shift), g and t in two-term bf16 so the vectors carry ~16 mantissa bits: one M = 4 GEMM + one combine per
        (block, GEMM), cached with the TimeState (both CFG branches and every clip reuse them)."""
        nl, d, dev = len(self.blocks), self.dim, self.device
        ffn = self.blocks[0].w_f0.shape[0]
        fv = FoldVectors(nl, d, ffn, dev)
        rows = torch.empty(nl, 2, 4, d, device=dev, dtype=torch.bfloat16)
        self.k.ln_fold_prepare(mods, nl, fv.g, rows)
        o1 = torch.empty(4, 3 * d, device=dev, dtype=torch.float32)
        o3 = torch.empty(4, ffn, device=dev, dtype=torch.float32)
        for i, bw in enumerate(self.blocks):
            self.k.gemm(rows[i, 0], bw.w_qkv, o1)
            self.k.ln_fold_combine(o1, bw.b_qkv, fv.u1[i], fv.c1[i])
            self.k.gemm(rows[i, 1], bw.w_f0, o3)
            self.k.ln_fold_combine(o3, bw.b_f0, fv.u3[i], fv.c3[i])
        return fv

    def _fold_consts(self):
        """Step-invariant part of the fold: the affine LayerNorm in front of the cross-attention q projection
        (norm3, wan_video_dit.py:333,368): u2 = W_q gamma, c2 = W_q beta + b_q per block, f32 [layers, d] each."""
        if self._fold_static is None:
            nl, d, dev = len(self.blocks), self.dim, self.device
            u2 = torch.empty(nl, d, device=dev, dtype=torch.float32)
            c2 = torch.empty(nl, d, device=dev, dtype=torch.float32)
            gb = torch.empty(2, d, device=dev, dtype=torch.float32)
            rows = torch.empty(2, 2 * d, device=dev, dtype=torch.bfloat16)
            o4 = torch.empty(4, d, device=dev, dtype=torch.float32)
            for i, bw in enumerate(self.blocks):
                gb[0].copy_(bw.n3w)
                gb[1].copy_(bw.n3b)
                self.k.split_f32_to_bf16x2(gb, rows)             # [gamma_hi | gamma_lo ; beta_hi | beta_lo] == [4, d] row-major
                self.k.gemm(rows.view(4, d), bw.w_cq, o4)
                self.k.ln_fold_combine(o4, bw.b_cq, u2[i], c2[i])
            self._fold_static = (u2, c2)
        return self._fold_static

    def time_state(self, timestep) -> TimeState:
        """TimeState of a scalar timestep (svi_video.py:90-91): time MLP and time projection in split precision, then the
        modulation rows of every block and of the head in one launch each.  Cached per timestep value (both CFG branches
        and every clip of a video use the same 50 values)."""
        tv = float(timestep.reshape(-1)[0]) if isinstance(timestep, torch.Tensor) else float(timestep)
        hit = self._time_cache.get(tv)
        if hit is not None:
            return hit
        d, dev, nl = self.dim, self.device, len(self.blocks)
        fd = self.freq_dim
        te = sinusoidal_embedding_1d(fd, torch.tensor([tv], dtype=torch.float64)).to(torch.float32).to(dev)
        te2 = torch.empty(1, 2 * fd, device=dev, dtype=torch.bfloat16)
        th, t = (torch.empty(1, d, device=dev, dtype=torch.float32) for _ in range(2))
        th2, ts2 = (torch.empty(1, 2 * d, device=dev, dtype=torch.bfloat16) for _ in range(2))
        t_mod = torch.empty(1, 6 * d, device=dev, dtype=torch.float32)
        mods = torch.empty(6 * nl + 2, d, device=dev, dtype=torch.float32)
        self.k.split_f32_to_bf16x2(te, te2)
        self._gemm_split(te2, self.w_t0, th, bias=self.b_t0)
        self.k.split_f32_to_bf16x2(th, th2, act=nv.ACT_SILU)
        self._gemm_split(th2, self.w_t2, t, bias=self.b_t2)
        self.k.split_f32_to_bf16x2(t, ts2, act=nv.ACT_SILU)
        self._gemm_split(ts2, self.w_tp, t_mod, bias=self.b_tp)
        self.k.add_rows(self.mod_table, t_mod.view(6, d), mods[:6 * nl])
        self.k.add_rows(self.head_mod, t, mods[6 * nl:])
        out = TimeState(t, t_mod.view(6, d), mods, self._fold_vectors(mods) if self.use_fold else None)
        self._time_cache[tv] = out
        while len(self._time_cache) > 256:
            self._time_cache.popitem(last=False)
        return out

    def context_state(self, context, clip_feature=None) -> ContextState:
        """Embed the prompt (and CLIP) tokens and project every layer's cross-attention K/V once."""
        self._sync_lora()
        # keyed by tensor IDENTITY (weak references): a freed tensor's address may be reused by different data; and by the
        # adapter state the K|V were projected with
        key = (id(context), context._version, None if clip_feature is None else (id(clip_feature), clip_feature._version),
               self._lora_version, tuple(self._lora_alphas.items()))
        hit = self._ctx_cache.get(key)
        if hit is not None and hit[0]() is context and (clip_feature is None or hit[1]() is clip_feature):
            self._ctx_cache.move_to_end(key)
            return hit[2]
        d, dev = self.dim, self.device
        ctx_in = context.reshape(-1, context.shape[-1])
        n_txt, td = ctx_in.shape
        # text MLP (wan_video_dit.py:433-437) in split precision: f32 rows -> [hi | lo] bf16 pairs -> two-pass GEMMs
        src = ctx_in.to(device=dev, dtype=torch.float32).contiguous()
        c2 = torch.empty(n_txt, 2 * td, device=dev, dtype=torch.bfloat16)
        self.k.split_f32_to_bf16x2(src, c2)
        n_img = 257 if self.has_image_input else 0
        emb = torch.empty(n_img + n_txt, d, device=dev, dtype=torch.bfloat16)
        hid = torch.empty(n_txt, d, device=dev, dtype=torch.float32)
        hid2 = torch.empty(n_txt, 2 * d, device=dev, dtype=torch.bfloat16)
        e32 = torch.empty(n_txt, d, device=dev, dtype=torch.float32)
        self._gemm_split(c2, self.w_te0, hid, bias=self.b_te0)
        self.k.split_f32_to_bf16x2(hid, hid2, act=nv.ACT_GELU_TANH)
        self._gemm_split(hid2, self.w_te2, e32, bias=self.b_te2)
        self.k.cast_f32_to_bf16(e32, emb[n_img:])
        if n_img:
            if clip_feature is None:
                raise RuntimeError("has_image_input model needs clip_feature")
            cf = clip_feature.reshape(-1, clip_feature.shape[-1]).to(device=dev, dtype=torch.float32).contiguous()
            if cf.shape[0] != 257:
                raise RuntimeError(f"clip_feature must have 257 tokens, got {cf.shape[0]}")
            cw = cf.shape[1]
            c0 = torch.empty(257, 2 * cw, device=dev, dtype=torch.bfloat16)
            c1 = torch.empty(257, cw, device=dev, dtype=torch.float32)
            c1s = torch.empty(257, 2 * cw, device=dev, dtype=torch.bfloat16)
            c3 = torch.empty(257, d, device=dev, dtype=torch.float32)
            self.k.layernorm_modulate_split(cf, c0, self.ie_ln0[2], gamma=self.ie_ln0[0], beta=self.ie_ln0[1])
            self._gemm_split(c0, self.ie_w1, c1, bias=self.ie_b1)
            self.k.split_f32_to_bf16x2(c1, c1s, act=nv.ACT_GELU_ERF)
            self._gemm_split(c1s, self.ie_w3, c3, bias=self.ie_b3)
            self.k.layernorm_modulate(c3, emb[:257], self.ie_ln4[2], gamma=self.ie_ln4[0], beta=self.ie_ln4[1])
        st = self.project_context(emb, n_img)
        self._ctx_cache[key] = (weakref.ref(context), None if clip_feature is None else weakref.ref(clip_feature), st)
        while len(self._ctx_cache) > 8:
            self._ctx_cache.popitem(last=False)
        return st

    def project_context(self, emb, n_img=0) -> ContextState:
        """Every layer's cross-attention K|V from EMBEDDED context rows (bf16 [n_img + n_txt, d]; image rows first):
        K = RMSNorm(k) * (w_k * w_q) — see _BlockWeights — and V, both bf16 (wan_video_dit.py:273-274, 296-299)."""
        self._sync_lora()
        d, dev = self.dim, self.device
        n_txt = emb.shape[0] - n_img
        st = ContextState(n_img, n_txt, len(self.blocks), d, dev)
        # row sums of squares of k as d/128 partials per row (stored, not accumulated: reproducible, nothing to zero)
        P = d // 128
        ss = torch.empty(2, max(n_txt, 257), 1, P, device=dev, dtype=torch.float32)
        for li, bw in enumerate(self.blocks):
            kv = st.kv_txt[li]
            sl = ss[0, :n_txt]
            self._proj(self._lora_of(li).get("ckv"), emb[n_img:], bw.w_ckv, kv, bias=bw.b_ckv, sumsq=sl, sumsq_group_cols=d)
            self.k.rmsnorm_rope(kv[:, :d], sl, 0, bw.eps_qk, bw.cnk_q)       # K * rms * (w_k * w_q): see _BlockWeights
            if n_img:
                kvi = st.kv_img[li]
                si = ss[1, :257]
                self.k.gemm(emb[:257], bw.w_ckv_img, kvi, bias=bw.b_ckv_img, sumsq=si, sumsq_group_cols=d)
                self.k.rmsnorm_rope(kvi[:, :d], si, 0, bw.eps_qk, bw.cnk_img_q)
        return st

    def audio_state(self, audio_embed_tuple) -> AudioState:
        """SVI-Talk: AudioProjModel (reference wan_video_dit.py:82-112) on the (first-frame, latter-frames) wav2vec window
        features, then every layer's audio K|V projection (models/attention.py:333-337) — all step-invariant, computed
        once per clip and branch.  audio_embed_tuple: ([1,1,5,12,768], [1,n,8,12,768])."""
        if not self.enable_multitalk:
            raise RuntimeError("svi_b200: audio conditioning needs a WanModel built with enable_multitalk=True")
        dev, d = self.device, self.dim
        a0, a1 = audio_embed_tuple
        x0 = a0.to(device=dev, dtype=torch.bfloat16).reshape(a0.shape[1], -1).contiguous()
        x1 = a1.to(device=dev, dtype=torch.bfloat16).reshape(a1.shape[1], -1).contiguous()
        n = x0.shape[0] + x1.shape[0]
        mid = self.ap_w2.shape[0]
        h1 = torch.empty(n, mid, device=dev, dtype=torch.bfloat16)
        self.k.gemm(x0, self.ap_w1, h1[:x0.shape[0]], bias=self.ap_b1, act=nv.ACT_RELU)
        self.k.gemm(x1, self.ap_w1v, h1[x0.shape[0]:], bias=self.ap_b1v, act=nv.ACT_RELU)
        h2 = torch.empty(n, mid, device=dev, dtype=torch.bfloat16)
        self.k.gemm(h1, self.ap_w2, h2, bias=self.ap_b2, act=nv.ACT_RELU)
        tok = torch.empty(n, self.ap_tokens * self.ap_dim, device=dev, dtype=torch.float32)
        self.k.gemm(h2, self.ap_w3, tok, bias=self.ap_b3)
        tokb = torch.empty(n * self.ap_tokens, self.ap_dim, device=dev, dtype=torch.bfloat16)
        self.k.layernorm_modulate(tok.view(n * self.ap_tokens, self.ap_dim), tokb, self.ap_ln[2], gamma=self.ap_ln[0], beta=self.ap_ln[1])
        st = AudioState(n, self.ap_tokens)
        for bw in self.blocks:
            kv = torch.empty(n * self.ap_tokens, 2 * d, device=dev, dtype=torch.bfloat16)
            self.k.gemm(tokb, bw.w_akv, kv, bias=bw.b_akv)
            st.kv.append(kv)
        return st

    def _attn_workspace(self, Lq, Lk):
        """Scratch for the sliced last wave of the self-attention launch (svi_attn_fwd workspace)."""
        n = nv.attention_workspace_bytes(Lq, Lk, self.H)
        return self._buf("attn_ws", ((n + 3) // 4,), torch.float32)

    # ------------------------------------------------------------------ block stack
    def _row_sums(self, L):
        """f32 [3 * L * d/128]: the GEMM epilogues' row sums of squares of one block (q | k of self-attention, q of
        cross-attention) as d/128 partial sums per row — one per 128-column segment, STORED by the epilogue and added in
        index order by the consumers, so a forward is bit-identical from run to run (with one atomically accumulated float
        per row the order of the adds, and with it the last bit, changed between runs).  Reused by every block; never
        zeroed."""
        return self._buf("row_sums", (3 * L * (self.dim // 128),), torch.float32)

    def run_block(self, i, x, mods, ctx: ContextState, cos, sin, sp=None, audio: Optional[AudioState] = None, row_sums=None,
                  fold=None):
        """x f32 [L,d] updated in place.  Reference DiTBlock.forward wan_video_dit.py:354-374.  `mods`: TimeState.mods (or
        any f32 [>= 6*(i+1), d] table whose rows 6i..6i+5 are this block's shift/scale/gate rows); `row_sums`: the
        _row_sums scratch buffer (None: fetched here).
        `fold` (a _FoldRun): the three LayerNorms of the block are folded into the GEMMs around them — the buffer `h` then
        already holds bf16(x * g) written by the previous residual GEMM's epilogue (or the patch embedding), every residual
        GEMM of this block emits the next one, and no LayerNorm kernel runs."""
        bw = self.blocks[i]
        L, d, H = x.shape[0], self.dim, self.H
        mod = mods[6 * i: 6 * i + 6]
        h = self._buf("h", (L, d), torch.bfloat16)
        qkv = self._buf("qkv", (L, 3 * d), torch.bfloat16)
        att = self._buf("att", (L, d), torch.bfloat16)
        ffn = self._buf("ffn", (L, bw.w_f0.shape[0]), torch.bfloat16)
        rs = self._row_sums(L) if row_sums is None else row_sums
        P = d // 128
        lora = self._lora_of(i)
        # --- self attention
        if fold is None:
            self.k.layernorm_modulate(x, h, bw.eps, scale=mod[1], shift=mod[0])
            b_qkv, ln1 = bw.b_qkv, None
        else:
            b_qkv, ln1 = fold.v.c1[i], (fold.stats[i, 0], fold.v.u1[i], d, bw.eps)
        ev = self.attn_events
        if sp is None:
            ss = rs[:2 * L * P].view(L, 2, P)
            self._proj(lora.get("qkv"), h, bw.w_qkv, qkv, bias=b_qkv, sumsq=ss, sumsq_group_cols=d, ln=ln1)
            self.k.qk_norm_rope(qkv[:, :2 * d], ss, bw.eps_qk, bw.nq, bw.nk, cos, sin, 0)
            q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
        else:
            # sequence parallel: q for the local rows; K|V written straight into this rank's rows of the full
            # [L_total, 2d] buffer, normalised + rotated with the rank's row offset.  GPUs: the rows are pushed into the
            # peers' buffers over NVLink while the attention kernel already works on the local rows (PeerExchange);
            # otherwise one in-place all-gather.
            q = qkv[:, :d]
            pe = sp.peer_exchange(L * sp.sp_size, 2 * d, x.device)
            if pe is not None:
                pbuf, kvl = pe.begin()
                kvf = pe.kv[pbuf]
            else:
                kvf = self._buf("kv_full", (L * sp.sp_size, 2 * d), torch.bfloat16)
                kvl = kvf[sp.sp_rank * L:(sp.sp_rank + 1) * L]
            ssq, ssk = rs[:L * P].view(L, 1, P), rs[L * P:2 * L * P].view(L, 1, P)
            sl = lora.get("qkv")          # U [L, 3R] holds the q | k | v groups: the two launches take their columns of it
            u = None if sl is None else self._lora_down(sl, h)
            if u is None:
                self.k.gemm(h, bw.w_kv, kvl, bias=b_qkv[d:], sumsq=ssk, sumsq_group_cols=d,
                            ln=None if ln1 is None else (ln1[0], ln1[1][d:], d, bw.eps))
            else:
                self.k.gemm_lora(h, bw.w_kv, kvl, u[:, sl.R:], sl.b[d:], sl.R, d, bias=b_qkv[d:], sumsq=ssk,
                                 sumsq_group_cols=d)
            self.k.rmsnorm_rope(kvl[:, :d], ssk, 0, bw.eps_qk, bw.nk, cos, sin, sp.sp_rank * L)
            if pe is not None:
                pe.push(pbuf)
            if u is None:
                self.k.gemm(h, bw.w_q, q, bias=b_qkv[:d], sumsq=ssq, sumsq_group_cols=d,
                            ln=None if ln1 is None else (ln1[0], ln1[1][:d], d, bw.eps))
            else:
                self.k.gemm_lora(h, bw.w_q, q, u[:, :sl.R], sl.b[:d], sl.R, 0, bias=b_qkv[:d], sumsq=ssq, sumsq_group_cols=d)
            self.k.rmsnorm_rope(q, ssq, 0, bw.eps_qk, bw.nq, cos, sin, sp.sp_rank * L)
            if pe is None:
                sp.all_gather_rows(kvf)
            k, v = kvf[:, :d], kvf[:, d:]
        if ev is not None:
            e0 = torch.cuda.Event(enable_timing=True)
            e0.record()
        ws = self._attn_workspace(L, k.shape[0])
        if sp is not None and pe is not None:
            self.k.attention_sp(q, k, v, att, H, pe.flags[pbuf], pe.epoch, L, sp.sp_rank, workspace=ws)
        else:
            self.k.attention(q, k, v, att, H, workspace=ws)
        if ev is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            ev.append((e0, e1))
        self._proj(lora.get("o"), att, bw.w_o, x, bias=bw.b_o, gate=mod[2], residual=x,
                   emit=None if fold is None else (h, bw.n3w, fold.stats[i, 1]))
        # --- cross attention: q stays un-normalised in memory; its RMS factor is applied inside the softmax and norm_q's
        #     weight already sits in the context K (context_state)
        cq = qkv[:, :d]
        ss1 = rs[2 * L * P:].view(L, 1, P)
        if fold is None:
            self.k.layernorm_modulate(x, h, bw.eps, gamma=bw.n3w, beta=bw.n3b)
            self._proj(lora.get("cq"), h, bw.w_cq, cq, bias=bw.b_cq, sumsq=ss1, sumsq_group_cols=d)
        else:
            self.k.gemm(h, bw.w_cq, cq, bias=fold.c2[i], sumsq=ss1, sumsq_group_cols=d,
                        ln=(fold.stats[i, 1], fold.u2[i], d, bw.eps))
        kv = ctx.kv_txt[i]
        self.k.attention_qscale(cq, kv[:, :d], kv[:, d:], att, H, ss1, d, bw.eps_qk)
        if ctx.n_img:
            kvi = ctx.kv_img[i]
            self.k.attention_qscale(cq, kvi[:, :d], kvi[:, d:], att, H, ss1, d, bw.eps_qk, accumulate=True)
        self._proj(lora.get("co"), att, bw.w_co, x, bias=bw.b_co, residual=x,
                   emit=None if fold is None else (h, fold.v.g[i, 1], fold.stats[i, 2]))
        # --- audio cross-attention (SVI-Talk, wan_video_dit.py:361-366): tokens of latent frame f attend to that frame's
        #     audio tokens (models/attention.py:318-371); 1/sqrt(head_dim) scale, no q/k norm
        if audio is not None:
            Ta = audio.tokens
            r0 = 0 if sp is None else sp.sp_rank * L                       # first global token row of this rank
            S = (L if sp is None else L * sp.sp_size) // audio.n_frames     # tokens per latent frame
            self.k.layernorm_modulate(x, h, bw.eps, gamma=bw.nxw, beta=bw.nxb)
            aq = qkv[:, :d]
            self.k.gemm(h, bw.w_aq, aq, bias=bw.b_aq)
            kva = audio.kv[i]
            for fr in range(audio.n_frames):                                # the rank's rows may start / end inside a frame
                lo, hi = max(fr * S, r0) - r0, min((fr + 1) * S, r0 + L) - r0
                if lo < hi:
                    kf = kva[fr * Ta:(fr + 1) * Ta]
                    self.k.attention(aq[lo:hi], kf[:, :d], kf[:, d:], att[lo:hi], H)
            self.k.gemm(att, bw.w_ap, x, bias=bw.b_ap, residual=x)
        # --- FFN
        if fold is None:
            self.k.layernorm_modulate(x, h, bw.eps, scale=mod[4], shift=mod[3])
            self._proj(lora.get("f0"), h, bw.w_f0, ffn, bias=bw.b_f0, act=nv.ACT_GELU_TANH)
            self._proj(lora.get("f2"), ffn, bw.w_f2, x, bias=bw.b_f2, gate=mod[5], residual=x)
        else:
            self.k.gemm(h, bw.w_f0, ffn, bias=fold.v.c3[i], act=nv.ACT_GELU_TANH, ln=(fold.stats[i, 2], fold.v.u3[i], d, bw.eps))
            last = i + 1 == len(self.blocks)
            self.k.gemm(ffn, bw.w_f2, x, bias=bw.b_f2, gate=mod[5], residual=x,
                        emit=None if last else (h, fold.v.g[i + 1, 0], fold.stats[i + 1, 0]))
        return x

    def forward(self, x, timestep, context, clip_feature=None, y=None, sp=None, out=None, tea_cache=None, add_condition=None,
                audio=None):
        """One DiT forward (svi_video.py:74-137).  x [1,C,f,Hl,Wl] (any float dtype, CUDA) -> f32 [1,16,f,Hl,Wl].

        `context` may be a tensor [1,Lc,text_dim] or a ContextState from context_state().  `tea_cache`: a
        pipelines.svi_video.TeaCache deciding per step whether the block stack runs or the cached residual is re-used.
        `add_condition`: [1, L, dim] token-space condition added to the patch embedding (SVI-Dance pose stem output,
        reference svi_video.py:102-103).  `audio`: an AudioState (audio_state()) or the (first, latter) window-feature tuple
        of an enable_multitalk model (SVI-Talk, svi_video_talk.py:123-124)."""
        dev, d = self.device, self.dim
        if x.dim() != 5 or x.shape[0] != 1:
            raise RuntimeError(f"svi_b200: DiT forward expects x of shape [1,C,f,h,w], got {tuple(x.shape)}")
        xs = x[0].to(device=dev, dtype=torch.float32).contiguous()
        ys = None
        if self.has_image_input:
            if y is None:
                raise RuntimeError("has_image_input model needs y")
            ys = y[0].to(device=dev, dtype=torch.float32).contiguous()
        C0, f, Hl, Wl = xs.shape
        if (C0 + (0 if ys is None else ys.shape[0])) * 4 != self.kpatch:
            raise RuntimeError("svi_b200: channel count does not match patch_embedding")
        hh, ww = Hl // 2, Wl // 2
        L = f * hh * ww
        self._sync_lora()
        ts = self.time_state(timestep)
        ctx = context if isinstance(context, ContextState) else self.context_state(context, clip_feature)
        cos, sin = self.rope(f, hh, ww)
        nh = self.w_head.shape[0]
        if out is None:
            out = torch.empty(1, nh // 4, f, Hl, Wl, device=dev, dtype=torch.float32)
        if audio is not None:       # audio K|V are tiny and replicated: under sequence parallelism every rank computes them
            if not isinstance(audio, AudioState):
                audio = self.audio_state(audio)
            if L % audio.n_frames or audio.n_frames != f:
                raise RuntimeError(f"svi_b200: {audio.n_frames} audio frames for {f} latent frames")
        if (self.use_graphs and sp is None and tea_cache is None and add_condition is None and audio is None
                and self.attn_events is None and self.k.events is None and out.is_contiguous()):
            return self._graph_forward(xs, ys, ts, ctx, cos, sin, out)
        return self._run(xs, ys, ts, ctx, cos, sin, out, sp, tea_cache, add_condition, audio)

    # ------------------------------------------------------------------ CUDA-graph replay (single GPU)
    def _graph_forward(self, xs, ys, ts, ctx, cos, sin, out):
        """The whole forward is ~460 launches of fixed shape: after one eager call per input geometry it is captured into a
        CUDA graph that reads fixed copies of (latents, y, t, t_mod, cross-attention K|V) and writes a fixed output, so a
        step costs a handful of small copies + one replay on the host instead of ~15 ms of Python per forward
        (`host_enqueue_ms_per_step` in bench.py).  TeaCache and timing modes stay eager; sequence-parallel ranks have their
        own capture (`_graph_forward_sp`)."""
        key = (tuple(xs.shape), None if ys is None else tuple(ys.shape), ctx.n_txt, ctx.n_img)
        ent = self._graphs.get(key)
        if ent is None:                       # first call of this geometry: eager (allocates every work buffer)
            self._graphs[key] = {"graph": None}
            return self._run(xs, ys, ts, ctx, cos, sin, out, None, None, None, None)
        if ent["graph"] is None:
            st = ContextState(ctx.n_img, ctx.n_txt, len(self.blocks), self.dim, self.device)
            ent.update(xs=torch.empty_like(xs), ys=None if ys is None else torch.empty_like(ys),
                       ts=TimeState(None, None, torch.empty_like(ts.mods),
                                    None if ts.fold is None else FoldVectors(len(self.blocks), self.dim, ts.fold.ffn, self.device)),
                       ctx=st, out=torch.empty_like(out))
            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            n0 = self.k.launches
            # thread_local: other threads (NCCL watchdog, the bench's clock sampler) may keep calling the CUDA runtime
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                self._run(ent["xs"], ent["ys"], ent["ts"], st, cos, sin, ent["out"], None, None, None, None)
            ent["launches"] = self.k.launches - n0
            self.k.launches = n0               # recorded, not executed
            ent["graph"] = g
        ent["xs"].copy_(xs)
        if ys is not None:
            ent["ys"].copy_(ys)
        ent["ts"].mods.copy_(ts.mods)
        if ts.fold is not None:
            ent["ts"].fold.copy_(ts.fold)
        ent["ctx"].kv_txt_all.copy_(ctx.kv_txt_all)
        if ctx.n_img:
            ent["ctx"].kv_img_all.copy_(ctx.kv_img_all)
        ent["graph"].replay()
        self.k.launches += ent["launches"]
        out.copy_(ent["out"])
        return out

    def _run(self, xs, ys, ts, ctx, cos, sin, out, sp, tea_cache, add_condition, audio=None):
        """Device work of one forward on prepared inputs (everything here is stream-ordered and allocation-free after the
        first call of a geometry, so it can be captured)."""
        dev, d = self.device, self.dim
        C0, f, Hl, Wl = xs.shape
        hh, ww = Hl // 2, Wl // 2
        L = f * hh * ww
        # patchify: im2col gather + GEMM (Conv3d k=s=(1,2,2), wan_video_dit.py:473-477); the latents enter as [hi | lo] bf16
        # pairs (two accumulating GEMM passes over K = 4*C columns each): a plain bf16 cast of the latents alone put
        # 5e-4 of the output std of error on every velocity prediction (tools/rounding_study.py)
        kp = self.kpatch
        tok = self._buf("tok", (L, 2 * kp), torch.bfloat16)
        self.k.patchify_gather(xs, ys, tok, split=True)
        if sp is None:
            Ll, tok_l = L, tok
        else:
            sp.set_tokens(L)
            Ll = sp.local_rows(L)
            tok_l = tok[sp.row_offset: sp.row_offset + Ll]
        xr = self._buf("x", (Ll, d), torch.float32)
        cond_l = None
        if add_condition is not None:
            if tuple(add_condition.shape) != (1, L, d):
                raise RuntimeError(f"svi_b200: add_condition must be [1, {L}, {d}], got {tuple(add_condition.shape)}")
            cond = add_condition[0].to(device=dev, dtype=torch.float32).contiguous()
            cond_l = cond if sp is None else cond[sp.row_offset: sp.row_offset + Ll]
        nl = len(self.blocks)
        fold = None
        if self.use_fold and ts.fold is not None and audio is None and self._lora is None:   # the LoRA GEMMs take no fold
            u2, c2 = self._fold_consts()
            fold = _FoldRun(ts.fold, u2, c2, self._buf("ln_stats", (nl, 3, Ll, 2), torch.float32))
            self.k.zero_(fold.stats)
        h0 = self._buf("h", (Ll, d), torch.bfloat16)
        # x = [add_condition +] patchify(x); with the fold its last pass also emits block 0's first operand + row statistics
        self._gemm_split(tok_l, self.w_patch, xr, bias=self.b_patch, residual=cond_l,
                         emit=None if fold is None else (h0, fold.v.g[0, 0], fold.stats[0, 0]))
        if tea_cache is not None and tea_cache.check(None, xr, ts.t_mod):
            tea_cache.update(xr)                      # skipped step: tokens + residual of the last computed step
        else:
            row_sums = self._row_sums(Ll)
            for i in range(nl):
                self.run_block(i, xr, ts.mods, ctx, cos, sin, sp, audio, row_sums, fold)
            if tea_cache is not None:
                tea_cache.store(xr)
        # head (wan_video_dit.py:401-404) + unpatchify (:479-484); the normalised tokens enter the head GEMM as [hi | lo]
        h2 = self._buf("h_split", (Ll, 2 * d), torch.bfloat16)
        self.k.layernorm_modulate_split(xr, h2, self.eps, scale=ts.mods[6 * nl + 1], shift=ts.mods[6 * nl])
        nh = self.w_head.shape[0]
        ho = self._buf("head_out", (L, nh), torch.float32)
        ho_l = ho if sp is None else ho[sp.row_offset: sp.row_offset + Ll]
        self._gemm_split(h2, self.w_head, ho_l, bias=self.b_head)
        if sp is not None:
            sp.all_gather_rows(ho)
        self.k.unpatchify(ho, out[0])
        return out



class WanModel(nn.Module):
    """Reference wan_video_dit.py:407-567 — same constructor, parameter names and public attributes."""

    def __init__(self, dim: int, in_dim: int, ffn_dim: int, out_dim: int, text_dim: int, freq_dim: int, eps: float,
                 patch_size: Tuple[int, int, int], num_heads: int, num_layers: int, has_image_input: bool,
                 enable_multitalk: bool = False):
        super().__init__()
        if dim // num_heads != HEAD_DIM or dim % num_heads:
            raise ValueError(f"svi_b200 kernels are specialised for head_dim 128 (got dim={dim}, heads={num_heads})")
        if tuple(patch_size) != (1, 2, 2):
            raise ValueError("svi_b200 kernels are specialised for patch_size (1,2,2)")
        self.dim, self.freq_dim, self.has_image_input = dim, freq_dim, has_image_input
        self.patch_size, self.num_heads, self.out_dim, self.eps = tuple(patch_size), num_heads, out_dim, eps
        self.patch_embedding = nn.Conv3d(in_dim, dim, kernel_size=self.patch_size, stride=self.patch_size)
        self.text_embedding = nn.Sequential(nn.Linear(text_dim, dim), nn.GELU(approximate="tanh"), nn.Linear(dim, dim))
        self.time_embedding = nn.Sequential(nn.Linear(freq_dim, dim), nn.SiLU(), nn.Linear(dim, dim))
        self.time_projection = nn.Sequential(nn.SiLU(), nn.Linear(dim, dim * 6))
        self.blocks = nn.ModuleList([DiTBlock(has_image_input, dim, num_heads, ffn_dim, eps, enable_multitalk)
                                     for _ in range(num_layers)])
        self.head = Head(dim, out_dim, self.patch_size, eps)
        with torch.device("cpu"):      # a table, not a parameter: must be real even when the loader constructs on "meta"
            self.freqs = precompute_freqs_cis_3d(dim // num_heads)
        if has_image_input:
            self.img_emb = MLP(1280, dim)
        self.enable_multitalk = enable_multitalk
        if enable_multitalk:        # reference :455-470: audio_window 5, vae_scale 4 -> windows of 5 and 8 wav2vec frames
            self.audio_proj = AudioProjModel(seq_len=5, seq_len_vf=8, intermediate_dim=512, output_dim=768, context_tokens=32,
                                             norm_output_audio=True)
        self._engine: Optional[WanDiTEngine] = None
        self._sig_params = None
        # unmerged LoRA adapters (plain attributes, not parameters or buffers: state_dict and the fingerprints ignore them)
        # adapters: name -> ({(block, module): (A bf16 [r, in], B bf16 [out, r])}, default alpha); active: name -> alpha,
        # in stacking order; version: bumped when the active set or an active adapter's weights change.  One holder that
        # the engine shares, so the engine needs no reference to the model.
        self._lora_state = types.SimpleNamespace(adapters={}, active={}, version=0)
        self._lora_adapters = self._lora_state.adapters

    # -- unmerged LoRA adapters ----------------------------------------------------------------
    @property
    def _lora_active(self):
        return self._lora_state.active

    def add_lora_adapter(self, name, state_dict, alpha=1.0):
        """Register a LoRA (peft keys, as ModelManager.load_lora_v2 takes them) under `name` without merging it: it runs as
        a second K segment of the block GEMMs once set_lora_adapters activates it.  Targets: q, k, v, o of the self- and
        cross-attention and ffn.0 / ffn.2 of every block; anything else raises ValueError (merge those with load_lora_v2).
        The factors are kept in bf16 on the CPU; `alpha` is the scale set_lora_adapters uses when given names only."""
        from .lora import adapter_weights
        self._lora_adapters[name] = (adapter_weights(self, state_dict), float(alpha))
        if name in self._lora_state.active:
            self._lora_state.version += 1

    def set_lora_adapters(self, adapters):
        """The active adapters: {name: alpha, ...} (stacked in this order, ranks concatenated, like several LoRA files
        merged one after the other), a list of names (each at its add_lora_adapter alpha), or {} / None for none.  Changing
        only the alphas keeps the captured CUDA graphs of the engine."""
        if adapters is None:
            adapters = {}
        elif isinstance(adapters, str):
            adapters = [adapters]
        if not isinstance(adapters, dict):
            adapters = {n: self._lora_adapters[n][1] if n in self._lora_adapters else 0.0 for n in adapters}
        unknown = [n for n in adapters if n not in self._lora_adapters]
        if unknown:
            raise ValueError(f"unknown LoRA adapter(s) {unknown}; loaded: {sorted(self._lora_adapters)}")
        new = {n: float(a) for n, a in adapters.items()}
        st = self._lora_state
        if list(new) != list(st.active):
            st.version += 1
        st.active = new

    def delete_lora_adapter(self, name):
        """Forget an adapter (and deactivate it)."""
        if name not in self._lora_adapters:
            raise ValueError(f"unknown LoRA adapter {name!r}")
        del self._lora_adapters[name]
        if name in self._lora_state.active:
            self.set_lora_adapters({n: a for n, a in self._lora_state.active.items() if n != name})

    # -- engine management -------------------------------------------------------------------
    def _param_signature(self):
        """Staleness stamp of the kernel-ready weight copies: storage pointer + in-place version counter of a fixed SAMPLE of
        parameters (first / last / every 97th).  Whole-model events — .to() / .cuda() / dtype casts (`_apply`),
        `load_state_dict`, LoRA merges (`invalidate_engine`) — drop the engine explicitly, so the per-call check only has to
        catch stray in-place edits and stays O(1) instead of a Python loop over ~1k tensors per forward."""
        ps = self._sig_params
        if ps is None:
            allp = list(self.parameters())
            ps = self._sig_params = allp[::97] + allp[-1:]
        s = 0
        for p in ps:
            s = (s * 1000003 + p.data_ptr() + 7919 * p._version) % (1 << 61)
        return s

    def _apply(self, fn, *a, **k):
        self._engine, self._sig_params = None, None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._engine, self._sig_params = None, None
        return super().load_state_dict(*a, **k)

    def engine(self, device=None) -> WanDiTEngine:
        if device is None:
            device = next(self.parameters()).device
            if device.type != "cuda":
                device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else device
        device = torch.device(device)
        eng = self._engine
        if eng is None or eng.device != device or eng.sig != self._param_signature():
            launches = 0 if eng is None else eng.k.launches
            eng = WanDiTEngine(self, device)
            eng.k.launches = launches
            self._engine = eng
        return eng

    def invalidate_engine(self):
        self._engine, self._sig_params = None, None

    # -- reference surface ---------------------------------------------------------------------
    def patchify(self, x: torch.Tensor):
        """'b c f h w -> b (f h w) c' tokens after the patch embedding (f32)."""
        eng = self.engine(x.device if x.is_cuda else None)
        xs = x[0].to(device=eng.device, dtype=torch.float32).contiguous()
        C, f, H, W = xs.shape
        tok = torch.empty(f * (H // 2) * (W // 2), eng.kpatch, device=eng.device, dtype=torch.bfloat16)
        nv.patchify_gather(xs, None, tok)
        out = torch.empty(tok.shape[0], self.dim, device=eng.device, dtype=torch.float32)
        nv.gemm(tok, eng.w_patch, out, bias=eng.b_patch)
        return out.unsqueeze(0), (f, H // 2, W // 2)

    def unpatchify(self, x: torch.Tensor, grid_size):
        f, h, w = (int(v) for v in grid_size)
        eng = self.engine(x.device if x.is_cuda else None)
        ho = x[0].to(device=eng.device, dtype=torch.float32).contiguous()
        out = torch.empty(1, ho.shape[1] // 4, f, 2 * h, 2 * w, device=eng.device, dtype=torch.float32)
        nv.unpatchify(ho, out[0])
        return out

    def forward(self, x, timestep, context, clip_feature=None, y=None, **kwargs):
        dev = x.device if x.is_cuda else None
        out = self.engine(dev).forward(x, timestep, context, clip_feature, y, add_condition=kwargs.get("add_condition"),
                                       audio=kwargs.get("audio_embed_tuple"))
        return out.to(x.dtype) if x.is_floating_point() else out

    @staticmethod
    def state_dict_converter():
        return WanModelStateDictConverter()


# checkpoint key-set hash -> constructor config (reference wan_video_dit.py:656-714).  NOTE the reference's
# 1.3B branch is shadowed by the following if/elif chain and ends up with `{}` (SURVEY.md headline 7); that
# is a reference bug, not behaviour to preserve: here the 1.3B hash resolves to its config.
_CIVITAI_CONFIGS = {
    "9269f8db9040a9d860eaca435be61814": dict(has_image_input=False, patch_size=[1, 2, 2], in_dim=16, dim=1536,
                                             ffn_dim=8960, freq_dim=256, text_dim=4096, out_dim=16, num_heads=12,
                                             num_layers=30, eps=1e-6),
    "aafcfd9672c3a2456dc46e1cb6e52c70": dict(has_image_input=False, patch_size=[1, 2, 2], in_dim=16, dim=5120,
                                             ffn_dim=13824, freq_dim=256, text_dim=4096, out_dim=16, num_heads=40,
                                             num_layers=40, eps=1e-6),
    "6bfcfb3b342cb286ce886889d519a77e": dict(has_image_input=True, patch_size=[1, 2, 2], in_dim=36, dim=5120,
                                             ffn_dim=13824, freq_dim=256, text_dim=4096, out_dim=16, num_heads=40,
                                             num_layers=40, eps=1e-6),
    # SVI-Talk / MultiTalk checkpoint: 14B-I2V + audio cross-attention (reference :670-684)
    "b6caaaa1388107ec24d25592901ca489": dict(has_image_input=True, patch_size=[1, 2, 2], in_dim=36, dim=5120,
                                             ffn_dim=13824, freq_dim=256, text_dim=4096, out_dim=16, num_heads=40,
                                             num_layers=40, eps=1e-6, enable_multitalk=True),
}


class WanModelStateDictConverter:
    def from_civitai(self, state_dict):
        from .utils import hash_state_dict_keys
        return state_dict, dict(_CIVITAI_CONFIGS.get(hash_state_dict_keys(state_dict), {}))

    def from_diffusers(self, state_dict):
        """diffusers-format Wan checkpoints (reference :578-655): key renaming only."""
        ren = {"attn1.norm_k": "self_attn.norm_k", "attn1.norm_q": "self_attn.norm_q", "attn1.to_k": "self_attn.k",
               "attn1.to_out.0": "self_attn.o", "attn1.to_q": "self_attn.q", "attn1.to_v": "self_attn.v",
               "attn2.norm_k": "cross_attn.norm_k", "attn2.norm_q": "cross_attn.norm_q", "attn2.to_k": "cross_attn.k",
               "attn2.to_out.0": "cross_attn.o", "attn2.to_q": "cross_attn.q", "attn2.to_v": "cross_attn.v",
               "ffn.net.0.proj": "ffn.0", "ffn.net.2": "ffn.2", "norm2": "norm3", "scale_shift_table": "modulation"}
        top = {"condition_embedder.text_embedder.linear_1": "text_embedding.0",
               "condition_embedder.text_embedder.linear_2": "text_embedding.2",
               "condition_embedder.time_embedder.linear_1": "time_embedding.0",
               "condition_embedder.time_embedder.linear_2": "time_embedding.2",
               "condition_embedder.time_proj": "time_projection.1", "patch_embedding": "patch_embedding",
               "proj_out": "head.head"}
        out = {}
        for name, p in state_dict.items():
            if name == "scale_shift_table":
                out["head.modulation"] = p
                continue
            if name.startswith("blocks."):
                _, idx, rest = name.split(".", 2)
                for a, b in ren.items():
                    if rest == a or rest.startswith(a + "."):
                        out[f"blocks.{idx}.{b}{rest[len(a):]}"] = p
                        break
                continue
            for a, b in top.items():
                if name.startswith(a + "."):
                    out[b + name[len(a):]] = p
                    break
        cfg = {}
        if any(k.startswith("blocks.39.") for k in out) and out.get("patch_embedding.weight") is not None \
                and out["patch_embedding.weight"].shape[1] == 16:
            cfg = dict(_CIVITAI_CONFIGS["aafcfd9672c3a2456dc46e1cb6e52c70"])
        return out, cfg
