"""CLIP ViT-H/14 image encoder (visual tower of open-clip XLM-RoBERTa-L / ViT-H-14) — host side (SURVEY.md §8f.1).

Same parameter names as the reference's ``WanImageEncoder`` (``diffsynth/models/wan_video_image_encoder.py``:
``VisionTransformer`` :386-478, ``AttentionBlock`` :289-330, ``SelfAttention`` :234-268, ``WanImageEncoder`` :852-880;
the converter :894-901 drops the text tower and prefixes ``model.``), so the checkpoint
`models_clip_open-clip-xlm-roberta-large-vit-huge-14.pth` loads unchanged.  Only the visual tower exists here — the
reference also sets ``textual = None`` (:709).  ``WanImageEncoderEngine`` runs the arithmetic on the kernel library:
patch embedding, qkv / proj / MLP products on ``svi_gemm_bf16`` (bias, GELU(erf) and the fp32 residual add fused in the
epilogue), LayerNorms on ``svi_layernorm_modulate`` / ``svi_layernorm_f32``, the 257-token attention (head width 80)
on ``svi_attn_small``.  No torch compute fallback; the bicubic resize of the input image is data preparation and
stays a torch call (as in the reference, :867-873).
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _native as nv

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)     # reference :792-793
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


class _SelfAttention(nn.Module):
    def __init__(self, dim, num_heads):
        super().__init__()
        self.dim, self.num_heads, self.head_dim = dim, num_heads, dim // num_heads
        self.to_qkv = nn.Linear(dim, dim * 3)
        self.proj = nn.Linear(dim, dim)


class AttentionBlock(nn.Module):
    def __init__(self, dim, mlp_ratio, num_heads, norm_eps=1e-5):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=norm_eps)
        self.attn = _SelfAttention(dim, num_heads)
        self.norm2 = nn.LayerNorm(dim, eps=norm_eps)
        self.mlp = nn.Sequential(nn.Linear(dim, int(dim * mlp_ratio)), nn.GELU(), nn.Linear(int(dim * mlp_ratio), dim))


class VisionTransformer(nn.Module):
    """Parameter container of the visual tower (pool_type 'token', pre_norm, activation 'gelu')."""

    def __init__(self, image_size=224, patch_size=14, dim=1280, mlp_ratio=4, out_dim=1024, num_heads=16, num_layers=32,
                 norm_eps=1e-5):
        super().__init__()
        self.image_size, self.patch_size, self.dim, self.num_heads, self.num_layers = image_size, patch_size, dim, num_heads, num_layers
        self.num_patches = (image_size // patch_size) ** 2
        self.norm_eps = norm_eps
        gain = 1.0 / math.sqrt(dim)
        self.patch_embedding = nn.Conv2d(3, dim, kernel_size=patch_size, stride=patch_size, bias=False)
        self.cls_embedding = nn.Parameter(gain * torch.randn(1, 1, dim))
        self.pos_embedding = nn.Parameter(gain * torch.randn(1, self.num_patches + 1, dim))
        self.pre_norm = nn.LayerNorm(dim, eps=norm_eps)
        self.transformer = nn.Sequential(*[AttentionBlock(dim, mlp_ratio, num_heads, norm_eps) for _ in range(num_layers)])
        self.post_norm = nn.LayerNorm(dim, eps=norm_eps)
        self.head = nn.Parameter(gain * torch.randn(dim, out_dim))


class _Clip(nn.Module):
    def __init__(self, **vision):
        super().__init__()
        self.image_size = vision.get("image_size", 224)
        self.visual = VisionTransformer(**vision)
        self.textual = None
        self.log_scale = nn.Parameter(math.log(1 / 0.07) * torch.ones([]))


class WanImageEncoderEngine:
    def __init__(self, vit: VisionTransformer, device):
        nv.require_cuda(device, "the image encoder")
        self.device = torch.device(device)
        self.dim, self.H, self.hd = vit.dim, vit.num_heads, vit.dim // vit.num_heads
        self.image_size, self.patch, self.eps = vit.image_size, vit.patch_size, vit.norm_eps
        bf = lambda t: t.detach().to(device=self.device, dtype=torch.bfloat16).contiguous()
        f32 = lambda t: t.detach().to(device=self.device, dtype=torch.float32).contiguous()
        k = 3 * self.patch * self.patch
        self.kpad = (k + 7) // 8 * 8                                   # GEMM K must be a multiple of 8
        wp = torch.zeros(vit.dim, self.kpad, dtype=torch.float32)
        wp[:, :k] = vit.patch_embedding.weight.detach().float().reshape(vit.dim, k).cpu()
        self.w_patch = bf(wp)
        self.cls, self.pos = f32(vit.cls_embedding.reshape(1, -1)), f32(vit.pos_embedding[0])
        self.pre_w, self.pre_b = f32(vit.pre_norm.weight), f32(vit.pre_norm.bias)
        self.layers = []
        for b in vit.transformer:
            self.layers.append(dict(
                n1w=f32(b.norm1.weight), n1b=f32(b.norm1.bias), n2w=f32(b.norm2.weight), n2b=f32(b.norm2.bias),
                w_qkv=bf(b.attn.to_qkv.weight), b_qkv=f32(b.attn.to_qkv.bias), w_proj=bf(b.attn.proj.weight), b_proj=f32(b.attn.proj.bias),
                w_m0=bf(b.mlp[0].weight), b_m0=f32(b.mlp[0].bias), w_m2=bf(b.mlp[2].weight), b_m2=f32(b.mlp[2].bias)))
        self.mean = torch.tensor(CLIP_MEAN, device=self.device).view(1, 3, 1, 1)
        self.std = torch.tensor(CLIP_STD, device=self.device).view(1, 3, 1, 1)
        self.launches = 0

    def preprocess(self, image):
        """encode_image :866-875: f32 [1,3,H,W] in [-1,1] -> bicubic resize -> [0,1] -> mean/std normalisation."""
        x = F.interpolate(image.to(device=self.device, dtype=torch.float32), size=(self.image_size,) * 2, mode="bicubic",
                          align_corners=False)
        return (x * 0.5 + 0.5 - self.mean) / self.std

    def forward(self, pixels, skip_last=True):
        """pixels f32 [1,3,S,S] (already normalised) -> f32 [1, 1 + n_patches, dim]; skip_last = use_31_block (:474-476)."""
        dev, d, P = self.device, self.dim, self.patch
        n_side = self.image_size // P
        n = n_side * n_side
        # im2col of the stride-P patch conv: [n, 3*P*P] rows in (c, py, px) order = Conv2d weight layout
        cols = pixels[0].reshape(3, n_side, P, n_side, P).permute(1, 3, 0, 2, 4).reshape(n, 3 * P * P)
        a = torch.zeros(n, self.kpad, device=dev, dtype=torch.bfloat16)
        a[:, :3 * P * P] = cols.to(torch.bfloat16)
        L = n + 1
        tok = torch.empty(L, d, device=dev, dtype=torch.float32)
        tok[0] = self.cls[0] + self.pos[0]
        nv.gemm(a, self.w_patch, tok[1:], residual=self.pos[1:])          # patch embedding + position embedding
        x = torch.empty(L, d, device=dev, dtype=torch.float32)
        nv.layernorm_f32(tok, self.pre_w, self.pre_b, self.eps, x)
        h = torch.empty(L, d, device=dev, dtype=torch.bfloat16)
        qkv = torch.empty(L, 3 * d, device=dev, dtype=torch.bfloat16)
        att = torch.empty(L, d, device=dev, dtype=torch.bfloat16)
        m = torch.empty(L, self.layers[0]["w_m0"].shape[0], device=dev, dtype=torch.bfloat16)
        scale = 1.0 / math.sqrt(self.hd)
        for ly in (self.layers[:-1] if skip_last else self.layers):
            nv.layernorm_modulate(x, h, self.eps, gamma=ly["n1w"], beta=ly["n1b"])
            nv.gemm(h, ly["w_qkv"], qkv, bias=ly["b_qkv"])
            nv.attention_small(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], att, self.H, self.hd, scale)
            nv.gemm(att, ly["w_proj"], x, bias=ly["b_proj"], residual=x)
            nv.layernorm_modulate(x, h, self.eps, gamma=ly["n2w"], beta=ly["n2b"])
            nv.gemm(h, ly["w_m0"], m, bias=ly["b_m0"], act=nv.ACT_GELU_ERF)
            nv.gemm(m, ly["w_m2"], x, bias=ly["b_m2"], residual=x)
            self.launches += 7
        self.launches += 2
        return x.unsqueeze(0)


class WanImageEncoder(nn.Module):
    def __init__(self, **vision):
        super().__init__()
        self.model = _Clip(**vision)
        self._engine = None

    def engine(self, device=None):
        p = self.model.visual.patch_embedding.weight
        dev = torch.device(device) if device is not None else p.device
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        sig = (str(dev), p.data_ptr(), p._version, self.model.visual.transformer[-1].mlp[2].weight.data_ptr())
        if self._engine is None or self._engine[0] != sig:
            self._engine = (sig, WanImageEncoderEngine(self.model.visual, dev))
        return self._engine[1]

    def encode_image(self, videos):
        """list of f32 [1,3,H,W] images in [-1,1] -> [B, 257, 1280] in the parameter dtype (bf16 for float8 parameters,
        see wan_video_text_encoder.output_dtype) (reference :864-880)."""
        from .wan_video_text_encoder import output_dtype
        p = self.model.visual.patch_embedding.weight
        eng = self.engine(p.device)
        outs = [eng.forward(eng.preprocess(u)) for u in videos]
        return torch.cat(outs, dim=0).to(output_dtype(p.dtype))

    @staticmethod
    def state_dict_converter():
        return WanImageEncoderStateDictConverter()


class WanImageEncoderStateDictConverter:
    def from_diffusers(self, state_dict):
        return state_dict

    def from_civitai(self, state_dict):
        """reference :894-901: drop the text tower, prefix the rest with `model.`."""
        return {"model." + name: param for name, param in state_dict.items() if not name.startswith("textual.")}
