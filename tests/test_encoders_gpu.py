"""GPU: the conditioning encoders on the native kernels (svi_gemm_bf16 + csrc/encoder_kernels.cu) against the CPU oracle
(oracle/wan_encoders_oracle.py, itself pinned to the reference modules by tests/golden/enc_tiny.npz).

Two yardsticks per encoder, both on bf16-rounded weights:
  * the fp32 oracle — the parity statement: mean |error| < 1.5 % of the output's standard deviation.  (bf16 operands
    with fp32 accumulation and an fp32 residual stream; the reference runs these encoders with bf16 residuals too.)
  * the same oracle with `bf16_points=True`, which rounds exactly where the native path stores bf16 tensors — the
    implementation check: what is left is accumulation order and exp/tanh approximations, so at the tiny sizes >= 85 %
    of the elements must agree to rtol 1e-2 / atol 1e-3 with a mean error below 0.4 % of the standard deviation
    (on an H100: 100 % inside, mean error <= 0.12 % of the std); at the real widths the long fp32 sums flip bf16 roundings and the bound is statistical."""
import math

import pytest
import torch

from tools import synth_enc as SE

pytestmark = pytest.mark.gpu


def _bf(sd):
    return {k: v.to(torch.bfloat16).float() for k, v in sd.items()}


def _stats(out, ref):
    err = (out - ref).abs()
    inside = (err <= 1e-3 + 1e-2 * ref.abs()).float().mean().item()
    return inside, err.max().item(), err.mean().item() / ref.std().item()


def test_attention_small_bias_mask_and_head_widths():
    """svi_attn_small vs torch: head widths 64 (umT5) / 80 (CLIP) / 128, ragged lengths, bucketed bias, key mask."""
    from diffsynth import _native as nv
    from diffsynth.models.wan_video_text_encoder import relative_position_buckets
    g = torch.Generator().manual_seed(0)
    for (Lq, Lk, H, hd, use_bias, n_valid) in [(24, 24, 2, 64, True, 17), (257, 257, 3, 80, False, None), (100, 77, 2, 128, False, 50),
                                               (512, 512, 4, 64, True, 300), (33, 65, 1, 16, True, None)]:
        q, k, v = (torch.randn(L, H * hd, generator=g).to(torch.bfloat16) for L in (Lq, Lk, Lk))
        scale = 1.0 if use_bias else 1.0 / math.sqrt(hd)
        table = torch.randn(32, H, generator=g) if use_bias else None
        bucket = relative_position_buckets(Lq, Lk, 32) if use_bias else None
        mask = None
        if n_valid is not None:
            mask = torch.zeros(Lk, dtype=torch.int32)
            mask[:n_valid] = 1
        out = torch.empty(Lq, H * hd, device="cuda", dtype=torch.bfloat16)
        nv.attention_small(q.cuda(), k.cuda(), v.cuda(), out, H, hd, scale,
                           bias_table=None if table is None else table.cuda(), bucket=None if bucket is None else bucket.cuda(),
                           key_mask=None if mask is None else mask.cuda())
        qf, kf, vf = (t.float().view(-1, H, hd).transpose(0, 1) for t in (q, k, v))
        s = qf @ kf.transpose(-1, -2) * scale
        if use_bias:
            s = s + table[bucket.long()].permute(2, 0, 1)
        if mask is not None:
            s = s.masked_fill(mask.view(1, 1, -1) == 0, float("-inf"))
        ref = (torch.softmax(s, dim=-1) @ vf).transpose(0, 1).reshape(Lq, H * hd)
        err = (out.float().cpu() - ref).abs().max().item()
        assert err < 2e-2, (Lq, Lk, H, hd, err)


def test_row_kernels_of_the_encoders():
    from diffsynth import _native as nv
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(37, 4096, generator=g) * 3).cuda()
    w = torch.randn(4096, generator=g).cuda()
    out = torch.empty(37, 4096, device="cuda", dtype=torch.bfloat16)
    nv.rmsnorm_affine(x, w, 1e-6, out)
    ref = w * x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6)
    assert (out.float() - ref).abs().max().item() < 2e-2 * ref.abs().max().item()
    x2 = torch.randn(10, 160, generator=g).cuda() + 0.5
    gam, bet = torch.randn(160, generator=g).cuda(), torch.randn(160, generator=g).cuda()
    y = torch.empty_like(x2)
    nv.layernorm_f32(x2, gam, bet, 1e-5, y)
    assert (y - torch.nn.functional.layer_norm(x2, (160,), gam, bet, 1e-5)).abs().max().item() < 1e-4
    table = torch.randn(50, 64, generator=g).to(torch.bfloat16).cuda()
    ids = torch.tensor([3, 0, 49, 7], dtype=torch.int64).cuda()
    emb = torch.empty(4, 64, device="cuda")
    nv.embedding_gather(ids, table, emb)
    assert torch.equal(emb, table[ids].float())
    a, b = (torch.randn(33, 64, generator=g).to(torch.bfloat16).cuda() for _ in range(2))
    c = torch.empty_like(a)
    nv.mul_bf16(a, b, c)
    assert torch.equal(c, (a.float() * b.float()).to(torch.bfloat16))


def _text_case(cfg, seq_len, valid, seed):
    from diffsynth.models.wan_video_text_encoder import WanTextEncoder
    from oracle import wan_encoders_oracle as E
    sd = _bf(SE.make_text_state_dict(cfg, seed=seed))
    ids, mask = SE.make_text_inputs(cfg, seq_len=seq_len, valid=valid, seed=seed)
    m = WanTextEncoder(**cfg).eval()
    m.load_state_dict(sd)
    m.to(device="cuda", dtype=torch.bfloat16)
    out = m(ids.cuda(), mask.cuda()).float().cpu()
    ref = E.text_encode(sd, cfg, ids, mask)
    emu = E.text_encode(sd, cfg, ids, mask, bf16_points=True)
    return out[:, :valid], ref[:, :valid], emu[:, :valid], m, ids, mask


def _check(name, out, ref, emu, emu_inside=0.85, emu_rel=4e-3):
    inside, mx, rel = _stats(out, ref)
    inside_e, mx_e, rel_e = _stats(out, emu)
    print(f"{name}: vs fp32 oracle inside={inside:.4f} max={mx:.4e} mean/std={rel:.4e} | vs bf16-point oracle "
          f"inside={inside_e:.4f} max={mx_e:.4e} mean/std={rel_e:.4e}")
    assert rel < 1.5e-2 and inside_e > emu_inside and rel_e < emu_rel


def test_tiny_text_encoder_matches_oracle_and_prompter_zero_fills():
    from diffsynth.prompters import WanPrompter
    out, ref, emu, m, ids, mask = _text_case(SE.TEXT_TINY, 24, 17, 0)
    _check("tiny umT5", out, ref, emu)
    p = WanPrompter()
    p.fetch_models(m)
    emb = p.encode_ids(ids, mask, device="cuda")
    assert emb.shape == (1, 24, SE.TEXT_TINY["dim"]) and float(emb[:, 17:].abs().max()) == 0.0
    assert torch.equal(emb[:, :17].float().cpu(), out.to(torch.bfloat16).float())


def test_tiny_image_encoder_matches_oracle():
    from diffsynth.models.wan_video_image_encoder import WanImageEncoder
    from oracle import wan_encoders_oracle as E
    cfg = SE.CLIP_TINY
    sd = _bf(SE.make_clip_state_dict(cfg, seed=0))
    m = WanImageEncoder(**cfg).eval()
    m.load_state_dict({**sd, "model.log_scale": torch.tensor(2.6593)})
    m.to(device="cuda", dtype=torch.bfloat16)
    img = SE.make_clip_image(50, 70, seed=0)
    out = m.encode_image([img.cuda()]).float().cpu()
    ref = E.image_encode(sd, cfg, img, SE.CLIP_MEAN, SE.CLIP_STD)
    emu = E.image_encode(sd, cfg, img, SE.CLIP_MEAN, SE.CLIP_STD, bf16_points=True)
    assert out.shape == (1, 10, cfg["dim"])
    _check("tiny CLIP ViT", out, ref, emu)


@pytest.mark.slow
def test_umt5_width_two_layers_matches_oracle():
    """Real widths (d 4096, 64 heads x 64, ffn 10240), 512 tokens with 300 valid, 2 layers, small vocabulary."""
    cfg = dict(SE.TEXT_UMT5_XXL, vocab=1000, num_layers=2)
    out, ref, emu, *_ = _text_case(cfg, 512, 300, 3)
    # K = 4096 / 10240 sums: a different fp32 accumulation order flips bf16 roundings in ~1/3 of the stored elements, so
    # the bf16-point oracle is only reproduced statistically at this width (on an H100: 0.66 / 5.5e-3)
    _check("umT5-width 2 layers", out, ref, emu, emu_inside=0.5, emu_rel=8e-3)


@pytest.mark.slow
def test_clip_vit_h_width_matches_oracle():
    """Real widths (1280, 16 heads x 80, mlp 5120, 224 px / 14 = 257 tokens), 3 layers (2 run: use_31_block)."""
    from diffsynth.models.wan_video_image_encoder import WanImageEncoder
    from oracle import wan_encoders_oracle as E
    cfg = dict(SE.CLIP_VIT_H, num_layers=3)
    sd = _bf(SE.make_clip_state_dict(cfg, seed=4))
    m = WanImageEncoder(**cfg).eval()
    m.load_state_dict({**sd, "model.log_scale": torch.tensor(2.6593)})
    m.to(device="cuda", dtype=torch.bfloat16)
    img = SE.make_clip_image(480, 832, seed=4)
    out = m.encode_image([img.cuda()]).float().cpu()
    ref = E.image_encode(sd, cfg, img, SE.CLIP_MEAN, SE.CLIP_STD)
    emu = E.image_encode(sd, cfg, img, SE.CLIP_MEAN, SE.CLIP_STD, bf16_points=True)
    assert out.shape == (1, 257, 1280)
    _check("CLIP ViT-H width", out, ref, emu, emu_inside=0.7, emu_rel=6e-3)      # on an H100: 0.82 / 2.9e-3
