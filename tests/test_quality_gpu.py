"""GPU: the quality-metric entry points (include/svi_b200_quality.h) — attention against an fp64 reference, the other
kernels against their torch stand-ins on the same operands, argument checks that return a status — then the full-size
towers against the fp32 oracle, the four scorers' score() on tiny weights, and reproducibility across batch sizes."""
import ctypes
import os

import numpy as np
import pytest
import torch

import nv_emulation_quality as emu
from oracle import quality_oracle as O
from tools import synth_quality as S

pytestmark = pytest.mark.gpu

COVERED = {
    "svi_quality_attn": ["test_attn_matches_fp64", "test_attn_rejects_bad_arguments"],
    "svi_quality_stage_pixels": ["test_stage_pixels_exact", "test_small_kernels_reject_bad_arguments"],
    "svi_quality_embed_ln": ["test_embed_ln_matches_torch", "test_small_kernels_reject_bad_arguments"],
    "svi_quality_quick_gelu": ["test_quick_gelu_matches_torch"],
    "svi_quality_pool": ["test_pool_matches_torch", "test_small_kernels_reject_bad_arguments"],
    "svi_quality_score": ["test_score_matches_torch", "test_small_kernels_reject_bad_arguments"],
}
DEV = "cuda"


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _qkv(batch, L, heads, hd, seed, pad=0):
    d = heads * hd
    t = torch.randn(batch * L, 3 * d + pad, generator=_g(seed)).to(torch.bfloat16)
    return t


@pytest.mark.parametrize("hd,L,causal", [(64, 77, True), (80, 257, False), (64, 257, False), (80, 100, False),
                                         (64, 131, True), (80, 320, False), (64, 1, True)])
@pytest.mark.parametrize("batch", [1, 7, 81])
def test_attn_matches_fp64(hd, L, causal, batch):
    """every output within 2^-7 of the fp64 softmax(Q K^T s) V scale, mean error well below it (bf16 P, bf16 output)"""
    from diffsynth import _native as nv
    heads = 4 if hd == 80 else 3
    d = heads * hd
    qkv = _qkv(batch, L, heads, hd, seed=hd + L + batch, pad=8)
    qkv[:, :d] *= 3.0                                    # sharper softmax rows
    ref = torch.zeros(batch * L, d, dtype=torch.float64)
    emu.quality_attn(qkv[:, :d].double(), qkv[:, d:2 * d].double(), qkv[:, 2 * d:3 * d].double(), ref, batch, heads, hd,
                     hd ** -0.5, causal)
    q = qkv.to(DEV)
    out = torch.full((batch * L, d + 16), 7.0, device=DEV, dtype=torch.bfloat16)
    nv.quality_attn(q[:, :d], q[:, d:2 * d], q[:, 2 * d:3 * d], out[:, :d], batch, heads, hd, hd ** -0.5, causal)
    torch.cuda.synchronize()
    got = out.cpu()
    assert (got[:, d:].float() == 7.0).all(), "columns past the heads were written"
    err = (got[:, :d].double() - ref).abs()
    scale = ref.abs().max().item()
    assert err.max().item() <= 2 ** -7 * max(scale, 1.0), (err.max().item(), scale)
    assert err.mean().item() <= 2e-3 * max(scale, 1.0)


def _status(fn, *args):
    from diffsynth import _native as nv
    rc = getattr(nv.load(), fn)(*args)
    return rc, nv.load().svi_last_error().decode()


def test_attn_rejects_bad_arguments():
    from diffsynth import _native as nv
    qkv = torch.zeros(2 * 77, 3 * 128, device=DEV, dtype=torch.bfloat16)
    o = torch.zeros(2 * 77, 128, device=DEV, dtype=torch.bfloat16)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    good = [p(qkv), 384, p(qkv[:, 128:]), 384, p(qkv[:, 256:]), 384, p(o), 128, 2, 77, 2, 64, 0.125, 1, s]
    assert _status("svi_quality_attn", *good)[0] == 0
    for i, v, msg in ((11, 96, "head_dim"), (11, 48, "head_dim"), (9, 0, "L ="), (9, 321, "L ="), (8, 0, "batch"),
                      (1, 100, "leading"), (7, 127, "leading"), (3, 383, "even"), (12, 0.0, "scale"),
                      (12, float("inf"), "scale"), (6, p(qkv), "overlaps"), (0, None, "null")):
        args = list(good)
        args[i] = v
        rc, err = _status("svi_quality_attn", *args)
        assert rc < 0 and msg in err, (i, v, rc, err)
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="head_dim"):
        nv.quality_attn(qkv[:, :96], qkv[:, 96:192], qkv[:, 192:288], o[:, :96], 2, 1, 96, 0.1)


def test_stage_pixels_exact():
    from diffsynth import _native as nv
    px = torch.rand(5, 3, 42, 42, generator=_g(1)) * 1.2 - 0.1
    ms = torch.tensor([*O.OPENAI_MEAN, *O.OPENAI_STD])
    want = torch.empty(5 * 9, 592, dtype=torch.bfloat16)
    emu.quality_stage_pixels(px, ms, want, 14)
    got = torch.full((5 * 9, 592), 3.0, device=DEV, dtype=torch.bfloat16)
    nv.quality_stage_pixels(px.to(DEV), ms.to(DEV), got, 14)
    assert torch.equal(got.cpu(), want)


@pytest.mark.parametrize("D", [1280, 1024, 768, 160])
def test_embed_ln_matches_torch(D):
    from diffsynth import _native as nv
    g = _g(D)
    B, n = 3, 16
    patch, cls, pos = torch.randn(B * n, D, generator=g), torch.randn(D, generator=g), torch.randn(n + 1, D, generator=g)
    gam, bet = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    want = torch.empty(B * (n + 1), D)
    emu.quality_embed_ln(patch, cls, pos, gam, bet, 1e-5, want)
    got = torch.empty(B * (n + 1), D, device=DEV)
    nv.quality_embed_ln(*(t.to(DEV) for t in (patch, cls, pos, gam, bet)), 1e-5, got)
    torch.testing.assert_close(got.cpu(), want, rtol=1e-5, atol=2e-5)


def test_quick_gelu_matches_torch():
    from diffsynth import _native as nv
    x = torch.randn(37, 200, generator=_g(3)) * 4
    x[0, :4] = torch.tensor([-100.0, 100.0, 0.0, -0.0])
    want = torch.empty(37, 192, dtype=torch.bfloat16)
    emu.quality_quick_gelu(x[:, :192], want)
    got = torch.zeros(37, 256, device=DEV, dtype=torch.bfloat16)
    nv.quality_quick_gelu(x.to(DEV)[:, :192], got[:, :192])
    diff = (got[:, :192].cpu().float() - want.float()).abs()
    assert (diff <= 2 ** -7 * want.float().abs()).all()        # one bf16 ulp at most (f32 exp differs in the last bits)
    assert (got[:, 192:] == 0).all()


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_pool_matches_torch(mode):
    from diffsynth import _native as nv
    n_seq, L, D = 5, 77, 96
    x = torch.randn(n_seq * L, D + 4, generator=_g(mode))
    ids = torch.randint(1, 500, (n_seq, L), generator=_g(10 + mode))
    ids[1, 30:] = 0                                            # padded prompt: argmax and first eos agree on 29
    ids[1, 29] = 999
    ids[2, 40], ids[2, 50] = 999, 999                          # two maxima: the first one
    ids[3] = 5                                                 # no eos at all: row 0 in mode 2
    want = torch.empty(n_seq, D)
    emu.quality_pool(x[:, :D], n_seq, want, mode, ids, 999)
    got = torch.empty(n_seq, D, device=DEV)
    nv.quality_pool(x.to(DEV)[:, :D], n_seq, got, mode, ids.to(DEV) if mode else None, 999)
    assert torch.equal(got.cpu(), want)


@pytest.mark.parametrize("T,head", [(1, False), (3, True), (0, True)])
def test_score_matches_torch(T, head):
    from diffsynth import _native as nv
    B, E = 81, 768
    img, txt = torch.randn(B, E, generator=_g(5)), torch.randn(max(T, 1), E, generator=_g(6))[:T]
    w = torch.randn(E, generator=_g(7)) if head else None
    cw, aw = (torch.empty(B, T) if T else None), (torch.empty(B) if head else None)
    emu.quality_score(img, txt if T else None, cw, w, 0.25, aw)
    cg = torch.empty(B, T, device=DEV) if T else None
    ag = torch.empty(B, device=DEV) if head else None
    nv.quality_score(img.to(DEV), txt.to(DEV) if T else None, cg, w.to(DEV) if head else None, 0.25, ag)
    if T:
        torch.testing.assert_close(cg.cpu(), cw, rtol=0, atol=2e-6)
    if head:
        torch.testing.assert_close(ag.cpu(), aw, rtol=1e-5, atol=1e-5)


def test_small_kernels_reject_bad_arguments():
    f = torch.zeros(64, 64, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for fn, args, msg in (
            ("svi_quality_stage_pixels", [p(f), 1, 30, 14, p(f), p(f), 592, s], "multiple of P"),
            ("svi_quality_stage_pixels", [p(f), 1, 28, 14, p(f), p(f), 500, s], "kpad"),
            ("svi_quality_embed_ln", [p(f), p(f), p(f), 1, 4, 6, 1e-5, p(f), p(f), p(f[32:]), s], "multiple of 4"),
            ("svi_quality_embed_ln", [p(f), p(f), p(f), 1, 4, 8, 1e-5, p(f), p(f), p(f), s], "overlaps"),
            ("svi_quality_pool", [p(f), 64, 2, 32, 64, None, 1, 0, p(f), s], "needs ids"),
            ("svi_quality_pool", [p(f), 64, 2, 32, 64, None, 5, 0, p(f), s], "mode"),
            ("svi_quality_score", [p(f), 4, None, 1, 64, None, 0.0, p(f), None, s], "txt"),
            ("svi_quality_score", [p(f), 4, None, 0, 64, None, 0.0, None, None, s], "nothing"),
            ("svi_quality_quick_gelu", [p(f), 10, 4, 16, p(f), 16, s], "ldx")):
        rc, err = _status(fn, *args)
        assert rc < 0 and msg in err, (fn, rc, err)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ full-size towers
def _rel(got, want):
    return (got - want).abs().mean().item() / want.std().item()


@pytest.fixture(scope="module")
def fp32_oracle():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = False


def _pixels(n, size, seed):
    from diffsynth.extensions.ImageQualityMetric import towers as T
    return torch.stack([T.openclip_pixels(f, size) for f in S.frames(n, 480, 832, seed=seed)])


def test_full_size_openclip_vit_h_14(fp32_oracle):
    from diffsynth.extensions.ImageQualityMetric import towers as T
    cfg = S.OPENCLIP_FULL
    sd = S.openclip_state_dict(cfg, seed=11)
    m = T.OpenCLIP(**cfg)
    m.load_state_dict(sd, strict=True)
    eng = m.engine(DEV)
    px = _pixels(4, 224, seed=12)
    ids = torch.randint(1, 49000, (2, 77), generator=_g(13))
    ids[0, 20], ids[0, 21:] = 49407, 0
    ids[1, 76] = 49407
    img, txt = eng.vision.encode_images(px), eng.text.encode_text(ids)
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        r_img = O.openclip_image(sdd, cfg, O.normalize(px).to(DEV))
        r_txt = O.openclip_text(sdd, cfg, ids.to(DEV))
    ei, et = _rel(img, r_img), _rel(txt, r_txt)
    cos = torch.empty(4, 2, device=DEV)
    from diffsynth import _native as nv
    nv.quality_score(img, txt, cos)
    ec = (cos - O.cosine(r_img, r_txt)).abs().max().item()
    print(f"open_clip ViT-H-14: image features {ei:.4%} of std, text {et:.4%}, |cos err| max {ec:.2e}")
    assert ei < 0.02 and et < 0.02 and ec < 5e-3


@pytest.mark.parametrize("which", ["pick", "large"])
def test_full_size_hf_towers(which, fp32_oracle):
    from diffsynth.extensions.ImageQualityMetric import towers as T
    conf = S.HF_FULL_PICK if which == "pick" else S.HF_FULL_LARGE
    sd = S.hf_state_dict(conf, seed=21)
    m = T.HFCLIPModel(conf)
    m.load_state_dict(sd, strict=True)
    eng = m.engine(DEV)
    px = _pixels(4, 224, seed=22)
    ids = torch.randint(1, 49000, (1, 19), generator=_g(23))
    ids[0, 0], ids[0, -1] = 49406, 49407
    img, txt = eng.vision.encode_images(px), eng.text.encode_text(ids)
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        r_img = O.hf_image(sdd, conf, O.normalize(px).to(DEV))
        r_txt = O.hf_text(sdd, conf, ids.to(DEV))
    ei, et = _rel(img, r_img), _rel(txt, r_txt)
    ec = (O.cosine(img, txt) - O.cosine(r_img, r_txt)).abs().max().item()
    print(f"CLIPModel {which}: image features {ei:.4%} of std, text {et:.4%}, |cos err| max {ec:.2e}")
    assert ei < 0.02 and et < 0.02 and ec < 5e-3


# ------------------------------------------------------------------------------------------------ the scorers
@pytest.fixture(scope="module")
def tiny_paths(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("quality"))
    return S.write_tiny_checkpoints(d)


def _tiny_frames(n):
    return [S.frames(1, h, w, seed=i)[0] for i, (h, w) in enumerate([(40, 70), (71, 33), (97, 120)] * (n // 3 + 1))][:n]


@pytest.mark.parametrize("name", ["CLIP", "HPSv2", "HPSv2.1", "PickScore", "Aesthetic"])
def test_scorers_against_oracle(name, tiny_paths):
    from diffsynth.extensions.ImageQualityMetric import load_preference_model
    paths, ref = tiny_paths
    model = load_preference_model(name, device=DEV, path=paths)
    frames = _tiny_frames(5)
    got = model.score(frames, S.PROMPTS[1])
    want = S.oracle_scores(name, paths, ref, frames, S.PROMPTS[1])
    err = np.abs(np.array(got) - np.array(want)).max()
    print(f"{name}: |score err| max {err:.2e}")
    assert len(got) == 5 and err < (2e-2 if name == "Aesthetic" else 5e-3)
    assert model.score(frames[0], S.PROMPTS[1]) == got[:1]
    if name == "PickScore":
        assert model.score(frames, S.PROMPTS[1], softmax=True) == [1.0] * 5


def test_score_is_batch_and_run_invariant(tiny_paths):
    from diffsynth.extensions.ImageQualityMetric import load_preference_model
    paths, _ = tiny_paths
    model = load_preference_model("CLIP", device=DEV, path=paths)
    frames = _tiny_frames(81)
    alone = model.score(frames[4], "a cat")[0]
    seven = model.score(frames[:7], "a cat")[4]
    all81 = model.score(frames, "a cat")
    again = model.score(frames, "a cat")
    assert alone == seven == all81[4] and all81 == again
    model.model.engine(DEV).vision.chunk = 16
    assert model.score(frames, "a cat") == all81
