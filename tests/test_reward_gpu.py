"""GPU: the cross-attention scorers' entry points (include/svi_b200_reward.h) — attention against an fp64 reference, the
other kernels against their torch stand-ins on the same operands, argument checks that return a status — then the
full-size ImageReward and MPS models against the fp32 oracle, both scorers on tiny weights, reproducibility across batch
sizes and chunking, and project-then-pool against pool-then-project on the existing text towers."""
import ctypes

import numpy as np
import pytest
import torch

import nv_emulation_reward as emu
from oracle import reward_oracle as O
from tools import synth_quality as SQ
from tools import synth_reward as R

pytestmark = pytest.mark.gpu

COVERED = {
    "svi_reward_attn": ["test_attn_matches_fp64", "test_attn_rejects_bad_arguments"],
    "svi_reward_layernorm": ["test_layernorm_matches_torch", "test_small_kernels_reject_bad_arguments"],
    "svi_reward_embed": ["test_embed_exact", "test_small_kernels_reject_bad_arguments"],
    "svi_reward_swiglu": ["test_swiglu_matches_torch", "test_small_kernels_reject_bad_arguments"],
    "svi_reward_rope": ["test_rope_exact", "test_small_kernels_reject_bad_arguments"],
    "svi_reward_cond_mask": ["test_cond_mask_matches_torch"],
    "svi_reward_head": ["test_head_matches_torch", "test_small_kernels_reject_bad_arguments"],
}
DEV = "cuda"


def _g(seed):
    return torch.Generator().manual_seed(seed)


# (Lq, Lk, heads, kv_heads, shared K/V, mask): BERT self (padding), BERT cross, MPS cross (multi-query, masked, one
# context), MPS self (multi-query), odd lengths, a first key chunk that is entirely masked
CASES = [(35, 35, 12, 12, False, "pad"), (35, 197, 12, 12, False, None), (257, 77, 16, 1, True, "shared"),
         (257, 257, 16, 1, False, None), (37, 101, 3, 3, False, "pad"), (1, 5, 2, 1, False, "pad"),
         (130, 77, 2, 1, True, "late")]


def _mask(kind, batch, Lk, seed):
    g = _g(seed)
    if kind == "pad":
        m = torch.zeros(batch, Lk, dtype=torch.uint8)
        for b in range(batch):
            m[b, :int(torch.randint(1, Lk + 1, (1,), generator=g))] = 1
        return m
    if kind == "shared":
        m = (torch.rand(Lk, generator=g) > 0.3).to(torch.uint8)
        m[0] = 0
        m[5] = 1
        return m
    if kind == "late":
        m = torch.zeros(Lk, dtype=torch.uint8)
        m[70:] = 1
        return m
    return None


@pytest.mark.parametrize("Lq,Lk,heads,kv_heads,shared,mask", CASES)
@pytest.mark.parametrize("batch", [1, 7, 81])
def test_attn_matches_fp64(Lq, Lk, heads, kv_heads, shared, mask, batch):
    """every output within 2^-7 of the fp64 masked softmax(Q K^T s) V scale, mean error well below it"""
    from diffsynth import _native as nv
    seed = Lq + 3 * Lk + batch
    q = (3.0 * torch.randn(batch * Lq, heads * 64 + 8, generator=_g(seed))).to(torch.bfloat16)
    kv_rows = Lk if shared else batch * Lk
    kv = torch.randn(kv_rows, 2 * kv_heads * 64 + 8, generator=_g(seed + 1)).to(torch.bfloat16)
    w = kv_heads * 64
    km = _mask(mask, batch, Lk, seed + 2)
    ref = torch.zeros(batch * Lq, heads * 64, dtype=torch.float64)
    emu.reward_attn(q.double(), kv[:, :w].double(), kv[:, w:2 * w].double(), ref, batch, heads, 0.125, kv_heads, shared, km)
    qd, kvd = q.to(DEV), kv.to(DEV)
    out = torch.full((batch * Lq, heads * 64 + 16), 7.0, device=DEV, dtype=torch.bfloat16)
    nv.reward_attn(qd[:, :heads * 64], kvd[:, :w], kvd[:, w:2 * w], out[:, :heads * 64], batch, heads, 0.125, kv_heads,
                   shared, km.to(DEV) if km is not None else None)
    torch.cuda.synchronize()
    got = out.cpu()
    assert (got[:, heads * 64:].float() == 7.0).all(), "columns past the heads were written"
    err = (got[:, :heads * 64].double() - ref).abs()
    scale = ref.abs().max().item()
    assert torch.isfinite(got.float()).all()
    assert err.max().item() <= 2 ** -7 * max(scale, 1.0), (err.max().item(), scale)
    assert err.mean().item() <= 2e-3 * max(scale, 1.0)


def _status(fn, *args):
    from diffsynth import _native as nv
    rc = getattr(nv.load(), fn)(*args)
    return rc, nv.load().svi_last_error().decode()


def test_attn_rejects_bad_arguments():
    from diffsynth import _native as nv
    q = torch.zeros(2 * 35, 128, device=DEV, dtype=torch.bfloat16)
    kv = torch.zeros(2 * 197, 256, device=DEV, dtype=torch.bfloat16)
    o = torch.zeros(2 * 35, 128, device=DEV, dtype=torch.bfloat16)
    m = torch.ones(2, 197, device=DEV, dtype=torch.uint8)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    good = [p(q), 128, p(kv), 256, p(kv[:, 128:]), 256, p(o), 128, 2, 35, 197, 2, 2, 197, p(m), 197, 0.125, s]
    assert _status("svi_reward_attn", *good)[0] == 0
    for i, v, msg in ((9, 0, "Lq ="), (10, 321, "Lk ="), (8, 0, "batch"), (12, 3, "kv_heads"), (13, 100, "kv_batch_stride"),
                      (15, 50, "mask_batch_stride"), (1, 64, "leading"), (3, 127, "leading"), (16, 0.0, "scale"),
                      (6, p(q), "overlaps"), (0, None, "null")):
        args = list(good)
        args[i] = v
        rc, err = _status("svi_reward_attn", *args)
        assert rc < 0 and msg in err, (i, v, rc, err)
    torch.cuda.synchronize()


@pytest.mark.parametrize("D,inplace", [(768, True), (128, False), (1024, True)])
def test_layernorm_matches_torch(D, inplace):
    from diffsynth import _native as nv
    g = _g(D)
    x = 3 * torch.randn(70, D, generator=g) + 1
    gam, bet = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    wy, wb = torch.empty(70, D), torch.empty(70, D, dtype=torch.bfloat16)
    emu.reward_layernorm(x, gam, bet, 1e-12, wy, wb)
    xd = x.to(DEV)
    y = xd if inplace else torch.empty_like(xd)
    yb = torch.empty(70, D, device=DEV, dtype=torch.bfloat16)
    nv.reward_layernorm(xd, gam.to(DEV), bet.to(DEV), 1e-12, y, yb)
    torch.testing.assert_close(y.cpu(), wy, rtol=1e-5, atol=2e-5)
    assert torch.equal(yb.cpu(), y.cpu().to(torch.bfloat16))
    assert ((yb.cpu().float() - wb.float()).abs() <= 2 ** -7 * wb.float().abs() + 1e-6).all()


def test_embed_exact():
    from diffsynth import _native as nv
    g = _g(2)
    B, n, D = 3, 196, 192
    patch, cls, pos = torch.randn(B * n, D, generator=g), torch.randn(D, generator=g), torch.randn(n + 1, D, generator=g)
    want = torch.empty(B * (n + 1), D)
    emu.reward_embed(patch, cls, pos, want)
    got = torch.empty(B * (n + 1), D, device=DEV)
    nv.reward_embed(patch.to(DEV), cls.to(DEV), pos.to(DEV), got)
    assert torch.equal(got.cpu(), want)


def test_swiglu_matches_torch():
    from diffsynth import _native as nv
    x = 4 * torch.randn(37, 2 * 96 + 8, generator=_g(3))
    x[0, :4] = torch.tensor([-100.0, 100.0, 0.0, -0.0])
    want = torch.empty(37, 96, dtype=torch.bfloat16)
    emu.reward_swiglu(x[:, :192], want)
    got = torch.zeros(37, 128, device=DEV, dtype=torch.bfloat16)
    nv.reward_swiglu(x.to(DEV)[:, :192], got[:, :96])
    diff = (got[:, :96].cpu().float() - want.float()).abs()
    assert (diff <= 2 ** -7 * want.float().abs() + 1e-30).all()        # one bf16 ulp at most (f32 exp)
    assert (got[:, 96:] == 0).all()


def test_rope_exact():
    from diffsynth import _native as nv
    from diffsynth.extensions.ImageQualityMetric.reward import rope_tables
    L, heads = 257, 17
    x = torch.randn(2 * L, heads * 64 + 64, generator=_g(4)).to(torch.bfloat16)
    cos, sin = rope_tables(L)
    want = x.clone()
    emu.reward_rope(want[:, :heads * 64], L, cos, sin)
    got = x.to(DEV)
    nv.reward_rope(got[:, :heads * 64], L, cos.to(DEV), sin.to(DEV))
    assert torch.equal(got.cpu(), want)


def test_cond_mask_matches_torch():
    from diffsynth import _native as nv
    g = _g(5)
    text = torch.randn(77, 1024, generator=g) * torch.linspace(-0.2, 1.0, 77)[:, None]   # ratios spread across 0.3
    cond = torch.randn(77, 1024, generator=g)
    wr, wk = torch.empty(77), torch.empty(77, dtype=torch.uint8)
    emu.reward_cond_mask(text, cond, 0.3, wr, wk)
    r, k = torch.empty(77, device=DEV), torch.empty(77, device=DEV, dtype=torch.uint8)
    nv.reward_cond_mask(text.to(DEV), cond.to(DEV), 0.3, r, k)
    torch.testing.assert_close(r.cpu(), wr, rtol=1e-5, atol=1e-5)
    far = (wr - 0.3).abs() > 1e-3
    assert torch.equal(k.cpu()[far], wk[far]) and 0 < int(wk.sum()) < 77


def test_head_matches_torch():
    from diffsynth import _native as nv
    x = torch.randn(5 * 35, 768 + 4, generator=_g(6))
    w = torch.randn(768, generator=_g(7))
    want = torch.empty(5)
    emu.reward_head(x[:, :768], 5, w, 0.25, want)
    got = torch.empty(5, device=DEV)
    nv.reward_head(x.to(DEV)[:, :768], 5, w.to(DEV), 0.25, got)
    torch.testing.assert_close(got.cpu(), want, rtol=1e-5, atol=1e-4)


def test_small_kernels_reject_bad_arguments():
    f = torch.zeros(64, 64, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for fn, args, msg in (
            ("svi_reward_layernorm", [p(f), 4, 6, 1e-5, p(f), p(f), p(f), p(f[32:]), s], "multiple of 4"),
            ("svi_reward_layernorm", [p(f), 4, 8, 1e-5, p(f), p(f), p(f), p(f), s], "yb overlaps"),
            ("svi_reward_embed", [p(f), p(f), p(f), 1, 4, 8, p(f), s], "overlaps patch"),
            ("svi_reward_swiglu", [p(f), 10, 4, 8, p(f), 8, s], "ldx"),
            ("svi_reward_rope", [p(f), 100, 4, 4, 2, p(f), p(f), s], "ldx"),
            ("svi_reward_head", [p(f), 8, 2, 4, 16, p(f), 0.0, p(f), s], "ldx"),
            ("svi_reward_head", [p(f), 64, 2, 4, 16, None, 0.0, p(f), s], "null")):
        rc, err = _status(fn, *args)
        assert rc < 0 and msg in err, (fn, rc, err)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ full-size models
def _rel(got, want):
    return (got - want).abs().mean().item() / want.std().item()


@pytest.fixture(scope="module")
def fp32_oracle():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def _frames_px(n, seed, fn):
    return torch.stack([fn(f) for f in SQ.frames(n, 480, 832, seed=seed)])


def test_full_size_imagereward(fp32_oracle):
    from diffsynth.extensions.ImageQualityMetric import towers as T
    from diffsynth.extensions.ImageQualityMetric.reward import ImageRewardEngine, ImageRewardModel
    sd = R.imagereward_state_dict(R.FULL_MED, R.FULL_VISION, seed=51, extra=False)
    with torch.device("meta"):
        m = ImageRewardModel(R.FULL_MED, **R.FULL_VISION)
    m.load_state_dict(sd, strict=True, assign=True)
    eng = ImageRewardEngine(m, DEV)
    px = _frames_px(4, 52, lambda f: T.blip_pixels(f, 224))
    ids = torch.randint(1000, 30000, (1, 35), generator=_g(53))
    ids[0, 0], ids[0, 20], ids[0, 21:] = 101, 102, 0
    mask = (ids != 0).long()
    got = eng.score(px, ids, mask).cpu()
    x0, _, _ = eng.prompt_states(ids, mask)
    img_states = eng.vision.image_states(px.to(DEV))
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        r_img, r_cls, r_score = O.imagereward(sdd, R.FULL_MED, 24, O.Q.normalize(px.to(DEV)), ids.to(DEV), mask.to(DEV))
        r_states = O.blip_image_states(sdd, O.Q.normalize(px.to(DEV)), 24)
    ctx = torch.empty(img_states.shape, device=DEV, dtype=torch.bfloat16)
    from diffsynth import _native as nv
    nv.layernorm_modulate(img_states, ctx, 1e-6, gamma=eng.vnorm[0], beta=eng.vnorm[1])
    ei = _rel(ctx.float().view(4, 197, -1), r_states)
    es = (got - r_score.cpu()).abs().max().item()
    print(f"ImageReward ViT-L/16 + BERT-base: image states {ei:.4%} of std, |reward err| max {es:.3e} "
          f"(reward std {r_score.std().item():.3e})")
    assert ei < 0.02 and es < 0.05


def test_full_size_mps(fp32_oracle):
    from diffsynth.extensions.ImageQualityMetric import towers as T
    from diffsynth.extensions.ImageQualityMetric.reward import CrossModel, MPSEngine, MPSModel
    conf = SQ.HF_FULL_PICK
    sd = R.mps_state_dict(conf, layers=4, seed=61)
    sd = {k: v for k, v in sd.items() if "inv_freq" not in k}
    with torch.device("meta"):
        m = MPSModel(conf, CrossModel.sizes(sd))
    m.load_state_dict(sd, strict=True, assign=True)
    mean, std = O.Q.OPENAI_MEAN, O.Q.OPENAI_STD
    eng = MPSEngine(m, DEV, mean, std)
    px = _frames_px(4, 62, lambda f: T.openclip_pixels(f, 224))
    ids = torch.randint(1, 49000, (1, 77), generator=_g(63))
    ids[0, 0], ids[0, 15], ids[0, 16:] = 49406, 49407, 49407
    cids = torch.randint(1, 49000, (1, 77), generator=_g(64))
    cids[0, 0], cids[0, 40], cids[0, 41:] = 49406, 49407, 49407
    got = eng.score(px, ids, cids)
    tb, eos, keep, ratio = eng.prompt(ids, cids)
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        r = O.mps(sdd, conf, 16, 4, O.Q.normalize(px.to(DEV)), ids.to(DEV), cids.to(DEV))
    et = _rel(tb.float(), r["text_f"])
    far = (r["ratio"] - 0.3).abs() > 1e-3
    near = int((~far).sum())
    assert torch.equal(keep.bool()[far], r["keep"][far]), "mask differs on a key far from the threshold"
    es = (got - r["scores"].cpu()).abs().max().item()
    print(f"MPS ViT-H/14 + cross model: text rows {et:.4%} of std, keys kept {int(keep.sum())}/77, "
          f"{near} keys within 1e-3 of the threshold, |score err| max {es:.3e} (score scale {r['scores'].abs().max().item():.3e})")
    assert et < 0.02 and es < 0.05 * max(1.0, r["scores"].abs().max().item())


# ------------------------------------------------------------------------------------------------ the scorers
@pytest.fixture(scope="module")
def tiny_paths(tmp_path_factory):
    return R.write_reward_checkpoints(str(tmp_path_factory.mktemp("reward")))


def _tiny_frames(n):
    return [SQ.frames(1, h, w, seed=i)[0] for i, (h, w) in enumerate([(240, 320), (300, 224), (97, 120)] * (n // 3 + 1))][:n]


@pytest.mark.parametrize("name", ["ImageReward", "MPS"])
def test_scorers_against_oracle_and_batch_invariant(name, tiny_paths):
    import test_reward_cpu as C
    from diffsynth.extensions.ImageQualityMetric import load_preference_model
    paths, ref = tiny_paths
    model = load_preference_model(name, device=DEV, path=paths)
    frames = _tiny_frames(5)
    prompt = R.PROMPTS[0] if name == "ImageReward" else R.PROMPTS[2]
    got = model.score(frames, prompt)
    want = (C._oracle_imagereward if name == "ImageReward" else C._oracle_mps)(paths, ref, frames, prompt)
    err = np.abs(np.array(got) - np.array(want)).max()
    print(f"{name}: |score err| max {err:.2e}")
    assert len(got) == 5 and err < 3e-2 * max(1.0, np.abs(want).max())
    many = _tiny_frames(81)
    alone = model.score(many[4], prompt)[0]
    seven = model.score(many[:7], prompt)[4]
    all81 = model.score(many, prompt)
    assert alone == seven == all81[4] and model.score(many, prompt) == all81
    eng = model.engine()
    eng.chunk = eng.vision.chunk = 16
    assert model.score(many, prompt) == all81


def test_project_then_pool_equals_pool_then_project():
    from diffsynth.extensions.ImageQualityMetric import towers as T
    V = 600
    oc = T.OpenCLIP(**SQ.openclip_tiny(V))
    oc.load_state_dict(SQ.openclip_state_dict(SQ.openclip_tiny(V), seed=1), strict=True)
    hf = T.HFCLIPModel(SQ.hf_tiny_pick(V))
    hf.load_state_dict(SQ.hf_state_dict(SQ.hf_tiny_pick(V), seed=2), strict=True)
    ids = torch.randint(1, V - 1, (3, 77), generator=_g(8))
    ids[:, 0], ids[0, 9], ids[1, 76], ids[2, 40] = V - 2, V - 1, V - 1, V - 1
    for model in (oc, hf):
        eng = model.engine(DEV).text
        rows, pooled = eng.encode_text_rows(ids)
        assert torch.equal(pooled, eng.encode_text(ids))
