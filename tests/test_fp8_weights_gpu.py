"""GPU: e4m3 (float8_e4m3fn) weights read straight by svi_gemm_bf16 — the reference's weight-only FP8 mode.

The kernel converts the e4m3 W tile exactly to bf16 in shared memory ahead of the unchanged bf16 wgmma and epilogue, so every
result must be bit-identical to the bf16 GEMM on W.to(bf16).  Covered: the conversion of all 256 codes, the GEMM over the
DiT / umT5 shapes and every epilogue, the DiT and umT5 engines on an e4m3 model against its bf16(e4m3(p)) twin, a LoRA merged
onto e4m3 weights, and the device memory of a 14B-I2V-shaped engine."""
import pytest
import torch

from tools import synth
from tools import synth_enc as SE

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn
NAN_CODES = (0x7F, 0xFF)


def _bits(t):
    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _rand_w8(N, K, seed, pad=0):
    """e4m3 W [N, K] (a column slice of [N, K + pad] whose pad columns hold NaN codes), every finite code possible."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    codes = torch.randint(0, 256, (N, K + pad), generator=g, device="cuda", dtype=torch.int32)
    codes = torch.where((codes & 0x7F) == 0x7F, codes ^ 0x01, codes)          # finite codes only in the data
    if pad:
        codes[:, K:] = 0x7F
    return codes.to(torch.uint8).view(E4M3)[:, :K]


def _rand_a(M, K, seed, pad=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K + pad, generator=g, device="cuda").to(torch.bfloat16)
    if pad:
        a[:, K:] = float("nan")
    return a[:, :K]


def test_exhaustive_conversion_of_all_256_codes():
    from diffsynth import _native as nv
    table = torch.arange(256, dtype=torch.uint8).view(E4M3).float().cuda()
    K = N = 256
    n = torch.arange(N, device="cuda").view(N, 1)
    k = torch.arange(K, device="cuda").view(1, K)
    codes = (n + k) % 256                                                     # every code at every tile position
    finite = torch.where((codes & 0x7F) == 0x7F, torch.zeros_like(codes), codes)   # NaN codes would poison every row
    w8 = finite.to(torch.uint8).view(E4M3)
    a = torch.eye(256, device="cuda", dtype=torch.bfloat16)                   # one-hot rows: out[m, n] = W[n, m]
    out = torch.full((256, N), float("nan"), device="cuda")
    nv.gemm(a, w8, out)
    want = table[finite.t()]
    assert torch.equal(out, want)                       # == also accepts -0 for +0: a sum of products cannot keep -0
    assert torch.equal(_bits(out[want != 0]), _bits(want[want != 0]))
    # the smallest subnormal and the largest normal, explicitly
    assert table[0x01].item() == 2.0 ** -9 and table[0x7E].item() == 448.0
    # NaN codes: columns 0 / 1 of W hold 0x7F / 0xFF, the rest 0
    wn = torch.zeros(N, K, device="cuda", dtype=torch.uint8)
    wn[0], wn[1] = NAN_CODES
    out.fill_(0.0)
    nv.gemm(a, wn.view(E4M3), out)
    assert torch.isnan(out[:, :2]).all() and torch.equal(out[:, 2:], torch.zeros_like(out[:, 2:]))


SHAPES = [  # (N, K)
    (3 * 1536, 1536), (1536, 1536), (8960, 1536), (1536, 8960), (64, 1536),           # 1.3B q|k|v, o, ffn, head
    (3 * 5120, 5120), (5120, 5120), (13824, 5120), (5120, 13824), (64, 5120),         # 14B
    (3 * 4096, 4096), (4096, 10240), (10240, 4096),                                   # umT5-XXL q|k|v, ffn
    (1536, 64), (5120, 144),                                                          # patch embedding
    (1536, 208), (256, 80),                                                           # K % 64 != 0
]


@pytest.mark.parametrize("M", [1, 7, 128, 3050, 32760])
def test_e4m3_gemm_is_bit_identical_to_bf16_gemm(M):
    from diffsynth import _native as nv
    for i, (N, K) in enumerate(SHAPES):
        if M == 32760 and N * K > 80e6:
            continue                       # the largest products at M = 32760 are covered by the 14B q|k|v / ffn shapes
        pad = 32 if i % 3 == 0 else 0      # ldw > K with NaN pad columns (and NaN pad columns of A)
        w8 = _rand_w8(N, K, seed=i, pad=pad)
        wb = torch.full((N, K + pad), float("nan"), device="cuda", dtype=torch.bfloat16)
        wb[:, :K] = w8.to(torch.bfloat16)
        wb = wb[:, :K]
        a = _rand_a(M, K, seed=100 + i, pad=pad)
        wide = 64 if i % 2 else 0          # column-slice output
        outs = {}
        for name, w in (("e4m3", w8), ("bf16", wb)):
            buf = torch.full((M, N + wide), float("nan"), device="cuda")
            nv.gemm(a, w, buf[:, wide:] if wide else buf)
            outs[name] = buf
        assert torch.equal(_bits(outs["e4m3"]), _bits(outs["bf16"])), (M, N, K)
        del outs, a, w8, wb


@pytest.mark.parametrize("M", [7, 3050])
def test_every_epilogue_is_bit_identical_with_e4m3_weights(M):
    from diffsynth import _native as nv
    N, K = 1536, 1536 + 64
    g = torch.Generator(device="cuda").manual_seed(7)
    w8 = _rand_w8(N, K, seed=7, pad=16)
    wb = w8.to(torch.bfloat16)
    a = _rand_a(M, K, seed=8)
    bias = torch.randn(N, generator=g, device="cuda")
    gate = torch.randn(N, generator=g, device="cuda")
    res0 = torch.randn(M, N, generator=g, device="cuda")
    stats = torch.stack([torch.randn(M, generator=g, device="cuda") * 10, torch.rand(M, generator=g, device="cuda") * 100 + 200], 1)
    u = torch.randn(N, generator=g, device="cuda")
    g_next = torch.randn(N, generator=g, device="cuda")

    def run(w, act=0, out_dtype=torch.float32, **kw):
        out = torch.full((M, N), float("nan"), device="cuda", dtype=out_dtype)
        extra = {}
        if kw.get("residual"):
            out.copy_(res0)
            extra["residual"] = out           # in place, the DiT's residual stream
        if kw.get("sumsq") == "atomic":
            extra["sumsq"], extra["sumsq_group_cols"] = torch.zeros(M, 3, device="cuda"), 512
        elif kw.get("sumsq") == "parts":
            extra["sumsq"], extra["sumsq_group_cols"] = torch.full((M, 3, 4), float("nan"), device="cuda"), 512
        if kw.get("ln"):
            extra["ln"] = (stats, u, K, 1e-6)
        if kw.get("emit"):
            extra["emit"] = (torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16), g_next,
                             torch.zeros(M, 2, device="cuda"))
        nv.gemm(a, w, out, bias=bias if kw.get("bias") else None, act=act, gate=gate if kw.get("gate") else None, **extra)
        return out, extra

    cases = [dict(bias=True, act=act) for act in range(5)] + [
        dict(out_dtype=torch.bfloat16, bias=True), dict(bias=True, gate=True, residual=True),
        dict(bias=True, sumsq="atomic"), dict(bias=True, sumsq="parts"), dict(bias=True, ln=True, act=1),
        dict(bias=True, gate=True, residual=True, emit=True)]
    for c in cases:
        c = dict(c)
        act, od = c.pop("act", 0), c.pop("out_dtype", torch.float32)
        o8, x8 = run(w8, act, od, **c)
        ob, xb = run(wb, act, od, **c)
        assert torch.equal(_bits(o8), _bits(ob)), c
        if c.get("sumsq") == "parts":
            assert torch.equal(_bits(x8["sumsq"]), _bits(xb["sumsq"]))
        elif c.get("sumsq") == "atomic":      # the atomicAdd order varies from run to run
            torch.testing.assert_close(x8["sumsq"], xb["sumsq"], rtol=1e-5, atol=0)
        if c.get("emit"):
            assert torch.equal(_bits(x8["emit"][0]), _bits(xb["emit"][0]))
            # (sum v, sum v^2) per row by atomicAdd over the column tiles: reassociation only, bounded by the sums of |terms|
            scale = torch.stack([o8.abs().sum(1), o8.pow(2).sum(1)], 1)
            assert ((x8["emit"][2] - xb["emit"][2]).abs() <= 1e-5 * scale).all()


def test_gemm_rejects_bad_e4m3_arguments_on_the_device():
    from diffsynth import _native as nv
    a = torch.zeros(4, 48, device="cuda", dtype=torch.bfloat16)
    out = torch.zeros(4, 16, device="cuda")
    w = torch.zeros(16, 48 + 8, device="cuda", dtype=torch.uint8).view(E4M3)[:, :48]     # row stride 56: not 16-byte
    with pytest.raises(RuntimeError, match="multiples of 16"):
        nv.gemm(a, w, out)
    with pytest.raises(RuntimeError, match="bf16 or float8_e4m3fn"):
        nv.gemm(a, torch.zeros(16, 48, device="cuda", dtype=torch.float8_e5m2), out)


def test_c_abi_validates_the_weight_format():
    """svi_gemm_bf16 itself (not only the Python binding) refuses a bad w_e4m3 and an e4m3 W whose K or ldw is not a
    multiple of 16, through svi_last_error, and launches nothing."""
    import ctypes
    from diffsynth import _native as nv
    lib = nv.load()
    a = torch.zeros(4, 64, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(16, 64, device="cuda", dtype=torch.uint8)
    out = torch.full((4, 16), 7.0, device="cuda")

    def call(w_e4m3, K, ldw):
        ep = nv.GemmEpilogue()
        ep.out, ep.ldo, ep.out_is_f32, ep.w_e4m3 = out.data_ptr(), 16, 1, w_e4m3
        rc = lib.svi_gemm_bf16(a.data_ptr(), 64, w.data_ptr(), ldw, 4, 16, K, ctypes.byref(ep), None)
        return rc, lib.svi_last_error().decode()

    for w_e4m3, K, ldw, msg in ((2, 64, 64, "w_e4m3 must be 0"), (-1, 64, 64, "w_e4m3 must be 0"),
                                (1, 40, 48, "multiples of 16"), (1, 48, 56, "multiples of 16")):
        rc, err = call(w_e4m3, K, ldw)
        assert rc != 0 and msg in err, (w_e4m3, K, ldw, rc, err)
    torch.cuda.synchronize()
    assert (out == 7.0).all()
    rc, err = call(1, 64, 64)                     # the same call with valid arguments runs
    torch.cuda.synchronize()
    assert rc == 0 and (out == 0.0).all()


def test_negative_zero_code_keeps_its_sign_like_the_bf16_path():
    """Code 0x80 is -0.  A row of W holding only -0, times positive A, sums -0 products only; the e4m3 GEMM must give the
    same bits as the bf16 GEMM on the same -0 values (and +0 codes the same bits as +0)."""
    from diffsynth import _native as nv
    M, N, K = 128, 256, 128
    codes = torch.zeros(N, K, device="cuda", dtype=torch.uint8)
    codes[::2] = 0x80                                                         # even rows -0, odd rows +0
    w8 = codes.view(E4M3)
    assert torch.equal(w8.to(torch.bfloat16).view(torch.int16)[0], torch.full((K,), -32768, device="cuda", dtype=torch.int16))
    a = torch.ones(M, K, device="cuda", dtype=torch.bfloat16)
    outs = []
    for w in (w8, w8.to(torch.bfloat16)):
        out = torch.full((M, N), float("nan"), device="cuda")
        nv.gemm(a, w, out)
        outs.append(out)
    assert torch.equal(_bits(outs[0]), _bits(outs[1])) and (outs[0] == 0).all()
    print(f"-0 rows come out as {'-0' if torch.signbit(outs[1][0, 0]).item() else '+0'} on both paths")


# ------------------------------------------------------------------------------------------------------------ engines
def _dit_pair(cfg, seed):
    from diffsynth.models.wan_video_dit import WanModel
    sd = synth.make_dit_state_dict(cfg, seed=seed)
    m8 = WanModel(**cfg).eval()
    m8.load_state_dict(sd)
    m8 = m8.to(device="cuda", dtype=E4M3)
    twin = WanModel(**cfg).eval()
    twin.load_state_dict({k: v.to(E4M3).to(torch.bfloat16) for k, v in sd.items()})
    return m8, twin.to(device="cuda", dtype=torch.bfloat16)


def _same(out, ref, spread):
    """Bit-identical when the bf16 path itself is (spread == 0); else within its own run-to-run spread (fp32 atomics)."""
    if spread == 0:
        return torch.equal(_bits(out), _bits(ref))
    return (out - ref).abs().max().item() <= 2 * spread + 1e-6


@pytest.mark.parametrize("cfg,f,h,w,fold", [(synth.CFG_TINY_I2V, 2, 8, 8, "0"), (synth.CFG_TINY_T2V, 3, 16, 24, "1"),
                                            (synth.CFG_TINY_TALK, 3, 8, 8, "0"), (synth.CFG_T2V_1_3B, 21, 24, 36, "0")])
def test_dit_forward_on_e4m3_weights_equals_upcast_twin(monkeypatch, cfg, f, h, w, fold):
    monkeypatch.setenv("SVI_LN_FOLD", fold)
    if cfg is synth.CFG_T2V_1_3B:
        cfg = dict(cfg, num_layers=2)      # 1.3B width, L = 21 * 12 * 18 = 4536 tokens
    m8, twin = _dit_pair(cfg, seed=11)
    kw = {}
    if cfg.get("enable_multitalk"):
        from diffsynth.pipelines.svi_video_talk import preprocess_audio
        kw["audio"] = tuple(t.cuda() for t in preprocess_audio(synth.make_audio_embed(4 * (f - 1) + 1, seed=4)))
    cases = []
    for k in range(3):
        inp = synth.make_dit_inputs(cfg, f, h, w, seed=30 + k, ctx_len=24)
        cases.append((inp["x"].cuda(), 900.0 - 250.0 * k, inp["context"].cuda(),
                      inp["clip_feature"].cuda() if "clip_feature" in inp else None, inp["y"].cuda() if "y" in inp else None))

    def outs(m):
        eng = m.engine("cuda")
        return [eng.forward(x, t, c, cf, y, **kw).clone() for x, t, c, cf, y in cases]   # call 1 eager, 2 captures, 3 replays

    ref = outs(twin)
    twin.invalidate_engine()
    spread = max((a - b).abs().max().item() for a, b in zip(ref, outs(twin)))
    got = outs(m8)
    print(f"DiT {cfg['dim']} fold={fold}: twin run-to-run spread {spread:.3e}")
    for a, b in zip(got, ref):
        assert _same(a, b, spread), (a - b).abs().max().item()


def test_teacache_denoise_on_e4m3_weights_equals_upcast_twin():
    from diffsynth import _native as nv
    from diffsynth.pipelines.svi_video import TeaCache, model_fn_wan_video
    from oracle import wan_dit_oracle as O
    cfg = synth.CFG_TINY_T2V
    m8, twin = _dit_pair(cfg, seed=3)
    a = synth.make_dit_inputs(cfg, 3, 8, 8, seed=3, ctx_len=32)
    b = synth.make_dit_inputs(cfg, 3, 8, 8, seed=4, ctx_len=32)

    def denoise(m):
        n_pos = TeaCache(8, rel_l1_thresh=22000.0, model_id="Wan2.1-I2V-14B-720P")
        n_neg = TeaCache(8, rel_l1_thresh=22000.0, model_id="Wan2.1-I2V-14B-720P")
        lat = a["x"].cuda().float().clone()
        sig = O.flow_match_sigmas(8, 5.0)
        for i in range(8):
            ts = (sig[i] * 1000).reshape(1)
            vc = model_fn_wan_video(m, lat, ts, a["context"].cuda(), tea_cache=n_pos)
            vu = model_fn_wan_video(m, lat, ts, b["context"].cuda(), tea_cache=n_neg)
            nv.cfg_euler_step(lat, vc, vu, 5.0, float(sig[i]), float(sig[i + 1]) if i + 1 < 8 else 0.0)
        return lat, n_pos.skipped

    l8, s8 = denoise(m8)
    lb, sb = denoise(twin)
    print(f"TeaCache skipped steps: {sb}")
    assert s8 == sb
    assert torch.equal(_bits(l8), _bits(lb))


def test_text_encoder_on_e4m3_weights_equals_upcast_twin():
    from diffsynth.models.wan_video_text_encoder import WanTextEncoder
    cfg = SE.TEXT_TINY
    sd = SE.make_text_state_dict(cfg, seed=5)
    m8 = WanTextEncoder(**cfg).eval()
    m8.load_state_dict(sd)
    m8.to(device="cuda", dtype=E4M3)
    twin = WanTextEncoder(**cfg).eval()
    twin.load_state_dict({k: v.to(E4M3).to(torch.bfloat16) for k, v in sd.items()})
    twin.to(device="cuda", dtype=torch.bfloat16)
    ids, mask = SE.make_text_inputs(cfg, seq_len=24, valid=17, seed=5)
    # the engines' f32 outputs
    o8 = m8.engine("cuda").forward(ids.cuda(), mask.cuda())
    ob = twin.engine("cuda").forward(ids.cuda(), mask.cuda())
    assert m8.engine("cuda").layers[0]["w_qkv"].dtype == E4M3
    assert torch.equal(_bits(o8), _bits(ob))
    # the module returns bf16 for e4m3 parameters (weight-only FP8 computes in bf16), the same bits as the twin's bf16
    e8, eb = m8(ids.cuda(), mask.cuda()), twin(ids.cuda(), mask.cuda())
    assert e8.dtype == torch.bfloat16 and torch.equal(_bits(e8), _bits(eb))


def test_lora_merge_onto_e4m3_weights():
    from diffsynth.models.lora import GeneralLoRAFromPeft
    from diffsynth.models.wan_video_dit import WanModel
    cfg = synth.CFG_TINY_T2V
    m = WanModel(**cfg).eval()
    m.load_state_dict(synth.make_dit_state_dict(cfg, seed=9))
    m.to(device="cuda", dtype=E4M3)
    g = torch.Generator().manual_seed(9)
    names = ["blocks.0.self_attn.q.weight", "blocks.1.ffn.0.weight", "head.head.weight"]
    params = dict(m.named_parameters())
    lora, before = {}, {}
    for n in names:
        out_f, in_f = params[n].shape
        key = n[: -len(".weight")]
        lora[f"diffusion_model.{key}.lora_B.default.weight"] = torch.randn(out_f, 16, generator=g) * 0.05
        lora[f"diffusion_model.{key}.lora_A.default.weight"] = torch.randn(16, in_f, generator=g) * 0.05
        before[n] = params[n].detach().float().cpu().double()
    eng0 = m.engine("cuda")
    alpha = 0.7
    GeneralLoRAFromPeft().load(m, lora, alpha=alpha)
    assert m.engine("cuda") is not eng0                       # the merge drops the engine: the next forward rebuilds it
    for n in names:
        key = n[: -len(".weight")]
        B = lora[f"diffusion_model.{key}.lora_B.default.weight"].to(torch.bfloat16).double()
        A = lora[f"diffusion_model.{key}.lora_A.default.weight"].to(torch.bfloat16).double()
        want = (before[n] + alpha * B @ A).float().to(E4M3).view(torch.uint8).to(torch.int32)
        got = params[n].detach().cpu().view(torch.uint8).to(torch.int32)
        assert params[n].dtype == E4M3
        same = (got == want).float().mean().item()
        assert same >= 0.999, (n, same)
        # a differing element may only be a rounding tie flipped by fp32 accumulation: one code apart, same sign
        d = (got - want)[got != want]
        assert d.abs().max().item() <= 1 if d.numel() else True


def test_engine_memory_of_a_14b_i2v_model_halves():
    from diffsynth.models.wan_video_dit import WanModel, precompute_freqs_cis_3d
    from test_fp8_weights_cpu import dit_engine_bytes
    cfg = synth.CFG_I2V_14B

    def build(dtype):
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        with torch.device("meta"):
            m = WanModel(**cfg)
        m = m.to(dtype)
        m.to_empty(device="cuda")
        g = torch.Generator(device="cuda").manual_seed(0)
        with torch.no_grad():
            for p in m.parameters():
                p.copy_((torch.randn(p.shape, generator=g, device="cuda") * 0.02).to(dtype))
        m.freqs = precompute_freqs_cis_3d(cfg["dim"] // cfg["num_heads"])
        eng = m.eval().engine("cuda")
        torch.cuda.synchronize()
        res = dit_engine_bytes(eng), torch.cuda.memory_allocated() - base
        del eng, m
        m = None
        torch.cuda.empty_cache()
        return res

    b8, alloc8 = build(E4M3)
    bb, allocb = build(torch.bfloat16)
    print(f"14B-I2V engine weights: e4m3 {b8 / 2**30:.2f} GiB, bf16 {bb / 2**30:.2f} GiB; model + engine allocated: "
          f"e4m3 {alloc8 / 2**30:.2f} GiB, bf16 {allocb / 2**30:.2f} GiB")
    assert b8 <= 0.52 * bb and alloc8 <= 0.52 * allocb


# ------------------------------------------------------------------------------------------------------------ pipeline
class _Tokenizer:
    """Fixed-length stand-in for the umT5 tokenizer directory (not available offline): one id per character."""

    def __init__(self, vocab, seq_len):
        self.vocab, self.seq_len = vocab, seq_len

    def __call__(self, prompt, return_mask=False, **kw):
        codes = [ord(c) % (self.vocab - 1) + 1 for c in prompt][: self.seq_len]
        ids = torch.zeros(1, self.seq_len, dtype=torch.int64)
        ids[0, : len(codes)] = torch.tensor(codes)
        mask = (ids > 0).to(torch.int64)
        return (ids, mask) if return_mask else ids


class _ClipStub:
    """CLIP ViT-H is loaded outside the ModelManager in the reference harness: a fixed projection of the pooled image."""

    def __init__(self):
        self.proj = torch.randn(3, 257 * 1280, generator=torch.Generator().manual_seed(99)) * 0.5

    def encode_image(self, images):
        return (images[0].float().cpu().mean(dim=(0, 2, 3)) @ self.proj).reshape(1, 257, 1280)


def test_svi_pipeline_from_e4m3_model_manager_with_lora_equals_upcast_pipeline():
    """The user-facing FP8 mode end to end: DiT, umT5 and VAE registered in a ModelManager(torch_dtype=float8_e4m3fn) and
    cast as its checkpoint loader casts them (model_manager.py:62), a LoRA merged through the manager, then one SVI clip
    through SVIVideoPipeline (compute dtype bf16, as in the reference harness).  Its uint8 frames must equal those of the same
    pipeline built from every parameter of those e4m3 models upcast to bf16."""
    import types
    import numpy as np
    from PIL import Image
    from diffsynth import ModelManager, SVIVideoPipeline
    from diffsynth.models.wan_video_dit import WanModel
    from diffsynth.models.wan_video_text_encoder import WanTextEncoder
    from diffsynth.models.wan_video_vae import WanVideoVAE
    from tools import synth_vae
    H, W, FRAMES, STEPS, CTX = 64, 96, 9, 3, 24
    tcfg = SE.TEXT_TINY
    cfg = dict(synth.CFG_TINY_I2V, text_dim=tcfg["dim"])
    specs = [("wan_video_dit", WanModel, cfg, synth.make_dit_state_dict(cfg, seed=2)),
             ("wan_video_text_encoder", WanTextEncoder, tcfg, SE.make_text_state_dict(tcfg, seed=1)),
             ("wan_video_vae", WanVideoVAE, {}, synth_vae.make_vae_state_dict(seed=0))]

    def manager(dtype, sds):
        mm = ModelManager(torch_dtype=dtype, device="cuda")
        for (name, cls, kw, _), sd in zip(specs, sds):
            m = cls(**kw).eval()
            m.load_state_dict(sd)
            mm.add_model(name, m.to(dtype=mm.torch_dtype, device=mm.device))
        return mm

    mm8 = manager(E4M3, [sd for *_, sd in specs])
    g = torch.Generator().manual_seed(4)
    lora = {}
    for key in ("blocks.0.self_attn.q", "blocks.1.cross_attn.k", "blocks.0.ffn.0", "head.head"):
        out_f, in_f = dict(mm8.fetch_model("wan_video_dit").named_parameters())[key + ".weight"].shape
        lora[f"diffusion_model.{key}.lora_B.default.weight"] = torch.randn(out_f, 8, generator=g) * 0.05
        lora[f"diffusion_model.{key}.lora_A.default.weight"] = torch.randn(8, in_f, generator=g) * 0.05
    mm8.load_lora(state_dict=lora, lora_alpha=0.8)
    assert mm8.fetch_model("wan_video_dit").blocks[0].self_attn.q.weight.dtype == E4M3
    mmb = manager(torch.bfloat16, [{k: v.to(torch.bfloat16) for k, v in mm8.fetch_model(name).state_dict().items()}
                                   for name, *_ in specs])

    img = Image.fromarray(np.random.default_rng(5).integers(0, 255, size=(H, W, 3), dtype=np.uint8))
    args = types.SimpleNamespace(ref_pad_cfg=False, ref_pad_num=-1, sequential_cfg="none")
    clips = []
    for mm in (mm8, mmb):
        pipe = SVIVideoPipeline.from_model_manager(mm, torch_dtype=torch.bfloat16, device="cuda", is_test=True)
        pipe.prompter.tokenizer = _Tokenizer(tcfg["vocab"], CTX)
        pipe.image_encoder = _ClipStub()
        frames = pipe(prompt="a red fox runs across the snow", negative_prompt="blurry, static", input_image=img,
                      num_inference_steps=STEPS, cfg_scale={"text": 5.0}, seed=42, tiled=False,
                      random_ref_frame=torch.from_numpy(np.array(img)), height=H, width=W, num_frames=FRAMES, args=args,
                      progress_bar_cmd=lambda x: x)
        clips.append(np.stack([np.array(f) for f in frames]))
        assert pipe.dit.engine("cuda").blocks[0].w_qkv.dtype == (E4M3 if mm is mm8 else torch.bfloat16)
    assert clips[0].shape == (FRAMES, H, W, 3) and np.array_equal(clips[0], clips[1])
    assert clips[0].std() > 1.0                   # a real clip, not a constant image


def test_sequence_parallel_two_ranks_on_e4m3_weights():
    """The rank-local q and k|v GEMMs of the sequence-parallel plan read row slices of the fused e4m3 q|k|v matrix."""
    import os
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29613", os.path.join(root, "tools", "fp8_sp_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=root)
    print(r.stdout[-4000:])
    assert r.returncode == 0 and "FP8_SP_CHECK PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
