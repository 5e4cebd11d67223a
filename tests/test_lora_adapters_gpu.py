"""GPU: unmerged LoRA adapters — svi_gemm_lora_bf16 (include/svi_b200_lora.h) bit for bit against svi_gemm_bf16 on the
concatenated operands, its argument checks on the device, and the DiT engine with adapters against the oracle on merged
weights, across adapter switches with CUDA graphs, on an FP8 model, through the SVI pipeline and (>= 2 GPUs) under the
sequence-parallel split."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tools import synth
from test_lora_adapters_cpu import TARGETS, make_lora, merged

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4M3 = torch.float8_e4m3fn

# every entry point of include/svi_b200_lora.h -> the cases here that run it (checked on the CPU)
COVERED = {"svi_gemm_lora_bf16": ["test_lora_segment_is_the_concatenated_gemm", "test_column_groups_equal_the_one_group_call",
                                  "test_e4m3_weight_equals_its_bf16_upcast", "test_zero_u_is_the_plain_gemm",
                                  "test_ragged_k_within_fp64_bound", "test_argument_checks_on_the_device"]}


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _operands(M, N, K, R, groups=1, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).to(torch.bfloat16).cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(torch.bfloat16).cuda()
    u = (torch.randn(M, groups * R, generator=g) * 0.3).to(torch.bfloat16).cuda()
    b = (torch.randn(N, R, generator=g) / R ** 0.5).to(torch.bfloat16).cuda()
    return a, w, u, b


def _epilogue(kind, M, N, seed=1):
    """(out, kwargs) of one epilogue the DiT blocks use."""
    g = torch.Generator().manual_seed(seed)
    bias = (torch.randn(N, generator=g) * 0.1).cuda()
    if kind == "bias":
        return torch.empty(M, N, device="cuda"), dict(bias=bias)
    if kind == "gelu_bf16":
        return torch.empty(M, N, device="cuda", dtype=torch.bfloat16), dict(bias=bias, act=1)
    if kind == "gate_residual":
        x = torch.randn(M, N, generator=g).cuda()
        return x, dict(bias=bias, gate=(torch.rand(N, generator=g) + 0.5).cuda(), residual=x)
    assert kind == "sumsq"
    return (torch.empty(M, N, device="cuda", dtype=torch.bfloat16),
            dict(bias=bias, sumsq=torch.full((M, N // 128, 1), float("nan"), device="cuda"), sumsq_group_cols=128))


def _run_pair(nv, a, w, u, b, R, kind, M, N):
    out1, kw1 = _epilogue(kind, M, N)
    out2, kw2 = _epilogue(kind, M, N)
    if kind == "gate_residual":
        kw2["residual"] = out2
    nv.gemm_lora(a, w, out1, u, b, R, 0, **kw1)
    nv.gemm(torch.cat([a, u], 1), torch.cat([w, b], 1), out2, **kw2)
    torch.cuda.synchronize()
    return out1, kw1, out2, kw2


@pytest.mark.parametrize("kind", ["bias", "gelu_bf16", "gate_residual", "sumsq"])
@pytest.mark.parametrize("M", [37, 1260, 4096])
@pytest.mark.parametrize("R", [64, 128, 192])
def test_lora_segment_is_the_concatenated_gemm(kind, M, R):
    """K % 64 == 0, one group: the LoRA k-blocks follow the main ones in the same order as in the GEMM on [A | U], [W | B];
    N = 1280 at M = 4096 makes 320 tiles (> 2 x 132: every CTA runs both consumer warpgroups, several tiles each)."""
    from diffsynth import _native as nv
    N = 1280 if M == 4096 else 384
    a, w, u, b = _operands(M, N, 512, R, seed=M + R)
    out1, kw1, out2, kw2 = _run_pair(nv, a, w, u, b, R, kind, M, N)
    assert torch.equal(_bits(out1), _bits(out2))
    if kind == "sumsq":
        assert torch.equal(_bits(kw1["sumsq"]), _bits(kw2["sumsq"]))


def test_column_groups_equal_the_one_group_call():
    from diffsynth import _native as nv
    M, d, K, R = 1260, 256, 256, 128
    a, w, u, b = _operands(M, 3 * d, K, R, groups=3, seed=3)
    out = torch.empty(M, 3 * d, device="cuda", dtype=torch.bfloat16)
    ss = torch.empty(M, 3, d // 128, device="cuda")
    bias = torch.randn(3 * d).cuda()
    nv.gemm_lora(a, w, out, u, b, R, d, bias=bias, sumsq=ss, sumsq_group_cols=d)
    for g in range(3):
        o = torch.empty(M, d, device="cuda", dtype=torch.bfloat16)
        s = torch.empty(M, 1, d // 128, device="cuda")
        cols = slice(g * d, (g + 1) * d)
        nv.gemm_lora(a, w[cols], o, u[:, g * R:(g + 1) * R], b[cols], R, 0, bias=bias[cols], sumsq=s, sumsq_group_cols=d)
        assert torch.equal(_bits(out[:, cols]), _bits(o)) and torch.equal(_bits(ss[:, g:g + 1]), _bits(s))
    # the sequence-parallel split: k | v as two groups of the same U, offset by one group
    o2 = torch.empty(M, 2 * d, device="cuda", dtype=torch.bfloat16)
    nv.gemm_lora(a, w[d:], o2, u[:, R:], b[d:], R, d, bias=bias[d:])
    nv.gemm_lora(a, w, out, u, b, R, d, bias=bias)
    assert torch.equal(_bits(o2), _bits(out[:, d:]))


@pytest.mark.parametrize("kind", ["bias", "gelu_bf16", "gate_residual"])
def test_e4m3_weight_equals_its_bf16_upcast(kind):
    from diffsynth import _native as nv
    M, N, K, R = 4096, 1280, 512, 128
    a, w, u, b = _operands(M, N, K, R, seed=5)
    w8 = w.float().to(E4M3)
    o8, kw8 = _epilogue(kind, M, N)
    ob, kwb = _epilogue(kind, M, N)
    if kind == "gate_residual":
        kwb["residual"] = ob
    nv.gemm_lora(a, w8, o8, u, b, R, 0, **kw8)
    nv.gemm_lora(a, w8.to(torch.bfloat16), ob, u, b, R, 0, **kwb)
    torch.cuda.synchronize()
    assert torch.equal(_bits(o8), _bits(ob))


@pytest.mark.parametrize("w_dtype", [torch.bfloat16, E4M3])
def test_zero_u_is_the_plain_gemm(w_dtype):
    from diffsynth import _native as nv
    M, N, K, R = 1260, 768, 512, 64
    a, w, u, b = _operands(M, N, K, R, seed=7)
    w = w.float().to(w_dtype)
    bias = torch.randn(N).cuda()
    o1, o2 = (torch.empty(M, N, device="cuda") for _ in range(2))
    nv.gemm_lora(a, w, o1, torch.zeros_like(u), b, R, 0, bias=bias)
    nv.gemm(a, w, o2, bias=bias)
    assert torch.equal(_bits(o1), _bits(o2))


def test_ragged_k_within_fp64_bound():
    """K % 64 != 0: the main segment's last k-block is zero-filled past K, then the LoRA k-blocks follow.  Bound: fp32
    accumulation over K + R products, |error| <= (K + R) 2^-23 sum |a w| + one f32 rounding."""
    from diffsynth import _native as nv
    M, N, K, R = 1000, 384, 200, 128
    a, w, u, b = _operands(M, N, K, R, seed=11)
    out = torch.empty(M, N, device="cuda")
    nv.gemm_lora(a, w, out, u, b, R, 0)
    A, W = torch.cat([a, u], 1).double().cpu(), torch.cat([w, b], 1).double().cpu()
    ref = A @ W.T
    bound = (K + R) * 2.0 ** -23 * (A.abs() @ W.abs().T) + 2.0 ** -24 * ref.abs()
    err = (out.double().cpu() - ref).abs()
    assert (err <= bound).all(), (err - bound).max().item()


def test_argument_checks_on_the_device():
    from diffsynth import _native as nv
    lib = nv.load()
    M, N, K, R = 256, 384, 128, 64
    a, w, u, b = _operands(M, N, K, 3 * R, seed=13)
    out = torch.empty(M, N, device="cuda")
    stats = torch.zeros(M, 2, device="cuda")
    lnu = torch.zeros(N, device="cuda")

    def call(R=R, group_cols=0, U=u.data_ptr(), ldu=u.stride(0), B=b.data_ptr(), ldb=b.stride(0), act=0, ln=False):
        ep = nv.GemmEpilogue()
        ep.out, ep.ldo, ep.out_is_f32, ep.act = out.data_ptr(), N, 1, act
        if ln:
            ep.ln_stats, ep.ln_u, ep.ln_dim, ep.ln_eps = stats.data_ptr(), lnu.data_ptr(), K, 1e-6
        lo = nv.GemmLoRA(U, ldu, B, ldb, R, group_cols)
        rc = lib.svi_gemm_lora_bf16(a.data_ptr(), K, w.data_ptr(), K, M, N, K, ctypes.byref(ep), ctypes.byref(lo),
                                    nv._stream())
        return rc, lib.svi_last_error().decode()

    assert call()[0] == 0
    cases = [(dict(R=96), "multiple of 64"), (dict(R=0), "multiple of 64"), (dict(group_cols=64), "group_cols"),
             (dict(group_cols=256), "group_cols"), (dict(U=None), "null"), (dict(U=u.data_ptr() + 2), "16-byte aligned"),
             (dict(B=b.data_ptr() + 8), "16-byte aligned"), (dict(group_cols=128, R=128, ldu=192), "ldu"),
             (dict(ldb=32), "ldb"), (dict(ldu=u.stride(0) - 4), "multiples of 8"), (dict(act=2), "activation"),
             (dict(ln=True), "LayerNorm fold")]
    for kw, msg in cases:
        rc, err = call(**kw)
        assert rc != 0 and msg in err and err.startswith("svi_gemm_lora_bf16"), (kw, rc, err)
    torch.cuda.synchronize()
    # the shared checks name the LoRA entry point too
    with pytest.raises(RuntimeError, match="svi_gemm_lora_bf16: .*multiples of 8"):
        nv.gemm_lora(a[:, :124], w[:, :124], out, u, b, R)


# ------------------------------------------------------------------------------------------- the DiT with adapters
def _model(cfg, sd, dtype=torch.bfloat16):
    from diffsynth.models.wan_video_dit import WanModel
    m = WanModel(**cfg).eval()
    m.load_state_dict(sd)
    return m.to(device="cuda", dtype=dtype)


def _stats(out, ref):
    err = (out - ref).abs()
    return (err <= 1e-3 + 1e-2 * ref.abs()).float().mean().item(), err.max().item(), err.mean().item() / ref.std().item()


@pytest.mark.parametrize("cfg,two", [(synth.CFG_TINY_T2V, False), (synth.CFG_TINY_I2V, False), (synth.CFG_TINY_I2V, True)])
def test_forward_with_adapters_matches_oracle_on_merged_weights(cfg, two):
    from oracle import wan_dit_oracle as O
    sd = {k: v.to(torch.bfloat16).float() for k, v in synth.make_dit_state_dict(cfg, seed=4).items()}
    m = _model(cfg, sd)
    inp = synth.make_dit_inputs(cfg, 3, 8, 12, seed=4, ctx_len=40)
    kw = {k: inp[k].cuda() for k in ("clip_feature", "y") if k in inp}
    ts = torch.tensor([937.5])
    eng = m.engine("cuda")
    base = eng.forward(inp["x"].cuda(), ts, inp["context"].cuda(), **kw).cpu()
    loras = [(make_lora(cfg, 40, rank=128), 0.7 if two else 1.0)]
    if two:
        loras.append((make_lora(cfg, 41, rank=16), -0.3))
    for j, (lsd, _) in enumerate(loras):
        m.add_lora_adapter(f"l{j}", lsd)
    m.set_lora_adapters({f"l{j}": al for j, (_, al) in enumerate(loras)})
    out = eng.forward(inp["x"].cuda(), ts, inp["context"].cuda(), **kw).cpu()
    ref = O.dit_forward(merged(sd, loras), cfg, inp["x"], ts, inp["context"], inp.get("clip_feature"), inp.get("y"))
    inside, mx, rel = _stats(out, ref)
    moved = (out - base).abs().mean().item()
    print(f"adapters={len(loras)}: inside={inside:.4f} max={mx:.3e} mean/std={rel:.3e}; mean |with - without| = {moved:.3e}")
    assert inside > 0.93 and mx < 0.012 and rel < 1.6e-3, (inside, mx, rel)
    assert moved >= 10 * (out - ref).abs().mean().item()


def test_switching_adapters_with_graphs_equals_fresh_engines(monkeypatch):
    monkeypatch.setenv("SVI_CUDA_GRAPHS", "1")
    cfg = synth.CFG_TINY_I2V
    sd = synth.make_dit_state_dict(cfg, seed=6)
    la, lb = make_lora(cfg, 60, rank=64), make_lora(cfg, 61, rank=128, targets=TARGETS[:5])
    inp = synth.make_dit_inputs(cfg, 3, 8, 12, seed=6, ctx_len=40)
    args = (inp["x"].cuda(), torch.tensor([700.0]), inp["context"].cuda())
    kw = {k: inp[k].cuda() for k in ("clip_feature", "y")}

    def fresh(active):
        m = _model(cfg, sd)
        m.add_lora_adapter("A", la)
        m.add_lora_adapter("B", lb)
        m.set_lora_adapters(active)
        return m.engine("cuda").forward(*args, **kw).clone()

    m = _model(cfg, sd)
    eng = m.engine("cuda")
    before = eng.forward(*args, **kw).clone()
    m.add_lora_adapter("A", la)
    m.add_lora_adapter("B", lb)
    for active in ({}, {"A": 1.0}, {"B": 0.5}, {}):
        m.set_lora_adapters(active)
        first = eng.forward(*args, **kw).clone()     # eager (the set changed: graphs dropped)
        second = eng.forward(*args, **kw).clone()    # captured and replayed
        assert any(e["graph"] is not None for e in eng._graphs.values())
        want = fresh(active)
        assert torch.equal(_bits(first), _bits(want)) and torch.equal(_bits(second), _bits(want)), active
    assert torch.equal(_bits(second), _bits(before))
    # an alpha change keeps the captured graph, which reads the new gates
    m.set_lora_adapters({"A": 1.0, "B": 0.5})
    eng.forward(*args, **kw)
    eng.forward(*args, **kw)
    graphs = {k: e["graph"] for k, e in eng._graphs.items()}
    m.set_lora_adapters({"A": -0.4, "B": 0.9})
    replay = eng.forward(*args, **kw).clone()
    assert {k: e["graph"] for k, e in eng._graphs.items()} == graphs
    monkeypatch.setenv("SVI_CUDA_GRAPHS", "0")
    assert torch.equal(_bits(replay), _bits(fresh({"A": -0.4, "B": 0.9})))


def test_fp8_model_keeps_the_adapter_that_a_merge_rounds_away():
    from diffsynth.models.lora import GeneralLoRAFromPeft
    from oracle import wan_dit_oracle as O
    cfg = synth.CFG_TINY_T2V
    m8 = _model(cfg, synth.make_dit_state_dict(cfg, seed=8), dtype=E4M3)
    sd8 = {k: v.float().cpu() for k, v in m8.state_dict().items()}            # the e4m3 values, exactly
    twin = _model(cfg, sd8)                                                     # bf16(e4m3(W)) upcast twin
    lsd = make_lora(cfg, 80, rank=128, scale=0.05)
    alpha = 0.8
    for m in (m8, twin):
        m.add_lora_adapter("a", lsd)
        m.set_lora_adapters({"a": alpha})
    inp = synth.make_dit_inputs(cfg, 3, 8, 12, seed=8, ctx_len=40)
    ts = torch.tensor([800.0])
    o8 = m8.engine("cuda").forward(inp["x"].cuda(), ts, inp["context"].cuda()).cpu()
    ob = twin.engine("cuda").forward(inp["x"].cuda(), ts, inp["context"].cuda()).cpu()
    assert torch.equal(_bits(o8), _bits(ob))
    ref = O.dit_forward(merged(sd8, [(lsd, alpha)]), cfg, inp["x"], ts, inp["context"])
    m8.set_lora_adapters({})
    GeneralLoRAFromPeft().load(m8, lsd, alpha=alpha)                           # the reference's merge, onto e4m3
    om = m8.engine("cuda").forward(inp["x"].cuda(), ts, inp["context"].cuda()).cpu()
    e_adapter, e_merge = (o8 - ref).abs().mean().item(), (om - ref).abs().mean().item()
    print(f"e4m3 model, mean |out - oracle(W_e4m3 + alpha B A)|: adapter {e_adapter:.3e}, load_lora_v2 merge {e_merge:.3e}")
    assert e_adapter * 4 < e_merge


def test_pipeline_clip_with_load_lora_adapter_matches_oracle_clip():
    import types
    import test_pipeline_gpu as P
    from tools import synth_vae
    from diffsynth import ModelManager, SVIVideoPipeline
    from diffsynth.models.wan_video_dit import WanModel
    from diffsynth.models.wan_video_vae import WanVideoVAE
    cfg = synth.CFG_TINY_I2V
    dit_sd = {k: v.to(torch.bfloat16).float() for k, v in synth.make_dit_state_dict(cfg, seed=2).items()}
    vae_sd = {k: v.to(torch.bfloat16).float() for k, v in synth_vae.make_vae_state_dict(seed=0).items()}
    lsd = {k.replace("diffusion_model.", "pipe.dit."): v for k, v in make_lora(cfg, 20, rank=64).items()}
    dit = WanModel(**cfg).eval()
    dit.load_state_dict(dit_sd)
    vae = WanVideoVAE().eval()
    vae.load_state_dict(vae_sd)
    mm = ModelManager(torch_dtype=torch.bfloat16, device="cuda")
    mm.add_model("wan_video_dit", dit.to("cuda"))
    mm.add_model("wan_video_vae", vae.to("cuda"))
    pipe = SVIVideoPipeline.from_model_manager(mm, torch_dtype=torch.bfloat16, device="cuda", is_test=True)
    pipe.prompter = P._prompter
    pipe.image_encoder = P._ClipStub()
    with pytest.raises(ValueError, match="load_lora_v2"):
        pipe.load_lora_adapter(state_dict=dict(lsd, **{"pipe.dwpose_embedding.0.weight": torch.zeros(4)}), adapter_name="dance")
    pipe.load_lora_adapter(state_dict=lsd, adapter_name="shot", lora_alpha=0.9)
    img = P._image()
    args = types.SimpleNamespace(ref_pad_cfg=False, ref_pad_num=-1, sequential_cfg="none")
    frames = pipe(prompt="p", negative_prompt="n", input_image=img, num_inference_steps=P.STEPS, cfg_scale={"text": 5.0},
                  seed=42, tiled=False, random_ref_frame=torch.from_numpy(np.array(img)), height=P.H, width=P.W,
                  num_frames=P.FRAMES, args=args, progress_bar_cmd=lambda x: x)
    got = np.stack([np.array(f) for f in frames]).astype(np.float32)
    _, ref = P._oracle_clip(merged(dit_sd, [(lsd, 0.9)]), vae_sd, cfg, img, seed=42)
    diff = np.abs(got - ref.astype(np.float32))
    print(f"clip parity with adapter: mean {diff.mean():.3f} levels, p99 {np.percentile(diff, 99):.1f}, max {diff.max():.0f}")
    assert diff.mean() < 2.0 and np.percentile(diff, 99) < 12
    pipe.set_lora_adapters({})
    pipe.delete_lora_adapter("shot")
    assert pipe.dit._lora_adapters == {}


@pytest.mark.slow
def test_sequence_parallel_forward_with_adapters_equals_one_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29613", os.path.join(ROOT, "tools", "lora_sp_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, cwd=ROOT)
    print(r.stdout[-4000:])
    assert r.returncode == 0 and "LORA_SP_CHECK PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
