"""GPU parity: the native DiT (C-ABI kernels) against the CPU oracle on identical seeded weights / inputs.

Tolerance (BASELINE.json north_star): rtol=1e-2 / atol=1e-3, counted per element.  A 30-block bf16-operand model cannot
satisfy a literal allclose (the reference's own bf16 path reaches 44 % of elements, SURVEY.md §7 hard part 1), so the
stacked-model tests assert the fraction of elements inside the tolerance and the max / mean error.  Where the bars come
from (tools/rounding_study.py, a CPU emulation of every bf16 rounding point of the native path on the oracle):
  * the noise floor is set by the bf16 A operand of the BLOCK GEMMs (97 % inside at cfg-1 with these weights if nothing
    else is rounded); q/k/v/P storage formats cost < 0.2 points; the small GEMMs around the block stack (embedding MLPs,
    patch embedding, head) cost 6 points when fed plain bf16 and are therefore fed two-term bf16 operands;
  * tools.synth draws matrices from N(0, 1/fan_in): a sqrt(3) larger weight std than the reference's constructors
    (nn.Linear default init), on which SURVEY.md measured its 97.5 % bar.  Both initialisations are asserted below.
Single ops / one block are asserted strictly (>= 99.5 % inside) here and in test_kernels_gpu.py.
"""
import pytest
import torch

from tools import synth

pytestmark = pytest.mark.gpu


def _stats(out, ref):
    err = (out - ref).abs()
    inside = (err <= 1e-3 + 1e-2 * ref.abs()).float().mean().item()
    return inside, err.max().item(), err.mean().item() / ref.std().item()


def _sd(cfg, seed):
    """Seeded weights rounded to bf16 (what a real Wan checkpoint holds) and upcast: oracle and native model
    consume IDENTICAL weights, so the comparison isolates the arithmetic."""
    return {k: v.to(torch.bfloat16).float() for k, v in synth.make_dit_state_dict(cfg, seed=seed).items()}


def _build(cfg, sd):
    from diffsynth.models.wan_video_dit import WanModel
    m = WanModel(**cfg).eval()
    m.load_state_dict(sd)
    return m.to("cuda")


@pytest.mark.parametrize("cfg,f,h,w,ctx_len,seed", [(synth.CFG_TINY_T2V, 3, 8, 12, 40, 0), (synth.CFG_TINY_I2V, 2, 6, 10, 24, 1),
                                                     (synth.CFG_TINY_T2V, 5, 18, 30, 512, 2)])
def test_tiny_dit_matches_oracle(cfg, f, h, w, ctx_len, seed):
    from oracle import wan_dit_oracle as O
    sd = _sd(cfg, seed)
    inp = synth.make_dit_inputs(cfg, f, h, w, seed=seed, ctx_len=ctx_len)
    ts = torch.tensor([937.5])
    ref = O.dit_forward(sd, cfg, inp["x"], ts, inp["context"], inp.get("clip_feature"), inp.get("y"))
    m = _build(cfg, sd)
    out = m(inp["x"].cuda(), ts, inp["context"].cuda(),
            clip_feature=None if "clip_feature" not in inp else inp["clip_feature"].cuda(),
            y=None if "y" not in inp else inp["y"].cuda()).float().cpu()
    inside, mx, rel = _stats(out, ref)
    print(f"tiny dit: inside={inside:.4f} max={mx:.4e} mean/std={rel:.4e}")
    # two blocks of bf16-operand GEMMs: on an H100, mean |err| 0.07-0.13 % of the output std and 0.953-0.989 inside over the
    # three cases
    assert inside > 0.93 and mx < 0.012 and rel < 1.6e-3


def test_golden_fixture_tiny_t2v():
    """Same check against the committed reference output itself (not via the oracle)."""
    import os
    import numpy as np
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "dit_tiny_t2v.npz"))
    cfg = synth.CFG_TINY_T2V
    f, h, w = (int(v) for v in g["fhw"])
    sd = synth.make_dit_state_dict(cfg, seed=int(g["seed"]))  # golden used fp32 weights
    inp = synth.make_dit_inputs(cfg, f, h, w, seed=int(g["seed"]), ctx_len=int(g["ctx_len"]))
    m = _build(cfg, sd)
    out = m(inp["x"].cuda(), torch.from_numpy(g["timestep"]), inp["context"].cuda()).float().cpu()
    inside, mx, rel = _stats(out, torch.from_numpy(g["out"]))
    print(f"golden tiny t2v: inside={inside:.4f} max={mx:.4e} mean/std={rel:.4e}")
    # the fixture was generated from fp32 weights, the engine rounds them to bf16 (what a Wan checkpoint holds): the weight
    # rounding, not the arithmetic, sets this bar (on an H100: 0.854 / 1.6e-2 / 2.7e-3; with identical weights: test above)
    assert inside > 0.82 and mx < 0.025 and rel < 3.5e-3


def test_model_fn_and_cfg_euler_step_match_oracle():
    from diffsynth import _native as nv
    from diffsynth.pipelines.svi_video import model_fn_wan_video
    from oracle import wan_dit_oracle as O
    cfg = synth.CFG_TINY_T2V
    sd = _sd(cfg, 3)
    a = synth.make_dit_inputs(cfg, 3, 8, 8, seed=3, ctx_len=32)
    b = synth.make_dit_inputs(cfg, 3, 8, 8, seed=4, ctx_len=32)
    m = _build(cfg, sd)
    ref = O.denoise(sd, cfg, a["x"], a["context"], b["context"], steps=2, cfg_scale=5.0)
    sig = O.flow_match_sigmas(2, 5.0)
    lat = a["x"].cuda().float().clone()
    for i in range(2):
        ts = (sig[i] * 1000).reshape(1)
        vc = model_fn_wan_video(m, lat, ts, a["context"].cuda())
        vu = model_fn_wan_video(m, lat, ts, b["context"].cuda())
        nv.cfg_euler_step(lat, vc, vu, 5.0, float(sig[i]), float(sig[i + 1]) if i + 1 < 2 else 0.0)
    inside, mx, rel = _stats(lat.cpu(), ref)
    print(f"2-step denoise: inside={inside:.4f} max={mx:.4e} mean/std={rel:.4e}")
    # CFG (scale 5) amplifies the per-forward bf16 noise by ~sqrt(5^2 + 4^2) = 6.4x before the Euler update
    # (on an H100: 0.816 / 2.7e-2 / 2.9e-3)
    assert inside > 0.75 and mx < 0.06 and rel < 4e-3


def test_graph_replay_equals_eager_forward():
    """From the second call of a geometry on, the single-GPU forward is a CUDA-graph replay on fixed copies of the inputs:
    it must return exactly what the eager kernel sequence returns, for changing latents, timesteps and prompts."""
    cfg = synth.CFG_TINY_I2V
    sd = _sd(cfg, 8)
    m = _build(cfg, sd)
    eng = m.engine("cuda")
    cases = []
    for k in range(4):
        inp = synth.make_dit_inputs(cfg, 2, 8, 8, seed=20 + k, ctx_len=24)
        cases.append((inp["x"].cuda(), 900.0 - 200.0 * k, inp["context"].cuda(), inp["clip_feature"].cuda(), inp["y"].cuda()))
    eng.use_graphs = False
    want = [eng.forward(x, t, c, cf, y).clone() for x, t, c, cf, y in cases]
    eng.use_graphs = True
    n0 = eng.k.launches
    got = [eng.forward(x, t, c, cf, y).clone() for x, t, c, cf, y in cases]       # call 1 eager, 2 captures, 3-4 replay
    assert len(eng._graphs) == 1 and next(iter(eng._graphs.values()))["graph"] is not None
    for a, b in zip(got, want):      # same kernels, same order; only the fp32 atomics of the row sums may reassociate
        assert (a - b).abs().max().item() < 1e-3
    per_forward = next(iter(eng._graphs.values()))["launches"]
    assert per_forward > 20 and eng.k.launches - n0 >= 4 * per_forward      # replays are counted like eager launches


def test_add_condition_is_added_to_the_patch_embedding():
    """model_fn_wan_video(add_condition=...) — the token-space hook the SVI-Dance pose stem feeds (svi_video.py:102-103)."""
    from diffsynth.pipelines.svi_video import model_fn_wan_video
    from oracle import wan_dit_oracle as O
    cfg = synth.CFG_TINY_T2V
    sd = _sd(cfg, 6)
    a = synth.make_dit_inputs(cfg, 3, 8, 8, seed=6, ctx_len=32)
    m = _build(cfg, sd)
    cond = torch.randn(1, 3 * 4 * 4, cfg["dim"], generator=torch.Generator().manual_seed(9)).to(torch.bfloat16).float()
    ts = torch.tensor([700.0])
    out = model_fn_wan_video(m, a["x"].cuda(), ts, a["context"].cuda(), add_condition=cond.cuda()).float().cpu()
    ref = O.dit_forward(sd, cfg, a["x"], ts, a["context"], add_condition=cond)
    base = O.dit_forward(sd, cfg, a["x"], ts, a["context"])
    inside, mx, rel = _stats(out, ref)
    print(f"add_condition: inside={inside:.4f} max={mx:.4e} mean/std={rel:.4e}")
    assert inside > 0.95 and rel < 1.5e-3 and (ref - base).abs().max() > 1e-2


def test_teacache_denoise_matches_oracle():
    """8-step CFG denoise with TeaCache (reference svi_video.py:23-72,114-126): the native path must take the same
    skip decisions as the oracle and land on the same latents.  Random-init weights make the modulation change by
    ~100 % per step, so the fitted polynomial of the 720P model returns thousands per step; a threshold of 22000
    yields a mixed compute / skip pattern with >= 10 % margin on every decision."""
    from diffsynth import _native as nv
    from diffsynth.pipelines.svi_video import TeaCache, model_fn_wan_video
    from oracle import wan_dit_oracle as O
    cfg = synth.CFG_TINY_T2V
    sd = _sd(cfg, 3)
    a = synth.make_dit_inputs(cfg, 3, 8, 8, seed=3, ctx_len=32)
    b = synth.make_dit_inputs(cfg, 3, 8, 8, seed=4, ctx_len=32)
    m = _build(cfg, sd)
    steps, thresh, mid = 8, 22000.0, "Wan2.1-I2V-14B-720P"
    sig = O.flow_match_sigmas(steps, 5.0)
    o_pos, o_neg = O.TeaCacheOracle(steps, thresh, mid), O.TeaCacheOracle(steps, thresh, mid)
    n_pos, n_neg = TeaCache(steps, rel_l1_thresh=thresh, model_id=mid), TeaCache(steps, rel_l1_thresh=thresh, model_id=mid)
    ref = a["x"].clone()
    lat = a["x"].cuda().float().clone()
    for i in range(steps):
        ts = (sig[i] * 1000).reshape(1)
        vc = O.dit_forward(sd, cfg, ref, ts, a["context"], tea_cache=o_pos)
        vu = O.dit_forward(sd, cfg, ref, ts, b["context"], tea_cache=o_neg)
        ref = O.flow_match_step(sig, i, O.cfg_combine(vc, vu, 5.0), ref)
        vc = model_fn_wan_video(m, lat, ts, a["context"].cuda(), tea_cache=n_pos)
        vu = model_fn_wan_video(m, lat, ts, b["context"].cuda(), tea_cache=n_neg)
        nv.cfg_euler_step(lat, vc, vu, 5.0, float(sig[i]), float(sig[i + 1]) if i + 1 < steps else 0.0)
    assert n_pos.skipped == o_pos.skipped == [1, 2, 4, 6] and n_neg.skipped == o_neg.skipped
    inside, mx, rel = _stats(lat.cpu(), ref)
    print(f"8-step TeaCache denoise: inside={inside:.4f} max={mx:.4e} mean/std={rel:.4e} skipped={n_pos.skipped}")
    assert inside > 0.80 and rel < 3.5e-3          # on an H100: 0.864 / 2.2e-3


@pytest.mark.slow
@pytest.mark.parametrize("init,min_inside,max_err,max_rel", [("normal", 0.95, 0.013, 1.2e-3), ("torch_default", 0.995, 0.003, 3e-4)])
def test_cfg1_1p3b_one_step_matches_oracle(init, min_inside, max_err, max_rel):
    """BASELINE config 1: Wan2.1-T2V-1.3B random-init, 1 denoise step, 17x320x512 (latent [1,16,5,40,64]).
    init="torch_default" is the reference constructors' own initialisation (the survey's 97.5 % / 0.005 bar);
    "normal" is tools.synth's wider N(0, 1/fan_in).  The CPU emulation of bf16 block-GEMM operands alone
    (tools/rounding_study.py `blk`) gives 0.963 / 0.0085 / 1.0e-3 and better than 0.987 / 0.0049 / 7.2e-4.
    """
    from oracle import wan_dit_oracle as O
    cfg = synth.CFG_T2V_1_3B
    sd = {k: v.to(torch.bfloat16).float() for k, v in synth.make_dit_state_dict(cfg, seed=0, init=init).items()}
    inp = synth.make_dit_inputs(cfg, 5, 40, 64, seed=0, ctx_len=512)
    ts = torch.tensor([1000.0])
    torch.set_num_threads(max(1, torch.get_num_threads()))
    v_ref = O.dit_forward(sd, cfg, inp["x"], ts, inp["context"])
    ref = inp["x"] - v_ref                                    # set_timesteps(1): sigma=[1.0] -> x + v*(0-1)
    m = _build(cfg, {k: v.to(torch.bfloat16) for k, v in sd.items()})
    del sd
    v = m(inp["x"].cuda(), ts, inp["context"].cuda()).float()
    out = (inp["x"].cuda() - v).cpu()
    inside, mx, rel = _stats(out, ref)
    print(f"cfg-1 1.3B init={init}: inside={inside:.4f} max={mx:.4e} mean/std={rel:.4e}")
    assert inside > min_inside and mx < max_err and rel < max_rel


@pytest.mark.slow
def test_block_at_bench_shape_matches_oracle():
    """ONE DiT block at the benchmark's shape (BASELINE configs[1]: L = 21*30*52 = 32760 tokens, d = 1536, 12 heads,
    512 context rows) against oracle.dit_block: the ragged last tile (32760 = 255*128 + 120), the sliced last wave of the
    attention launch plan + its merge kernel, and the full-size GEMM tilings are all live.  Per-block bar
    (BASELINE.md section 2): >= 99.6 % of elements inside rtol 1e-2 / atol 1e-3."""
    from oracle import wan_dit_oracle as O
    cfg = dict(synth.CFG_T2V_1_3B, num_layers=1)
    f, h, w = 21, 30, 52
    L, d = f * h * w, cfg["dim"]
    sd = _sd(cfg, 0)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, L, d, generator=g)
    ctx = torch.randn(1, 512, d, generator=g).to(torch.bfloat16).float()      # embedded context rows (a GEMM A operand)
    t_mod = torch.randn(1, 6, d, generator=g) * 0.1
    ref = O.dit_block(sd, 0, x, ctx, t_mod, O.rope_angles_3d(128, f, h, w), cfg)[0]
    m = _build(cfg, sd)
    eng = m.engine("cuda")
    st = eng.project_context(ctx[0].to("cuda", torch.bfloat16))
    mods = (sd["blocks.0.modulation"].reshape(6, d) + t_mod[0]).cuda().contiguous()
    cos, sin = eng.rope(f, h, w)
    xg = x[0].cuda().contiguous()
    eng.run_block(0, xg, mods, st, cos, sin)
    torch.cuda.synchronize()
    inside, mx, rel = _stats(xg.cpu(), ref)
    print(f"block @ L={L}: inside={inside:.5f} max={mx:.4e} mean/std={rel:.4e}")
    assert inside > 0.999 and mx < 0.008 and rel < 4.5e-4          # on an H100: 0.99991 / 2.9e-3 / 2.9e-4


@pytest.mark.slow
def test_14b_width_single_layer_matches_oracle():
    """Wan2.1-I2V-14B geometry (d=5120, 40 heads, ffn 13824, image branch) with ONE layer at a small token count:
    exercises the wide shapes of every kernel (N=15360 QKV, K=13824 FFN, LayerNorm over 5120, 40-head attention,
    257-token image cross-attention with accumulate)."""
    from oracle import wan_dit_oracle as O
    cfg = dict(synth.CFG_I2V_14B, num_layers=1, text_dim=256)
    sd = _sd(cfg, 11)
    inp = synth.make_dit_inputs(cfg, 2, 12, 20, seed=11, ctx_len=77)
    ts = torch.tensor([640.0])
    ref = O.dit_forward(sd, cfg, inp["x"], ts, inp["context"], inp["clip_feature"], inp["y"])
    m = _build(cfg, sd)
    out = m(inp["x"].cuda(), ts, inp["context"].cuda(), clip_feature=inp["clip_feature"].cuda(), y=inp["y"].cuda()).float().cpu()
    inside, mx, rel = _stats(out, ref)
    print(f"14B-width 1 layer: inside={inside:.4f} max={mx:.4e} mean/std={rel:.4e}")
    assert inside > 0.95 and mx < 0.012 and rel < 1.5e-3
