"""CPU: the UniAnimate-DiT pipelines (reference pipelines/wan_video.py:411-1202).

* the context schedule and the oracle against the reference's own results (tests/golden/unianimate_tiny.npz);
* the reference-pose stem's launch plan (kt = 1 slot table, space-to-depth strides) against nn.Conv2d;
* both pipelines on kernel stand-ins (nv_emulation_unianimate) against the oracle, the input checks, stem loading
  through load_lora_v2, and the short pipeline under the 2-rank gloo `use_usp` plan.
"""
import os
import re

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tools import synth, synth_unianimate as SU

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "unianimate_tiny.npz")
HEADER = os.path.join(ROOT, "include", "svi_b200_unianimate.h")


def _bf(t):
    return t.to(torch.bfloat16).float()


# ------------------------------------------------------------------------------------------------ schedule
def test_context_scheduler_matches_golden():
    from diffsynth.pipelines.wan_video import context_scheduler
    from oracle import unianimate_oracle as U
    g = np.load(GOLD)
    keys = [k for k in g.files if k.startswith("sched_")]
    assert len(keys) == 2 * 9 * 3 * 3
    for k in keys:
        stride, n, size, ov = map(int, k.split("_")[1:])
        want = g[k].tolist()
        assert list(context_scheduler(0, 31, n, context_size=size, context_stride=stride, context_overlap=ov)) == want, k
        assert U.context_scheduler(0, n, size, stride, ov) == want, k


def test_context_windows_realign_the_last_window_and_count_every_frame():
    from diffsynth.pipelines.wan_video import context_windows, window_counts
    from oracle import unianimate_oracle as U
    assert context_windows(9, 5, 2) == [list(range(0, 5)), list(range(3, 8)), list(range(4, 9))]
    assert context_windows(41, 21, 4) == [list(range(0, 21)), list(range(17, 38)), list(range(20, 41))]
    assert window_counts(context_windows(41, 21, 4), 41) == [1] * 19 + [2, 2, 1] + [2] * 16 + [1] * 3
    for n, cs, ov in ((9, 5, 2), (41, 21, 4), (21, 21, 4), (30, 8, 3), (60, 21, 2)):
        wins = context_windows(n, cs, ov)
        assert wins == U.windows(n, cs, ov)
        assert all(w == list(range(w[0], w[0] + cs)) for w in wins)
        assert min(window_counts(wins, n)) >= 1


# ------------------------------------------------------------------------------------------------ stems
def test_slot_table_kt1_is_conv2d_per_frame():
    """kt = 1 (a Conv2d): output frame t reads input frame t; kt = 3 keeps the symmetric padding of 1."""
    from diffsynth.models.dwpose_embedding import slot_table
    assert slot_table([0], 1, 1, 1, 1) == [[0]]
    assert slot_table([5, 6, 7], 9, 3, 1, 1) == [[5], [6], [7]]
    assert slot_table([0, 1, 2], 3, 3, 1, 3) == [[3, 0, 1], [0, 1, 2], [1, 2, 3]]


@pytest.mark.parametrize("H,W", [(48, 64), (80, 112)])
def test_ref_stem_engine_matches_conv2d(monkeypatch, H, W):
    """RandomRefEmbeddingEngine on the conv stand-in (the kernel's slot table, padding, space-to-depth packing and SiLU
    staging) against nn.Conv2d in fp32."""
    import nv_emulation_unianimate
    nv_emulation_unianimate.install(monkeypatch)
    from diffsynth.models.dwpose_embedding import RandomRefEmbeddingEngine, make_randomref_embedding_pose
    from oracle import unianimate_oracle as U
    sd = SU.ref_stem_sd(seed=12)
    seq = make_randomref_embedding_pose()
    seq.load_state_dict(sd)
    img = SU.ref_pose(H, W, seed=13)
    got = RandomRefEmbeddingEngine(seq, "cpu").forward(img.permute(2, 0, 1) / 255.0)
    want = U.ref_stem(sd, img)
    assert got.shape == want.shape == (1, 20, 1, H // 8, W // 8)
    rel = (got - want).abs().mean().item() / want.std().item()
    assert rel < 1e-2, rel


def test_oracle_ref_stem_matches_golden():
    from oracle import unianimate_oracle as U
    g = np.load(GOLD)
    out = U.ref_stem(SU.ref_stem_sd(seed=12), SU.ref_pose(80, 112, seed=13))
    np.testing.assert_allclose(out.numpy(), g["stem_out_80x112"], rtol=1e-5, atol=1e-5)
    L = SU.LONG
    out = U.ref_stem(SU.ref_stem_sd(seed=8), SU.ref_pose(L["H"], L["W"], seed=11))
    np.testing.assert_allclose(out.numpy(), g["ref_stem_out"], rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------ long loop
def _long_inputs(cfg, pose_sd, ref_sd, H, W, nf, cs, ov, ctx_len, seed):
    """Conditioning of the long loop as the pipeline builds it: the pose tokens of each window (bf16), y + the
    reference-pose term (bf16), on the CPU oracles."""
    from oracle import dwpose_oracle as DO
    from oracle import unianimate_oracle as U
    h, w = H // 8, W // 8
    pos, neg, clip, y = SU.conditioning(cfg, cs, h, w, ctx_len, seed=seed)
    pose = SU.pose_video(nf, H, W, seed=10)
    ref = SU.ref_pose(H, W, seed=11)
    wins = U.windows((nf - 1) // 4 + 1, cs, ov)
    conds = [_bf(DO.pose_condition(pose_sd, pose[:, 4 * win[0]:4 * win[-1] + 1])) for win in wins]
    r = U.ref_stem(ref_sd, ref).to(torch.bfloat16)
    return dict(pos=pos, neg=neg, clip=clip, y=y, r=r, pose=pose, ref=ref, wins=wins, conds=conds)


def test_oracle_long_loop_matches_golden():
    """The oracle's sliding-window loop equals the reference __call__'s latents (fp32, one-layer 5120-wide DiT)."""
    from oracle import unianimate_oracle as U
    g = np.load(GOLD)
    L, cfg = SU.LONG, SU.CFG_5120
    torch.set_num_threads(os.cpu_count())
    sd = synth.make_dit_state_dict(cfg, seed=3)
    inp = _long_inputs(cfg, SU.pose_stem_sd(cfg["dim"], seed=7), SU.ref_stem_sd(seed=8), L["H"], L["W"], L["num_frames"],
                       L["context_size"], L["context_overlap"], L["ctx_len"], seed=9)
    assert [w[0] for w in inp["wins"]] == [0, 3, 4]
    noise = torch.randn(g["long_noise"].shape, generator=torch.Generator().manual_seed(L["seed"]))
    assert torch.equal(noise, torch.from_numpy(g["long_noise"]))
    carries = list(torch.from_numpy(g["long_carries"]).split(1, dim=0))
    with torch.no_grad():
        got = U.long_loop(sd, cfg, noise, inp["pos"], inp["neg"], inp["clip"], inp["y"] + inp["r"], inp["conds"],
                          inp["wins"], carries, L["steps"], L["cfg_scale"])
    want = torch.from_numpy(g["long_latents"])
    err = (got - want).abs().max().item()
    assert err < 1e-4 * want.abs().max().item(), err


# ------------------------------------------------------------------------------------------------ pipelines on stand-ins
H, W, STEPS, CTX = 32, 48, 2, 24


def _pipe(cls, cfg, pose_sd, ref_sd, device="cpu", **kw):
    from diffsynth import ModelManager
    from diffsynth.models.wan_video_dit import WanModel
    dit = WanModel(**cfg).eval()
    dit.load_state_dict({k: _bf(v) for k, v in synth.make_dit_state_dict(cfg, seed=2).items()})
    mm = ModelManager(torch_dtype=torch.bfloat16, device=device)
    mm.add_model("wan_video_dit", dit)
    mm.state_dict_new_module = {"pipe.dwpose_embedding." + k: v for k, v in pose_sd.items()}
    mm.state_dict_new_module.update({"pipe.randomref_embedding_pose." + k: v for k, v in ref_sd.items()})
    return cls.from_model_manager(mm, torch_dtype=torch.bfloat16, device=device, **kw)


def _stub_encoders(pipe, pos, neg, clip, y):
    """Fixed prompt / image conditioning; decode_video returns the latents it is given (captured)."""
    pipe.image_encoder = object()
    pipe.encode_prompt = lambda prompt, positive=True: {"context": pos if positive else neg}
    pipe.encode_image = lambda image, num_frames, height, width: {"clip_feature": clip,
                                                                  "y": y[:, :, :(num_frames - 1) // 4 + 1].to(torch.bfloat16)}
    captured = {}

    def decode(latents, **kw):
        captured["latents"] = latents.clone()
        return torch.zeros(1, 3, 4 * (latents.shape[2] - 1) + 1, 8 * latents.shape[3], 8 * latents.shape[4])
    pipe.decode_video = decode
    return captured


def _record_randn_like(monkeypatch):
    draws = []
    orig = torch.randn_like

    def rec(t, *a, **k):
        r = orig(t, *a, **k)
        draws.append(r.clone())
        return r
    monkeypatch.setattr(torch, "randn_like", rec)
    return draws


def _rel(got, want):
    return (got - want).abs().mean().item() / want.std().item()


def test_long_pipeline_on_stand_ins_matches_oracle(monkeypatch):
    import nv_emulation_unianimate
    from diffsynth import WanUniAnimateLongVideoPipeline
    from oracle import unianimate_oracle as U
    nv_emulation_unianimate.install(monkeypatch)
    monkeypatch.setenv("SVI_CUDA_GRAPHS", "0")
    cfg = synth.CFG_TINY_I2V
    pose_sd, ref_sd = SU.pose_stem_sd(cfg["dim"], seed=7), SU.ref_stem_sd(seed=8)
    nf, cs, ov = 33, 5, 2
    inp = _long_inputs(cfg, pose_sd, ref_sd, H, W, nf, cs, ov, CTX, seed=9)
    pipe = _pipe(WanUniAnimateLongVideoPipeline, cfg, pose_sd, ref_sd)
    captured = _stub_encoders(pipe, inp["pos"], inp["neg"], inp["clip"], inp["y"])
    draws = _record_randn_like(monkeypatch)
    pipe(prompt="p", negative_prompt="n", input_image=SU.dummy_image(H, W), seed=5, height=H, width=W, num_frames=nf,
         num_inference_steps=STEPS, tiled=False, progress_bar_cmd=lambda x: x, dwpose_data=inp["pose"],
         random_ref_dwpose=inp["ref"], context_size=cs, context_overlap=ov)
    assert len(draws) == 3 and all(d.dtype == torch.bfloat16 and d.shape == (1, 16, 2, H // 8, W // 8) for d in draws)
    noise = _bf(torch.randn(1, 16, 9, H // 8, W // 8, generator=torch.Generator().manual_seed(5)))
    sd = {k: _bf(v) for k, v in synth.make_dit_state_dict(cfg, seed=2).items()}
    y = (inp["y"].to(torch.bfloat16) + inp["r"]).float()
    with torch.no_grad():
        want = U.long_loop(sd, cfg, noise, _bf(inp["pos"]), _bf(inp["neg"]), _bf(inp["clip"]), y, inp["conds"], inp["wins"],
                           [d.float() for d in draws], STEPS)
    rel = _rel(captured["latents"], want)
    assert rel < 1e-2, rel


def test_short_pipeline_on_stand_ins_matches_oracle(monkeypatch):
    import nv_emulation_unianimate
    from diffsynth import WanUniAnimateVideoPipeline
    from oracle import dwpose_oracle as DO
    from oracle import unianimate_oracle as U
    nv_emulation_unianimate.install(monkeypatch)
    monkeypatch.setenv("SVI_CUDA_GRAPHS", "0")
    cfg = synth.CFG_TINY_I2V
    pose_sd, ref_sd = SU.pose_stem_sd(cfg["dim"], seed=7), SU.ref_stem_sd(seed=8)
    nf = 9
    pos, neg, clip, y = SU.conditioning(cfg, 3, H // 8, W // 8, CTX, seed=9)
    pose, ref = SU.pose_video(nf, H, W, seed=10), SU.ref_pose(H, W, seed=11)
    pipe = _pipe(WanUniAnimateVideoPipeline, cfg, pose_sd, ref_sd)
    captured = _stub_encoders(pipe, pos, neg, clip, y)
    pipe(prompt="p", negative_prompt="n", input_image=SU.dummy_image(H, W), seed=5, height=H, width=W, num_frames=nf,
         num_inference_steps=STEPS, tiled=False, progress_bar_cmd=lambda x: x, dwpose_data=pose, random_ref_dwpose=ref)
    noise = _bf(torch.randn(1, 16, 3, H // 8, W // 8, generator=torch.Generator().manual_seed(5)))
    sd = {k: _bf(v) for k, v in synth.make_dit_state_dict(cfg, seed=2).items()}
    yr = (y.to(torch.bfloat16) + U.ref_stem(ref_sd, ref).to(torch.bfloat16)).float()
    with torch.no_grad():
        want = U.short_loop(sd, cfg, noise, _bf(pos), _bf(neg), _bf(clip), yr, _bf(DO.pose_condition(pose_sd, pose)), STEPS)
    rel = _rel(captured["latents"], want)
    assert rel < 1e-2, rel


# ------------------------------------------------------------------------------------------------ input checks
@pytest.mark.parametrize("case,match", [
    ("no_image", "input_image"), ("no_pose", "dwpose_data"), ("no_ref", "random_ref_dwpose"),
    ("pose_frames", "num_frames"), ("short_video", "fewer latent frames|fewer than context_size"),
    ("overlap_1", "at least 2"), ("overlap_size", "smaller than context_size")])
def test_long_pipeline_input_checks(case, match):
    from diffsynth import WanUniAnimateLongVideoPipeline
    pipe = WanUniAnimateLongVideoPipeline(device="cpu", torch_dtype=torch.bfloat16)
    pipe.image_encoder = object()
    pipe.load_pose_stems({"dwpose_embedding." + k: v for k, v in SU.pose_stem_sd(256, 1).items()} |
                         {"randomref_embedding_pose." + k: v for k, v in SU.ref_stem_sd(2).items()})
    kw = dict(input_image=SU.dummy_image(H, W), dwpose_data=SU.pose_video(33, H, W, 1), random_ref_dwpose=SU.ref_pose(H, W, 2),
              num_frames=33, context_size=5, context_overlap=2)
    if case == "no_image":
        kw["input_image"] = None
    elif case == "no_pose":
        kw["dwpose_data"] = None
    elif case == "no_ref":
        kw["random_ref_dwpose"] = None
    elif case == "pose_frames":
        kw["dwpose_data"] = SU.pose_video(29, H, W, 1)
    elif case == "short_video":
        kw.update(num_frames=13, dwpose_data=SU.pose_video(13, H, W, 1))
    elif case == "overlap_1":
        kw["context_overlap"] = 1
    elif case == "overlap_size":
        kw["context_overlap"] = 5
    with pytest.raises(ValueError, match=match):
        pipe(prompt="p", height=H, width=W, num_inference_steps=1, progress_bar_cmd=None, **kw)


def test_short_pipeline_input_checks_and_missing_stems():
    from diffsynth import WanUniAnimateVideoPipeline
    pipe = WanUniAnimateVideoPipeline(device="cpu", torch_dtype=torch.bfloat16)
    pipe.image_encoder = object()
    img, pose, ref = SU.dummy_image(H, W), SU.pose_video(9, H, W, 1), SU.ref_pose(H, W, 2)
    call = lambda **kw: pipe(prompt="p", height=H, width=W, num_frames=9, num_inference_steps=1, progress_bar_cmd=None,
                             **({"input_image": img, "dwpose_data": pose, "random_ref_dwpose": ref} | kw))
    with pytest.raises(ValueError, match="input_image"):
        call(input_image=None)
    with pytest.raises(ValueError, match="dwpose_data"):
        call(dwpose_data=pose[:, :5])
    with pytest.raises(ValueError, match="random_ref_dwpose"):
        call(random_ref_dwpose=ref[:16])
    pipe.encode_prompt = lambda prompt, positive=True: {"context": torch.zeros(1, 4, 96)}
    pipe.encode_image = lambda *a: {"clip_feature": None, "y": torch.zeros(1, 20, 3, H // 8, W // 8)}
    with pytest.raises(RuntimeError, match="dwpose_embedding"):
        call()
    pipe.load_pose_stems({"dwpose_embedding." + k: v for k, v in SU.pose_stem_sd(256, 1).items()})
    with pytest.raises(RuntimeError, match="randomref_embedding_pose"):
        pipe.encode_ref_pose(ref)


def test_load_lora_v2_keeps_both_stems_and_fetch_models_builds_them():
    from diffsynth import ModelManager, WanUniAnimateLongVideoPipeline, WanUniAnimateVideoPipeline
    from diffsynth.models.wan_video_dit import WanModel
    cfg = synth.CFG_TINY_I2V
    mm = ModelManager(torch_dtype=torch.bfloat16, device="cpu")
    mm.add_model("wan_video_dit", WanModel(**cfg).eval())
    d = cfg["dim"]
    sd = {"pipe.dit.blocks.0.self_attn.q.lora_A.default.weight": torch.zeros(4, d),
          "pipe.dit.blocks.0.self_attn.q.lora_B.default.weight": torch.zeros(d, 4)}
    sd.update({"pipe.dwpose_embedding." + k: v for k, v in SU.pose_stem_sd(d, 3).items()})
    sd.update({"pipe.randomref_embedding_pose." + k: v for k, v in SU.ref_stem_sd(4).items()})
    if torch.cuda.is_available():
        mm.load_lora_v2("unianimate.ckpt", state_dict=sd)
    else:       # the LoRA merge needs the native GEMM; the stem keys are kept before it runs
        with pytest.raises(RuntimeError, match="CUDA"):
            mm.load_lora_v2("unianimate.ckpt", state_dict=sd)
    assert set(mm.state_dict_new_module) == {k for k in sd if "lora" not in k}
    for cls in (WanUniAnimateVideoPipeline, WanUniAnimateLongVideoPipeline):
        pipe = cls.from_model_manager(mm, device="cpu")
        assert pipe.dwpose_embedding[12].out_channels == d
        assert torch.equal(pipe.randomref_embedding_pose[10].weight, sd["pipe.randomref_embedding_pose.10.weight"])
        assert torch.equal(pipe.dwpose_embedding[0].bias, sd["pipe.dwpose_embedding.0.bias"])


def test_exports_and_header():
    import diffsynth
    from diffsynth import _native as nv
    from diffsynth import pipelines
    assert diffsynth.WanUniAnimateVideoPipeline is pipelines.WanUniAnimateVideoPipeline
    assert diffsynth.WanUniAnimateLongVideoPipeline is pipelines.WanUniAnimateLongVideoPipeline
    names = set(re.findall(r"^int (svi_\w+)\(", open(HEADER).read(), re.M))
    assert names == {"svi_window_accumulate", "svi_window_normalize"} == set(nv.UNIANIMATE_SIGNATURES)
    others = (nv.SIGNATURES | nv.LORA_SIGNATURES | nv.RIFE_SIGNATURES | nv.ESRGAN_SIGNATURES | nv.FASTBLEND_SIGNATURES)
    assert not names & set(others)


# ------------------------------------------------------------------------------------------------ use_usp
def _usp_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), SVI_CUDA_GRAPHS="0")
    import sys
    for p in (ROOT, os.path.join(ROOT, "stable-video-infinity_b200"), os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    import nv_emulation_unianimate
    nv_emulation_unianimate.install()
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        res = {}
        outs = []
        for use_usp in (False, True):
            pipe = _short_pipe_with_vae(use_usp)
            frames = _short_call(pipe)
            outs.append(np.stack([np.array(f) for f in frames]).astype(np.int32))
            if use_usp:
                res["plan"] = pipe.sp_group().describe()
        res["max_diff"] = int(np.abs(outs[1] - outs[0]).max())
        q.put((rank, res))
    except Exception as ex:  # noqa: BLE001
        import traceback
        q.put((rank, {"error": traceback.format_exc()[-2500:] + repr(ex)}))
    finally:
        dist.destroy_process_group()


def _short_pipe_with_vae(use_usp):
    import test_pipeline_gpu as P
    from diffsynth.models.wan_video_vae import WanVideoVAE
    from diffsynth import WanUniAnimateVideoPipeline
    from tools import synth_vae
    cfg = synth.CFG_TINY_I2V
    pipe = _pipe(WanUniAnimateVideoPipeline, cfg, SU.pose_stem_sd(cfg["dim"], seed=7), SU.ref_stem_sd(seed=8))
    vae = WanVideoVAE().eval()
    vae.load_state_dict({k: _bf(v) for k, v in synth_vae.make_vae_state_dict(seed=0).items()})
    pipe.vae = vae
    if use_usp:
        pipe.enable_usp()
    pipe.prompter = P._prompter
    pipe.image_encoder = P._ClipStub()
    return pipe


def _short_call(pipe):
    from PIL import Image
    img = Image.fromarray(np.random.default_rng(5).integers(0, 255, size=(H, W, 3), dtype=np.uint8))
    return pipe(prompt="p", negative_prompt="n", input_image=img, seed=7, height=H, width=W, num_frames=5,
                num_inference_steps=STEPS, tiled=False, progress_bar_cmd=lambda x: x,
                dwpose_data=SU.pose_video(5, H, W, seed=10), random_ref_dwpose=SU.ref_pose(H, W, seed=11))


def test_short_pipeline_with_use_usp():
    """use_usp=True installs the shared multi-GPU plan (CFG branches on two ranks, row-band VAE); on 2 gloo ranks every
    rank returns the single-process frames."""
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29600 + (os.getpid() % 150)
    procs = [ctx.Process(target=_usp_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = [q.get(timeout=900) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, res in got:
        assert "error" not in res, res["error"]
        assert res["plan"].startswith("cfg2"), res
        assert res["max_diff"] <= 1, res
