"""CPU: the UniAnimate-DiT Replace-Anyone pipeline (reference pipelines/wan_video.py:1207-1584).

* the oracle against the reference's own results (tests/golden/replace_anyone_tiny.npz): the masked VAE input, both
  stems in bf16 and f32, and the latents at cfg_scale 5 and 1;
* both stems' launch plans on the conv stand-ins against nn.Conv3d, and the repeated-first-frame slot table;
* the pipeline on kernel stand-ins (nv_emulation_replace) against the oracle and the golden latents;
* the input checks, strict stem loading, the missing-stem error, the exports and the header.
"""
import os
import re

import numpy as np
import pytest
import torch

from tools import synth, synth_replace_anyone as SR, synth_unianimate as SU

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "replace_anyone_tiny.npz")
HEADER = os.path.join(ROOT, "include", "svi_b200_replace.h")
RP = SR.REPLACE


def _bf(t):
    return t.to(torch.bfloat16).float()


def _rel(got, want):
    return (got - want).abs().mean().item() / want.std().item()


def _golden_inputs():
    H, W, nf = RP["H"], RP["W"], RP["num_frames"]
    return SR.video(nf, H, W, seed=30), SR.segmentation(nf, H, W, seed=31)


# ------------------------------------------------------------------------------------------------ oracle vs reference
def test_oracle_mask_and_stems_match_golden():
    from oracle import replace_anyone_oracle as R
    g = np.load(GOLD)
    video, seg = _golden_inputs()
    assert torch.equal(torch.from_numpy(g["vae_input"]), R.masked_video(video, seg).unsqueeze(0))
    h, w, f = RP["H"] // 8, RP["W"] // 8, (RP["num_frames"] - 1) // 4 + 1
    li_in = _bf(R.learn_in_input(video, seg))
    ip_in = _bf(SR.masked_latents(f, h, w, seed=22))
    for name, out, ref_bf16, ref_f32 in (
            ("learn_in", R.learn_in(SR.learn_in_sd(seed=20), li_in), g["learn_in_bf16"], g["learn_in_f32"]),
            ("inpaint", R.inpaint(SR.inpaint_sd(seed=21), ip_in), g["inpaint_bf16"], g["inpaint_f32"])):
        np.testing.assert_allclose(out.numpy(), ref_f32, rtol=1e-5, atol=1e-5 * np.abs(ref_f32).max(), err_msg=name)
        # the reference ran the stem in bf16: within bf16 rounding of the f32 result, layer by layer
        assert _rel(out, torch.from_numpy(ref_bf16)) < 2e-2, name
    off = R.offset(SR.learn_in_sd(seed=20), SR.inpaint_sd(seed=21), video, seg, SR.masked_latents(f, h, w, seed=22))
    bf_sum = torch.from_numpy(g["learn_in_bf16"]) + torch.from_numpy(g["inpaint_bf16"])
    assert _rel(off, bf_sum) < 2e-2


def _golden_conditioning():
    from oracle import dwpose_oracle as DO
    from oracle import unianimate_oracle as U
    cfg, H, W, nf = SU.CFG_5120, RP["H"], RP["W"], RP["num_frames"]
    h, w, f = H // 8, W // 8, (nf - 1) // 4 + 1
    pos, neg, clip, y = SU.conditioning(cfg, f, h, w, RP["ctx_len"], seed=9)
    pose, ref = SU.pose_video(nf, H, W, seed=10), SU.ref_pose(H, W, seed=11)
    cond = _bf(DO.pose_condition(SU.pose_stem_sd(cfg["dim"], seed=7), pose))
    r = U.ref_stem(SU.ref_stem_sd(seed=8), ref).to(torch.bfloat16)
    return dict(pos=pos, neg=neg, clip=clip, y=y, r=r, pose=pose, ref=ref, cond=cond)


@pytest.mark.parametrize("cfg_scale", [5.0, 1.0])
def test_oracle_loop_matches_golden(cfg_scale):
    """The oracle's loop, with the conditional branch on latents + offset and the unconditional one on the latents,
    equals the reference __call__'s latents (fp32, one-layer 5120-wide DiT)."""
    from oracle import replace_anyone_oracle as R
    g = np.load(GOLD)
    torch.set_num_threads(os.cpu_count())
    cfg = SU.CFG_5120
    sd = synth.make_dit_state_dict(cfg, seed=3)
    c = _golden_conditioning()
    noise = torch.randn(g["noise"].shape, generator=torch.Generator().manual_seed(RP["seed"]))
    assert torch.equal(noise, torch.from_numpy(g["noise"]))
    off = torch.from_numpy(g["learn_in_bf16"]) + torch.from_numpy(g["inpaint_bf16"])
    with torch.no_grad():
        got = R.replace_loop(sd, cfg, noise, off, c["pos"], c["neg"], c["clip"], c["y"] + c["r"], c["cond"], RP["steps"],
                             cfg_scale)
    want = torch.from_numpy(g["latents_cfg5" if cfg_scale != 1.0 else "latents_cfg1"])
    err = (got - want).abs().max().item()
    assert err < 1e-4 * want.abs().max().item(), err


# ------------------------------------------------------------------------------------------------ stems
def test_slot_table_with_repeated_first_frame_is_the_materialised_cat():
    """frames [0, 0, 0, 0, 1, .., T-1] over a ring of the T video frames reads, tap by tap, the same video frames as the
    plain table over a ring holding the reference's materialised cat([x[:, :1] x3, x]) (None: the zero slot)."""
    from diffsynth.models.dwpose_embedding import slot_table
    for T, ts in ((5, 1), (9, 1), (9, 2), (21, 2)):
        cat = [0, 0, 0] + list(range(T))              # video frame held by each slot of the materialised ring
        n = len(cat)
        T_out = (n - 1) // ts + 1
        repeated = slot_table([0, 0, 0] + list(range(T)), T, T_out, ts, 3)
        plain = slot_table(list(range(n)), n, T_out, ts, 3)
        assert [[None if s == T else s for s in row] for row in repeated] == \
            [[None if s == n else cat[s] for s in row] for row in plain]
    assert slot_table([0, 0, 0, 0, 1], 2, 5, 1, 3)[:2] == [[2, 0, 0], [0, 0, 0]]


@pytest.mark.parametrize("T,H,W", [(5, 48, 80), (9, 32, 64)])
def test_learn_in_engine_matches_conv3d(monkeypatch, T, H, W):
    """LearnInEmbeddingEngine on the stand-ins (mask stage, slot table with the repeated frame, space-to-depth packing,
    SiLU staging) against nn.Conv3d on the materialised input; 48 x 80 is a multiple of 16 but not of 32."""
    import nv_emulation_replace
    nv_emulation_replace.install(monkeypatch)
    from diffsynth.models.dwpose_embedding import LearnInEmbeddingEngine, make_learn_in_embedding
    from oracle import replace_anyone_oracle as R
    seq = make_learn_in_embedding()
    seq.load_state_dict(SR.learn_in_sd(seed=T))
    video, seg = SR.video(T, H, W, seed=1), SR.segmentation(T, H, W, seed=2)
    masked = torch.empty_like(video)
    eng = LearnInEmbeddingEngine(seq, "cpu")
    got = eng.forward(video, seg[0], masked)
    with torch.no_grad():
        want = seq(R.learn_in_input(video, seg))
    assert got.shape == want.shape == (1, 16, (T - 1) // 4 + 1, H // 8, W // 8)
    assert _rel(got, want) < 1e-2
    assert torch.equal(masked, R.masked_video(video, seg))


@pytest.mark.parametrize("f,h,w", [(3, 6, 10), (5, 4, 8)])
def test_inpaint_engine_matches_conv3d(monkeypatch, f, h, w):
    import nv_emulation_replace
    nv_emulation_replace.install(monkeypatch)
    from diffsynth.models.dwpose_embedding import InpaintEmbeddingEngine, make_inpaint_embedding
    seq = make_inpaint_embedding()
    seq.load_state_dict(SR.inpaint_sd(seed=f))
    lat = SR.masked_latents(f, h, w, seed=3)
    got = InpaintEmbeddingEngine(seq, "cpu").forward(lat)
    with torch.no_grad():
        want = seq(lat)
    assert got.shape == want.shape and _rel(got, want) < 1e-2


def test_pose_stem_launches_unchanged(monkeypatch):
    """The pose stem runs on the shared layer loop with the launches it had before: for 8 frames, 16 to stage the input,
    16 SiLU restages, 6 full-resolution conv launches, 8 + 8 + 4 space-to-depth stagings, 2 + 1 + 1 strided conv launches
    and 3 for the projection."""
    import nv_emulation_replace
    nv_emulation_replace.install(monkeypatch)
    from diffsynth.models.dwpose_embedding import DWPoseEmbeddingEngine, make_dwpose_embedding
    from oracle import dwpose_oracle as DO
    seq = make_dwpose_embedding(dim=64)
    sd = SU.pose_stem_sd(64, seed=5)
    seq.load_state_dict(sd)
    T, H, W = 8, 32, 48
    pose = torch.rand(3, T, H, W, generator=torch.Generator().manual_seed(0))
    eng = DWPoseEmbeddingEngine(seq, "cpu")
    got = eng.forward(pose)
    want = DO.stem(sd, pose.unsqueeze(0)).flatten(2).transpose(1, 2)
    assert _rel(got, want) < 1e-2
    assert eng.launches == 65


# ------------------------------------------------------------------------------------------------ pipeline on stand-ins
H, W, CTX = 32, 48, 24


def _replace_pipe(cfg, dit_sd, device="cpu"):
    from diffsynth import ModelManager, WanRepalceAnyoneVideoPipeline
    from diffsynth.models.wan_video_dit import WanModel
    dit = WanModel(**cfg).eval()
    dit.load_state_dict({k: _bf(v) for k, v in dit_sd.items()})
    mm = ModelManager(torch_dtype=torch.bfloat16, device=device)
    mm.add_model("wan_video_dit", dit)
    mm.state_dict_new_module = {"pipe.dwpose_embedding." + k: v for k, v in SU.pose_stem_sd(cfg["dim"], seed=7).items()}
    mm.state_dict_new_module.update({"pipe.randomref_embedding_pose." + k: v for k, v in SU.ref_stem_sd(seed=8).items()})
    mm.state_dict_new_module.update({"pipe.learn_in_embedding." + k: v for k, v in SR.learn_in_sd(seed=20).items()})
    mm.state_dict_new_module.update({"pipe.inpaint_embedding." + k: v for k, v in SR.inpaint_sd(seed=21).items()})
    return WanRepalceAnyoneVideoPipeline.from_model_manager(mm, torch_dtype=torch.bfloat16, device=device)


def _stub(pipe, pos, neg, clip, y, lat_masked):
    """Fixed prompt / image conditioning; encode_video records the masked video and returns `lat_masked` in the pipeline
    dtype; decode_video records the latents."""
    rec = {}
    pipe.image_encoder = object()
    pipe.encode_prompt = lambda prompt, positive=True: {"context": pos if positive else neg}
    pipe.encode_image = lambda image, num_frames, height, width: {"clip_feature": clip, "y": y.to(torch.bfloat16)}

    def encode_video(input_video, **kw):
        rec["vae_input"] = input_video.clone()
        return lat_masked.to(torch.bfloat16)

    def decode(latents, **kw):
        rec["latents"] = latents.clone()
        return torch.zeros(1, 3, 4 * (latents.shape[2] - 1) + 1, 8 * latents.shape[3], 8 * latents.shape[4])
    pipe.encode_video, pipe.decode_video = encode_video, decode
    return rec


@pytest.mark.parametrize("cfg_scale", [5.0, 1.0])
def test_pipeline_on_stand_ins_matches_oracle(monkeypatch, cfg_scale):
    import nv_emulation_replace
    from oracle import dwpose_oracle as DO
    from oracle import replace_anyone_oracle as R
    from oracle import unianimate_oracle as U
    nv_emulation_replace.install(monkeypatch)
    monkeypatch.setenv("SVI_CUDA_GRAPHS", "0")
    cfg = synth.CFG_TINY_I2V
    nf, h, w = 9, H // 8, W // 8
    pipe = _replace_pipe(cfg, synth.make_dit_state_dict(cfg, seed=2))
    pos, neg, clip, y = SU.conditioning(cfg, 3, h, w, CTX, seed=9)
    lat_m = SR.masked_latents(3, h, w, seed=22)
    rec = _stub(pipe, pos, neg, clip, y, lat_m)
    video, seg = SR.video(nf, H, W, seed=30), SR.segmentation(nf, H, W, seed=31)
    pose, ref = SU.pose_video(nf, H, W, seed=10), SU.ref_pose(H, W, seed=11)
    pipe(prompt="p", negative_prompt="n", input_image=SU.dummy_image(H, W), seed=5, height=H, width=W, num_frames=nf,
         cfg_scale=cfg_scale, num_inference_steps=2, tiled=False, progress_bar_cmd=lambda x: x, dwpose_data=pose,
         random_ref_dwpose=ref, batch={"video": video, "segmentation_data": seg})
    assert torch.equal(rec["vae_input"][0], R.masked_video(video, seg))
    noise = _bf(torch.randn(1, 16, 3, h, w, generator=torch.Generator().manual_seed(5)))
    sd = {k: _bf(v) for k, v in synth.make_dit_state_dict(cfg, seed=2).items()}
    yr = (y.to(torch.bfloat16) + U.ref_stem(SU.ref_stem_sd(seed=8), ref).to(torch.bfloat16)).float()
    off = R.offset(SR.learn_in_sd(seed=20), SR.inpaint_sd(seed=21), video, seg, lat_m)
    with torch.no_grad():
        want = R.replace_loop(sd, cfg, noise, off, _bf(pos), _bf(neg), _bf(clip), yr,
                              _bf(DO.pose_condition(SU.pose_stem_sd(cfg["dim"], seed=7), pose)), 2, cfg_scale)
    rel = _rel(rec["latents"], want)
    assert rel < 1e-2, rel


@pytest.mark.parametrize("cfg_scale", [5.0, 1.0])
def test_pipeline_on_stand_ins_matches_golden(monkeypatch, cfg_scale):
    """The fixture's call (one-layer 5120-wide DiT) through the public pipeline on the stand-ins, against the reference's
    latents.  The pipeline holds bf16 weights and rounds the initial noise to bf16, as every pipeline here does."""
    import nv_emulation_replace
    nv_emulation_replace.install(monkeypatch)
    monkeypatch.setenv("SVI_CUDA_GRAPHS", "0")
    torch.set_num_threads(os.cpu_count())
    g = np.load(GOLD)
    cfg, nf = SU.CFG_5120, RP["num_frames"]
    h, w, f = RP["H"] // 8, RP["W"] // 8, (nf - 1) // 4 + 1
    pipe = _replace_pipe(cfg, synth.make_dit_state_dict(cfg, seed=3))
    c = _golden_conditioning()
    rec = _stub(pipe, c["pos"], c["neg"], c["clip"], c["y"], SR.masked_latents(f, h, w, seed=22))
    video, seg = _golden_inputs()
    pipe(prompt="p", negative_prompt="n", input_image=SU.dummy_image(RP["H"], RP["W"]), seed=RP["seed"], height=RP["H"],
         width=RP["W"], num_frames=nf, cfg_scale=cfg_scale, num_inference_steps=RP["steps"], tiled=False,
         progress_bar_cmd=lambda x: x, dwpose_data=c["pose"], random_ref_dwpose=c["ref"],
         batch={"video": video, "segmentation_data": seg})
    assert torch.equal(rec["vae_input"], torch.from_numpy(g["vae_input"]))
    want = torch.from_numpy(g["latents_cfg5" if cfg_scale != 1.0 else "latents_cfg1"])
    rel = _rel(rec["latents"], want)
    assert rel < 2e-2, rel


# ------------------------------------------------------------------------------------------------ input checks
def _checked_pipe():
    from diffsynth import WanRepalceAnyoneVideoPipeline
    pipe = WanRepalceAnyoneVideoPipeline(device="cpu", torch_dtype=torch.bfloat16)
    pipe.image_encoder = object()
    return pipe


def _kw(nf=9, **over):
    kw = dict(input_image=SU.dummy_image(H, W), dwpose_data=SU.pose_video(nf, H, W, 1), random_ref_dwpose=SU.ref_pose(H, W, 2),
              num_frames=nf, batch={"video": SR.video(nf, H, W, 3), "segmentation_data": SR.segmentation(nf, H, W, 4)})
    kw.update(over)
    return kw


@pytest.mark.parametrize("case,match", [
    ("no_batch", "batch="), ("no_video", "batch="), ("no_seg", "batch="),
    ("video_frames", r'batch\["video"\]'), ("video_channels", r'batch\["video"\]'),
    ("video_unrounded", r'batch\["video"\]'), ("seg_3d", "segmentation_data"), ("seg_size", "segmentation_data"),
    ("no_image", "input_image"), ("no_pose", "dwpose_data"), ("pose_frames", "dwpose_data"),
    ("no_ref", "random_ref_dwpose")])
def test_input_checks(case, match):
    pipe = _checked_pipe()
    kw = _kw()
    b = kw["batch"]
    if case == "no_batch":
        kw["batch"] = None
    elif case == "no_video":
        kw["batch"] = {"segmentation_data": b["segmentation_data"]}
    elif case == "no_seg":
        kw["batch"] = {"video": b["video"]}
    elif case == "video_frames":
        b["video"] = b["video"][:, :5]
    elif case == "video_channels":
        b["video"] = torch.cat([b["video"], b["video"][:1]])
    elif case == "video_unrounded":          # 7 frames round up to 9: the video must have 9
        kw = _kw(nf=7, dwpose_data=SU.pose_video(9, H, W, 1))
        kw["batch"]["segmentation_data"] = SR.segmentation(9, H, W, 4)
    elif case == "seg_3d":
        b["segmentation_data"] = b["segmentation_data"][0]
    elif case == "seg_size":
        b["segmentation_data"] = b["segmentation_data"][..., :16]
    elif case == "no_image":
        kw["input_image"] = None
    elif case == "no_pose":
        kw["dwpose_data"] = None
    elif case == "pose_frames":
        kw["dwpose_data"] = SU.pose_video(5, H, W, 1)
    elif case == "no_ref":
        kw["random_ref_dwpose"] = None
    with pytest.raises(ValueError, match=match):
        pipe(prompt="p", height=H, width=W, num_inference_steps=1, progress_bar_cmd=None, **kw)


def test_missing_stems_raise_and_loading_is_strict():
    pipe = _checked_pipe()
    pipe.encode_prompt = lambda prompt, positive=True: {"context": torch.zeros(1, 4, 96)}
    pipe.encode_image = lambda *a: {"clip_feature": None, "y": torch.zeros(1, 20, 3, H // 8, W // 8)}
    pipe.load_pose_stems({"dwpose_embedding." + k: v for k, v in SU.pose_stem_sd(256, 1).items()} |
                         {"randomref_embedding_pose." + k: v for k, v in SU.ref_stem_sd(2).items()})
    pipe.encode_pose = lambda d: torch.zeros(1, 8, 256)
    pipe.encode_ref_pose = lambda r: torch.zeros(1, 20, 1, H // 8, W // 8)
    call = lambda: pipe(prompt="p", height=H, width=W, num_inference_steps=1, progress_bar_cmd=None, **_kw())
    with pytest.raises(RuntimeError, match="learn_in_embedding"):
        call()
    pipe.load_replace_stems({"learn_in_embedding." + k: v for k, v in SR.learn_in_sd(3).items()})
    assert pipe.inpaint_embedding is None
    with pytest.raises(RuntimeError, match="inpaint_embedding"):
        call()
    li = {"learn_in_embedding." + k: v for k, v in SR.learn_in_sd(3).items()}
    with pytest.raises(RuntimeError, match="Missing key"):
        pipe.load_replace_stems({k: v for k, v in li.items() if not k.endswith("6.bias")})
    with pytest.raises(RuntimeError, match="Unexpected key"):
        pipe.load_replace_stems(li | {"learn_in_embedding.8.weight": torch.zeros(1)})
    ip = {"inpaint_embedding." + k: v for k, v in SR.inpaint_sd(4).items()}
    with pytest.raises(RuntimeError, match="Unexpected key"):
        pipe.load_replace_stems(ip | {"inpaint_embedding.6.bias": torch.zeros(16)})


def test_load_lora_v2_keeps_the_stems_and_fetch_models_builds_them():
    from diffsynth import ModelManager, WanReplaceAnyoneVideoPipeline
    from diffsynth.models.wan_video_dit import WanModel
    cfg = synth.CFG_TINY_I2V
    mm = ModelManager(torch_dtype=torch.bfloat16, device="cpu")
    mm.add_model("wan_video_dit", WanModel(**cfg).eval())
    d = cfg["dim"]
    sd = {"pipe.dit.blocks.0.self_attn.q.lora_A.default.weight": torch.zeros(4, d),
          "pipe.dit.blocks.0.self_attn.q.lora_B.default.weight": torch.zeros(d, 4)}
    sd.update({"pipe.dwpose_embedding." + k: v for k, v in SU.pose_stem_sd(d, 3).items()})
    sd.update({"pipe.randomref_embedding_pose." + k: v for k, v in SU.ref_stem_sd(4).items()})
    sd.update({"pipe.learn_in_embedding." + k: v for k, v in SR.learn_in_sd(5).items()})
    sd.update({"pipe.inpaint_embedding." + k: v for k, v in SR.inpaint_sd(6).items()})
    if torch.cuda.is_available():
        mm.load_lora_v2("replace_anyone.ckpt", state_dict=sd)
    else:       # the LoRA merge needs the native GEMM; the extra-module keys are kept before it runs
        with pytest.raises(RuntimeError, match="CUDA"):
            mm.load_lora_v2("replace_anyone.ckpt", state_dict=sd)
    assert set(mm.state_dict_new_module) == {k for k in sd if "lora" not in k}
    pipe = WanReplaceAnyoneVideoPipeline.from_model_manager(mm, device="cpu")
    assert torch.equal(pipe.learn_in_embedding[6].weight, sd["pipe.learn_in_embedding.6.weight"])
    assert torch.equal(pipe.inpaint_embedding[4].bias, sd["pipe.inpaint_embedding.4.bias"])
    assert pipe.dwpose_embedding[12].out_channels == d


def test_exports_and_header():
    import diffsynth
    from diffsynth import _native as nv
    from diffsynth import pipelines
    assert diffsynth.WanRepalceAnyoneVideoPipeline is pipelines.WanRepalceAnyoneVideoPipeline
    assert diffsynth.WanReplaceAnyoneVideoPipeline is diffsynth.WanRepalceAnyoneVideoPipeline
    assert issubclass(diffsynth.WanRepalceAnyoneVideoPipeline, diffsynth.WanUniAnimateVideoPipeline)
    text = open(HEADER).read()
    names = set(re.findall(r"^int (svi_\w+)\(", text, re.M))
    assert names == {"svi_replace_mask_stage"} == set(nv.REPLACE_SIGNATURES)
    others = (nv.SIGNATURES | nv.LORA_SIGNATURES | nv.RIFE_SIGNATURES | nv.ESRGAN_SIGNATURES | nv.FASTBLEND_SIGNATURES |
              nv.UNIANIMATE_SIGNATURES)
    assert not names & set(others)
    args = re.search(r"int svi_replace_mask_stage\(([^)]*)\)", text).group(1).split(",")
    assert len(args) == len(nv.REPLACE_SIGNATURES["svi_replace_mask_stage"][1])
    consts = dict(re.findall(r"#define (SVI_SEG_\w+) (\d+)", text))
    assert (int(consts["SVI_SEG_U8"]), int(consts["SVI_SEG_F32"])) == (nv.SEG_U8, nv.SEG_F32)
