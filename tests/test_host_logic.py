"""CPU tests of the host-side logic and of the C-ABI surface (no kernel is launched here)."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


# ------------------------------------------------------------------------------------------- C ABI
def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "svi_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(svi_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from diffsynth import _native as nv
    lib = nv.load()                       # raises if the .so is missing (build() must have run)
    declared = _declared_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/svi_b200.h but not exported"
        assert name in nv.SIGNATURES, f"{name} has no ctypes signature in diffsynth/_native.py"
    assert sorted(nv.SIGNATURES) == declared
    assert lib.svi_abi_version() == 4


def test_header_is_plain_c():
    """The drop-in boundary is a C ABI: the header must compile as C99 (no C++ or torch types in the signatures)."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    r = subprocess.run(["gcc", "-fsyntax-only", "-x", "c", "-std=c99", "-Wall", "-pedantic", os.path.join(ROOT, "include", "svi_b200.h")],
                       capture_output=True, text=True)
    assert r.returncode == 0 and r.stderr.strip() == "", r.stderr


def test_library_contains_hopper_tensor_and_tma_instructions():
    """SASS evidence that the hot kernels are wgmma / TMA code for sm_90a (HGMMA, UTMALDG), with no warp-level mma.sync path."""
    from diffsynth import _native as nv
    try:
        sass = subprocess.run(["cuobjdump", "-sass", nv.lib_path()], capture_output=True, text=True, timeout=300).stdout
    except FileNotFoundError:
        pytest.skip("cuobjdump not available")
    assert "sm_90a" in subprocess.run(["cuobjdump", "-lelf", nv.lib_path()], capture_output=True, text=True).stdout
    for mnemonic in ("HGMMA.64x256x16.F32.BF16", "HGMMA.64x128x16.F32.BF16", "UTMALDG"):
        assert mnemonic in sass, f"{mnemonic} not found in the library's SASS"
    assert "HMMA.16816" not in sass       # no legacy mma.sync tensor path


def test_attention_launch_plan_slices_only_the_partial_wave():
    """svi_attn_plan (host logic of svi_attn_fwd): whole units for the full waves, K/V slices for the last partial one."""
    from diffsynth import _native as nv
    big = 1 << 40
    slice_bytes = 128 * 128 * 4 + 128 * 8
    # bench shape on one H100 (132 SMs): 12 heads x 256 Q tiles = 3072 units = 23.27 waves
    n_full, split = nv.attention_plan(3072, 256, 132, big)
    tail = 3072 - n_full
    assert split > 1 and n_full % 132 == 0 and 0 < tail <= 2 * 132
    waves = n_full / 132 + -(-tail * split // 132) / split
    assert waves < 23.75                                            # 24 waves unsliced
    # sequence-parallel shape sp = 2: 11.64 waves
    nf, sp = nv.attention_plan(1536, 256, 132, big)
    assert sp > 1 and nf / 132 + -(-(1536 - nf) * sp // 132) / sp < -(-1536 // 132) - 0.3
    # sp = 4: 768 units = 5.82 waves, the last one 82 % full: slicing cannot save 1.5 %, so nothing is sliced
    assert nv.attention_plan(768, 256, 132, big) == (768, 1)
    assert nv.attention_plan(3072, 256, 132, 0) == (3072, 1)        # no workspace: nothing sliced
    assert nv.attention_plan(3036, 256, 132, big) == (3036, 1)      # exact multiple of the SM count
    assert nv.attention_plan(3072, 4, 132, big) == (3072, 1)        # cross-attention: K/V stream too short to slice
    nf, sp = nv.attention_plan(3072, 256, 132, 100 * slice_bytes)   # workspace for 100 slices only
    assert sp > 1 and (3072 - nf) * sp <= 100


def test_native_calls_refuse_cpu_tensors():
    from diffsynth import _native as nv
    a = torch.zeros(8, 8, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="CUDA"):
        nv.gemm(a, a, torch.zeros(8, 8))


def test_models_fail_loudly_without_cuda():
    from diffsynth.models.wan_video_dit import WanModel
    from diffsynth.models.wan_video_vae import WanVideoVAE
    from tools import synth
    m = WanModel(**synth.CFG_TINY_T2V)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.engine("cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        WanVideoVAE().engine("cpu")


def test_encoders_fail_loudly_without_cuda_and_host_tables_match_the_oracle():
    from diffsynth.models.wan_video_image_encoder import WanImageEncoder
    from diffsynth.models.wan_video_text_encoder import WanTextEncoder, relative_position_buckets
    from oracle import wan_encoders_oracle as E
    from tools import synth_enc as SE
    with pytest.raises(RuntimeError, match="CUDA"):
        WanTextEncoder(**SE.TEXT_TINY).engine("cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        WanImageEncoder(**SE.CLIP_TINY).engine("cpu")
    for L in (24, 512):
        assert torch.equal(relative_position_buckets(L, L, 32).long(), E.t5_relative_buckets(L, L, 32))


def test_meta_construction_keeps_constant_tables_real():
    """ModelManager builds models under init_weights_on_device() (device 'meta') and then assigns the checkpoint tensors
    (reference model_manager.py:57-105).  Tables that are not parameters — the RoPE frequencies, the VAE latent
    statistics — must stay real tensors, or the first forward after loading a real checkpoint would read meta data."""
    from diffsynth.models.utils import init_weights_on_device
    from diffsynth.models.wan_video_dit import WanModel
    from diffsynth.models.wan_video_vae import WanVideoVAE
    from tools import synth
    with init_weights_on_device():
        m = WanModel(**synth.CFG_TINY_I2V)
        v = WanVideoVAE()
    assert all(p.is_meta for p in m.parameters())
    assert all(not f.is_meta and f.device.type == "cpu" for f in m.freqs) and m.freqs[0].shape == (1024, 22)
    assert not v.mean.is_meta and not v.std.is_meta and v.mean.numel() == 16
    sd = synth.make_dit_state_dict(synth.CFG_TINY_I2V, seed=0)
    m.load_state_dict(sd, assign=True)
    assert not any(p.is_meta for p in m.parameters())


def test_encoder_key_contracts():
    """umT5: the parameter names hash to the reference's checkpoint fingerprint (model_config.py:122).  CLIP: the real
    checkpoint also carries the text tower, which the converter drops (wan_video_image_encoder.py:894-901); what is left
    must be exactly the visual-tower names the reference module registers."""
    from diffsynth.models.model_manager import ModelManager
    from diffsynth.models.utils import hash_state_dict_keys
    from diffsynth.models.wan_video_image_encoder import WanImageEncoder
    from diffsynth.models.wan_video_text_encoder import WanTextEncoder
    from tools import synth_enc as SE
    with torch.device("meta"):
        te = WanTextEncoder()
        ie = WanImageEncoder()
    sd = te.state_dict()
    assert hash_state_dict_keys(sd, with_shape=True) == "9c8818c2cbea55eca56c7b447df170da"
    det = ModelManager(torch_dtype=torch.bfloat16, device="cpu").model_detector[0]
    names, classes, _ = det._lookup(sd)
    assert names == ["wan_video_text_encoder"] and classes == [WanTextEncoder]
    want = set(SE.clip_param_shapes(SE.CLIP_VIT_H)) | {"model.log_scale"}
    have = {k: tuple(v.shape) for k, v in ie.state_dict().items()}
    assert set(have) == want and all(have[k] == v for k, v in SE.clip_param_shapes(SE.CLIP_VIT_H).items())
    ckpt = {"log_scale": 0, "visual.head": 1, "textual.token_embedding.weight": 2, "visual.transformer.0.norm1.weight": 3}
    conv = WanImageEncoder.state_dict_converter().from_civitai(ckpt)
    assert set(conv) == {"model.log_scale", "model.visual.head", "model.visual.transformer.0.norm1.weight"}


# ------------------------------------------------------------------------------------------- key contracts
def test_parameter_names_hash_to_the_reference_checkpoint_fingerprints():
    """The reference detects checkpoints by md5 of sorted 'key:shape' strings (model_config.py:117-125)."""
    from diffsynth.models.utils import hash_state_dict_keys
    from diffsynth.models.wan_video_dit import WanModel
    from diffsynth.models.wan_video_vae import WanVideoVAE
    from tools import synth
    for cfg, want in ((synth.CFG_T2V_1_3B, "9269f8db9040a9d860eaca435be61814"), (synth.CFG_I2V_14B, "6bfcfb3b342cb286ce886889d519a77e")):
        with torch.device("meta"):
            m = WanModel(**cfg)
        assert hash_state_dict_keys(m.state_dict()) == want
    vae = WanVideoVAE()
    assert hash_state_dict_keys({k[len("model."):]: v for k, v in vae.state_dict().items()}) == "ccc42284ea13e1ad04693284c7a09be6"


def test_model_detector_resolves_wan_checkpoints_and_fixes_the_1p3b_config():
    from diffsynth.models.model_manager import ModelDetectorFromSingleFile, _loader_table
    from diffsynth.models.wan_video_dit import WanModel, WanModelStateDictConverter
    from tools import synth
    det = ModelDetectorFromSingleFile(_loader_table())
    sd = {k: torch.empty(s, device="meta") for k, s in synth.dit_param_shapes(synth.CFG_T2V_1_3B).items()}
    names, classes, resource = det._lookup(sd)
    assert names == ["wan_video_dit"] and classes == [WanModel] and resource == "civitai"
    _, cfg = WanModelStateDictConverter().from_civitai(sd)
    assert cfg["dim"] == 1536 and cfg["num_layers"] == 30      # the reference returns {} here (SURVEY.md headline 7)
    assert det._lookup({"foo.weight": torch.empty(1, device="meta")}) is None


def test_lora_key_matching():
    from diffsynth.models.lora import GeneralLoRAFromPeft
    from diffsynth.models.wan_video_dit import WanModel
    from tools import synth
    with torch.device("meta"):
        m = WanModel(**synth.CFG_TINY_T2V)
    lora = GeneralLoRAFromPeft()
    sd = {"blocks.0.self_attn.q.lora_A.default.weight": torch.zeros(4, 256), "blocks.0.self_attn.q.lora_B.default.weight": torch.zeros(256, 4),
          "diffusion_model.blocks.1.ffn.0.lora_A.weight": torch.zeros(4, 256), "diffusion_model.blocks.1.ffn.0.lora_B.weight": torch.zeros(512, 4)}
    names = lora.get_name_dict(sd)
    assert set(names) == {"blocks.0.self_attn.q.weight", "blocks.1.ffn.0.weight"}
    assert lora.match(m, sd) == ("", "")
    assert lora.match(m, {"pipe.dit.blocks.0.self_attn.q.lora_B.default.weight": torch.zeros(1)}) is None


def test_load_lora_v2_strips_pipe_dit_prefix_and_raises_when_nothing_matches():
    from diffsynth.models.model_manager import ModelManager
    mm = ModelManager(device="cpu")
    with pytest.raises(RuntimeError, match="Cannot load LoRA"):
        mm.load_lora_v2("x.safetensors", state_dict={"pipe.dit.blocks.0.q.lora_B.default.weight": torch.zeros(2, 2),
                                                     "pipe.dit.blocks.0.q.lora_A.default.weight": torch.zeros(2, 2)})
    assert "blocks.0.q.lora_B.default.weight" in mm.state_dict_new
    assert mm.fetch_model("wan_video_dit") is None


# ------------------------------------------------------------------------------------------- scheduler
def test_scheduler_matches_reference_golden():
    from diffsynth.schedulers.flow_match import FlowMatchScheduler
    g = np.load(os.path.join(GOLD, "flow_match.npz"))
    for steps in (1, 4, 50):
        s = FlowMatchScheduler(shift=5, sigma_min=0.0, extra_one_step=True)
        s.set_timesteps(steps, denoising_strength=1.0, shift=5.0)
        np.testing.assert_allclose(s.sigmas.numpy(), g[f"sigmas_{steps}"], atol=1e-7)
        np.testing.assert_allclose(s.timesteps.numpy(), g[f"timesteps_{steps}"], atol=1e-4)
    s = FlowMatchScheduler(shift=5, sigma_min=0.0, extra_one_step=True)
    s.set_timesteps(4, shift=5.0)
    x = torch.from_numpy(g["step_x"][0])
    for i in range(4):
        x = s.step(torch.from_numpy(g["step_v"][i]), s.timesteps[i], x)
        np.testing.assert_allclose(x.numpy(), g["step_x"][i + 1], rtol=1e-6, atol=1e-6)
    assert s.sigma_pair(s.timesteps[3]) == (pytest.approx(float(s.sigmas[3])), 0.0)


# ------------------------------------------------------------------------------------------- harness helpers
def test_calculate_dimensions_matches_survey_geometry():
    from PIL import Image
    from utils.image_process import calculate_dimensions
    # SURVEY.md §4: toy inputs -> (H, W) with max_width 832
    for (w, h), want in (((1024, 571), (448, 832)), ((832, 480), (480, 832)), ((1129, 779), (560, 832)),
                         ((604, 1080), (1072, 592)), ((572, 499), (496, 560))):
        assert calculate_dimensions(Image.new("RGB", (w, h)), max_width=832) == want


def test_pipeline_size_rounding_and_noise_seed():
    from diffsynth.pipelines.svi_video import SVIVideoPipeline
    p = SVIVideoPipeline(device="cpu", torch_dtype=torch.bfloat16)
    assert p.check_resize_height_width(470, 832) == (480, 832)
    a = p.generate_noise((1, 16, 2, 4, 4), seed=7, device="cpu", dtype=torch.float32)
    b = p.generate_noise((1, 16, 2, 4, 4), seed=7, device="cpu", dtype=torch.float32)
    assert torch.equal(a, b)
    with pytest.raises(RuntimeError, match="prompt encoder"):
        p.encode_prompt("a cat")


def test_vae_weight_packing_space_to_depth_equivalence():
    """The stride-2 conv re-packing used by the native VAE equals the original conv (checked with torch on CPU)."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(0)
    w = torch.randn(5, 3, 3, 3, generator=g)
    x = torch.randn(1, 3, 8, 10, generator=g)
    ref = F.conv2d(F.pad(x, (0, 1, 0, 1)), w, stride=2)
    w2 = torch.zeros(5, 12, 2, 2)
    for bh in range(2):
        for bw in range(2):
            for dy in range(2):
                for dx in range(2):
                    a, b = 2 * bh + dy, 2 * bw + dx
                    if a <= 2 and b <= 2:
                        w2[:, (dy * 2 + dx) * 3:(dy * 2 + dx + 1) * 3, bh, bw] = w[:, :, a, b]
    s2d = x.view(1, 3, 4, 2, 5, 2).permute(0, 3, 5, 1, 2, 4).reshape(1, 12, 4, 5)
    out = F.conv2d(F.pad(s2d, (0, 1, 0, 1)), w2)
    torch.testing.assert_close(out, ref, rtol=1e-5, atol=1e-5)


def test_pose_stem_strided_conv_repacking():
    """nn.Conv3d(k=3, stride (1|2, 2, 2), padding 1) of the SVI-Dance pose stem == 2x2 spatial taps over the space-to-depth
    input with one block of zero padding in front (models/wan_video_vae._Conv(s2d="before")); checked with torch ops."""
    import torch.nn.functional as F
    from diffsynth.models.wan_video_vae import _Conv
    g = torch.Generator().manual_seed(0)
    C, O, T, H, W = 16, 16, 5, 8, 12
    bf = lambda t: t.to(torch.bfloat16).float()
    w = bf(torch.randn(O, C, 3, 3, 3, generator=g) * 0.2)
    b = torch.randn(O, generator=g)
    x = torch.randn(1, C, T, H, W, generator=g)
    cv = _Conv(w, b, "cpu", s2d="before")
    assert (cv.kt, cv.kh, cv.kw, cv.c_in) == (3, 2, 2, 4 * C)
    w2 = cv.w.float().reshape(cv.w.shape[0], 3, 2, 2, cv.cpad)[:O, :, :, :, :4 * C].permute(0, 4, 1, 2, 3)   # [O, 4C, 3, 2, 2]
    # space-to-depth: channel (dy*2+dx)*C + c of block (by, bx) = pixel (2by+dy, 2bx+dx)
    xs = x.reshape(1, C, T, H // 2, 2, W // 2, 2).permute(0, 4, 6, 1, 2, 3, 5).reshape(1, 4 * C, T, H // 2, W // 2)
    xs = F.pad(xs, (1, 0, 1, 0, 1, 1))                       # one zero block before in W and H; symmetric in time
    for ts in (1, 2):
        want = F.conv3d(x, w, b, stride=(ts, 2, 2), padding=(1, 1, 1))
        got = F.conv3d(xs, w2, b, stride=(ts, 1, 1))
        assert got.shape == want.shape and (got - want).abs().max().item() < 1e-4


def test_pose_stem_plan_reproduces_the_reference_stem_on_cpu():
    """Everything of DWPoseEmbeddingEngine that is host logic — weight packing of the seven convolutions, frame-slot
    tables (symmetric temporal padding, temporal stride), SiLU / space-to-depth staging order, the final projection as
    space-to-depth + matrix product — replayed with torch ops on the CPU in place of the kernels, against the oracle."""
    import torch.nn.functional as F
    from diffsynth.models.dwpose_embedding import StemPlan, make_dwpose_embedding, slot_table
    from oracle import dwpose_oracle as DO
    g = torch.Generator().manual_seed(1)
    dim, T, H, W = 64, 5, 16, 32
    seq = make_dwpose_embedding(dim=dim)
    sd = {k: (torch.randn(v.shape, generator=g) * (0.1 if k.endswith("bias") else 1.5 / v[0].numel() ** 0.5)).to(torch.bfloat16).float()
          for k, v in seq.state_dict().items()}
    seq.load_state_dict(sd)
    plan = StemPlan(seq, "cpu")
    pose = torch.randint(0, 256, (3, T, H, W), generator=g).float()
    want = DO.pose_condition(sd, pose)

    def conv(cv, frames_cl, T_out, ts):
        """frames_cl: list of channels-last frames [H, W, C_ring] (what the ring slots hold); kernel semantics of
        svi_conv3d_causal: out[t] = bias + sum over taps of w[o, a, kh, kw, c] * ring[slot[t][a]][y+kh-1][x+kw-1][c]."""
        Hh, Ww, Cr = frames_cl[0].shape
        zero = torch.zeros_like(frames_cl[0])
        w = cv.w.float().reshape(cv.w.shape[0], cv.kt, cv.kh, cv.kw, cv.cpad)[:cv.c_out, :, :, :, :Cr]
        table = slot_table(list(range(len(frames_cl))), len(frames_cl), T_out, ts, cv.kt)
        outs = []
        for t in range(T_out):
            acc = cv.b[:cv.c_out].view(1, -1, 1, 1).expand(1, cv.c_out, Hh, Ww).clone()
            for a in range(cv.kt):
                src = zero if table[t][a] == len(frames_cl) else frames_cl[table[t][a]]
                xin = F.pad(src.permute(2, 0, 1).unsqueeze(0), (1, cv.kw - 2, 1, cv.kh - 2))   # pad 1 before; after: k-2
                acc = acc + F.conv2d(xin, w[:, a].permute(0, 3, 1, 2))
            outs.append(acc[0].permute(1, 2, 0))
        return outs

    x = torch.cat([pose[:, :1].repeat(1, 3, 1, 1), pose], dim=1) / 255.0
    Tn = x.shape[1]
    frames = [F.pad(x[:, t].permute(1, 2, 0), (0, plan.full[0].c_in - 3)) for t in range(Tn)]
    cur = conv(plan.full[0], frames, Tn, 1)
    for cv in plan.full[1:]:
        frames = [F.pad(F.silu(f), (0, cv.c_in - f.shape[-1])) for f in cur]
        cur = conv(cv, frames, Tn, 1)

    def s2d(f):
        Hh, Ww, C = f.shape
        return f.reshape(Hh // 2, 2, Ww // 2, 2, C).permute(0, 2, 1, 3, 4).reshape(Hh // 2, Ww // 2, 4 * C)

    for cv, ts in zip(plan.down, plan.t_stride):
        frames = [s2d(F.silu(f)) for f in cur]
        cur = conv(cv, frames, (len(cur) + 2 - 3) // ts + 1, ts)
    a = torch.stack([F.pad(s2d(F.silu(f)), (0, plan.kproj - 4 * f.shape[-1])) for f in cur]).reshape(-1, plan.kproj)
    got = (a @ plan.w_proj.float().T + plan.b_proj).unsqueeze(0)
    assert got.shape == want.shape
    assert (got - want).abs().max().item() < 1e-3 * max(1.0, want.abs().max().item())


def test_talk_model_key_contract_and_audio_windows():
    """SVI-Talk: the enable_multitalk 14B-I2V parameter names hash to the reference fingerprint (model_config.py:120,
    wan_video_dit.py:670-684) and the detector hands WanModel the multitalk config; preprocess_audio equals the oracle's
    window selection (itself pinned to svi_video_talk.py:432-446 by the golden fixture)."""
    from diffsynth.models.model_manager import ModelManager
    from diffsynth.models.utils import hash_state_dict_keys
    from diffsynth.models.wan_video_dit import WanModel
    from diffsynth.pipelines.svi_video_talk import preprocess_audio
    from oracle import wan_dit_oracle as O
    from tools import synth
    with torch.device("meta"):
        m = WanModel(**dict(synth.CFG_I2V_14B, enable_multitalk=True))
    sd = m.state_dict()
    assert hash_state_dict_keys(sd, with_shape=True) == "b6caaaa1388107ec24d25592901ca489"
    det = ModelManager(torch_dtype=torch.bfloat16, device="cpu").model_detector[0]
    names, classes, resource = det._lookup(sd)
    assert names == ["wan_video_dit"] and classes == [WanModel] and resource == "civitai"
    _, cfg = WanModel.state_dict_converter().from_civitai(sd)
    assert cfg["enable_multitalk"] is True and cfg["dim"] == 5120 and cfg["has_image_input"] is True
    a = synth.make_audio_embed(13, seed=2)
    for x, y in zip(preprocess_audio(a), O.preprocess_audio(a)):
        assert torch.equal(x, y)
    with pytest.raises(ValueError):
        preprocess_audio(synth.make_audio_embed(11))


def test_model_manager_loads_a_sharded_vae_checkpoint_end_to_end(tmp_path):
    """The whole checkpoint path of test_svi.py:253-262 on a real-size file set: a Wan VAE state dict (un-prefixed keys,
    fingerprint ccc42284…) written as two safetensors shards -> ModelManager.load_models([[shard, shard]]) merges them
    (reference model_manager.py:660-663), detects the model by its key hash, constructs on 'meta', converts the keys,
    assigns the tensors and casts -> fetch_model returns a usable WanVideoVAE whose constant tables are real tensors."""
    from safetensors.torch import save_file
    from diffsynth import ModelManager
    from diffsynth.models.wan_video_vae import WanVideoVAE
    from tools import synth_vae
    sd = {k[len("model."):]: v.to(torch.bfloat16).contiguous() for k, v in synth_vae.make_vae_state_dict(seed=0).items()}
    keys = sorted(sd)
    a, b = str(tmp_path / "vae-00001-of-00002.safetensors"), str(tmp_path / "vae-00002-of-00002.safetensors")
    save_file({k: sd[k] for k in keys[::2]}, a)
    save_file({k: sd[k] for k in keys[1::2]}, b)
    mm = ModelManager(torch_dtype=torch.float32, device="cpu")
    mm.load_models([[a, b]])
    hit = mm.fetch_model("wan_video_vae", require_model_path=True)
    assert hit is not None and isinstance(hit[0], WanVideoVAE) and hit[1] == [a, b]
    vae = hit[0]
    assert not any(p.is_meta for p in vae.parameters()) and all(p.dtype == torch.float32 for p in vae.parameters())
    assert not vae.mean.is_meta and vae.mean.shape == (16,)
    got = dict(vae.named_parameters())
    for k in (keys[0], keys[len(keys) // 2], keys[-1]):
        assert torch.equal(got["model." + k], sd[k].float())
    assert mm.fetch_model("wan_video_dit") is None
    with pytest.raises(RuntimeError, match="cannot detect"):
        bad = str(tmp_path / "other.safetensors")
        save_file({"foo.weight": torch.zeros(2, 2)}, bad)
        mm.load_models([bad])


def test_streaming_video_writer_appends_clips(tmp_path):
    """StreamingVideoWriter (the clip loop's append-only output, SURVEY 8f.3): frames of successive clips land in one output
    in order, whatever writer backend this image has (none here: PNG frames)."""
    import numpy as np
    from PIL import Image
    from diffsynth import StreamingVideoWriter
    mk = lambda v: Image.fromarray(np.full((8, 12, 3), v, dtype=np.uint8))
    w = StreamingVideoWriter(str(tmp_path / "out.mp4"), fps=16)
    assert w.append([mk(1), mk(2), mk(3)]) == 3
    assert w.append([mk(4), mk(5)]) == 5
    out = w.close()
    assert os.path.exists(out)
    if os.path.isdir(out):
        vals = [int(np.array(Image.open(os.path.join(out, f"{i}.png")))[0, 0, 0]) for i in range(5)]
        assert vals == [1, 2, 3, 4, 5]


def test_ctypes_mirrors_match_the_c_struct_layouts(tmp_path):
    """The two descriptor structs of the C ABI (svi_gemm_epilogue, svi_conv_desc) are mirrored by hand in _native.py: compile a
    probe against include/svi_b200.h with the C compiler and compare sizeof / offsetof of every field with ctypes."""
    import ctypes
    import subprocess
    from diffsynth import _native as nv
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    structs = {"svi_gemm_epilogue": nv.GemmEpilogue, "svi_conv_desc": nv.ConvDesc}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "svi_b200.h"', 'int main(void) {']
    for cname, mirror in structs.items():
        lines.append(f'  printf("{cname} sizeof %zu\\n", sizeof({cname}));')
        for fname, _ in mirror._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    seen = 0
    for line in filter(None, out):
        cname, fname, val = line.split()
        mirror = structs[cname]
        want = ctypes.sizeof(mirror) if fname == "sizeof" else getattr(mirror, fname).offset
        assert int(val) == want, (cname, fname, int(val), want)
        seen += 1
    assert seen == sum(len(m._fields_) + 1 for m in structs.values())


def test_conv_kernel_choice_is_validated_before_anything_touches_the_gpu():
    """svi_conv_desc.variant (include/svi_b200.h): kept for ABI compatibility — 2 is accepted only with k_w = 3 and pad_w = 1,
    anything outside 0..2 is refused (every accepted value runs the same kernel).  The checks run before any tensor map / launch, so the error path is testable without a GPU."""
    from diffsynth import _native as nv
    lib = nv.load()

    def desc(kw, pad, variant):
        d = nv.ConvDesc()
        d.x_ring, d.w_packed, d.out = 0x1000, 0x2000, 0x3000          # never dereferenced: validation fails first
        d.ring_slots, d.in_H, d.in_W, d.C_in = 4, 8, 256, 64
        d.w_rows, d.w_ld = 96, 3 * 3 * kw * 64
        d.kt, d.kh, d.kw, d.pad_h, d.pad_w = 3, 3, kw, 1, pad
        d.H, d.W, d.T = 8, 256, 1
        for a in range(3):
            d.slot[a] = a
        d.C_out, d.tile_w, d.out_ld, d.out_frame_stride = 96, 16, 96, 8 * 256 * 96
        d.variant = variant
        return d

    import ctypes
    for kw, pad, variant, needle in [(1, 0, 2, "variant 2 needs"), (3, 1, 7, "variant must be"), (3, 0, 2, "variant 2 needs")]:
        d = desc(kw, pad, variant)
        rc = lib.svi_conv3d_causal(ctypes.byref(d), None)
        assert rc != 0
        assert needle in lib.svi_last_error().decode(), lib.svi_last_error().decode()
