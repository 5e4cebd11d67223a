"""GPU: the wav2vec2 audio feature extractor on the native kernels (csrc/audio_kernels.cu + svi_gemm_bf16 + svi_attn_small)
against torch and the CPU oracle (oracle/wav2vec2_oracle.py, itself pinned to the reference module by
tests/golden/wav2vec_tiny.npz), and SVI-Talk driven by an audio file through the public pipeline API.

Yardsticks as in test_encoders_gpu.py, on bf16-rounded weights: the fp32 oracle (parity: mean |error| < 1.5 % of the
std) and the oracle's bf16-point mode (implementation check; at the tiny width the bf16 roundings of two accumulation
orders decorrelate, see test_audio_cpu.py)."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tools import synth_audio as SA

pytestmark = pytest.mark.gpu


def _bf(sd):
    return {k: v.to(torch.bfloat16).float() for k, v in sd.items()}


def _rel(out, ref):
    err = (out - ref).abs()
    return err.mean().item() / ref.std().item(), (err <= 1e-3 + 1e-2 * ref.abs()).float().mean().item()


def test_col_stats_exact_and_reproducible():
    """svi_col_stats vs fp64 torch: ragged T (1 row, a partial row block, more than 1024 blocks' worth), C = 1, 512 and a
    48-column window of a wider matrix; two runs are bit-identical."""
    from diffsynth import _native as nv
    g = torch.Generator().manual_seed(0)
    for T, C, ld in ((1, 512, 512), (37, 1, 1), (70001, 512, 512), (3000, 48, 768), (300000, 32, 32)):
        x = (torch.randn(T, ld, generator=g) * 3 + 1.5).cuda()
        v = x[:, 16:16 + C] if ld > C else x
        mean, var = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
        ws = torch.empty(nv.col_stats_workspace_bytes(T, C), device="cuda", dtype=torch.uint8)
        nv.col_stats(v, mean, var, ws)
        vd = v.double().cpu()
        assert (mean.cpu().double() - vd.mean(0)).abs().max().item() < 1e-6 * (1 + vd.abs().max().item())
        vr = vd.var(0, unbiased=False)
        assert (var.cpu().double() - vr).abs().max().item() < 1e-5 * (1 + vr.max().item())
        m2, v2 = torch.empty_like(mean), torch.empty_like(var)
        nv.col_stats(v, m2, v2, ws)
        assert torch.equal(mean, m2) and torch.equal(var, v2)


def test_col_norm_act_matches_torch():
    from diffsynth import _native as nv
    g = torch.Generator().manual_seed(1)
    for T, C in ((5, 1), (1001, 512)):
        x = torch.randn(T, C, generator=g).cuda()
        mean, var = torch.randn(C, generator=g).cuda(), torch.rand(C, generator=g).cuda() + 0.1
        gam, bet = torch.randn(C, generator=g).cuda(), torch.randn(C, generator=g).cuda()
        out = torch.empty(T, C, device="cuda", dtype=torch.bfloat16)
        nv.col_norm_act(x, mean, var, 1e-5, gam, bet, nv.ACT_GELU_ERF, out)
        ref = F.gelu((x - mean) * torch.rsqrt(var + 1e-5) * gam + bet)
        assert (out.float() - ref).abs().max().item() <= 1e-2 * ref.abs().max().item()


@pytest.mark.parametrize("src_dtype,T_in,C,ld,col0,k,s,pl,pr,T_out,split", [
    (torch.float32, 1001, 1, 1, 0, 10, 5, 0, 0, None, True),          # conv 0 of the waveform, two-term form
    (torch.bfloat16, 777, 512, 512, 0, 3, 2, 0, 0, None, False),      # k = 3 / s = 2 layers
    (torch.float32, 151, 48, 768, 96, 128, 1, 64, 64, 151, False),    # one group of the positional conv, last output dropped
    (torch.float32, 3, 16, 64, 48, 16, 1, 8, 8, 3, False),            # fewer rows than taps
    (torch.bfloat16, 64, 24, 40, 8, 2, 2, 0, 0, None, False),         # Kpad > k * C (zero tail)
])
def test_conv1d_gather_matches_torch(src_dtype, T_in, C, ld, col0, k, s, pl, pr, T_out, split):
    import nv_emulation_audio as E
    from diffsynth import _native as nv
    g = torch.Generator().manual_seed(2)
    src = torch.randn(T_in, ld, generator=g).to(src_dtype)
    T_out = T_out or (T_in + pl + pr - k) // s + 1
    kpad = (k * C + 7) // 8 * 8 + (8 if C == 24 else 0)
    out = torch.full((T_out, kpad * (2 if split else 1)), 7.0, device="cuda", dtype=torch.bfloat16)
    nv.conv1d_gather(src.cuda(), out, k, s, pl, pr, col0=col0, C=C, split=split)
    ref = torch.empty(T_out, kpad * (2 if split else 1), dtype=torch.bfloat16)
    E.conv1d_gather(src, ref, k, s, pl, pr, col0=col0, C=C, split=split)
    assert torch.equal(out.cpu(), ref)


@pytest.mark.parametrize("T_in,T_out,C", [(299, 150, 512), (50, 1, 512), (7, 61, 32), (3042, 1521, 512), (2, 2, 48)])
def test_interp_layernorm_matches_torch(T_in, T_out, C):
    from diffsynth import _native as nv
    g = torch.Generator().manual_seed(3)
    x = torch.randn(T_in, C, generator=g)
    gam, bet = torch.randn(C, generator=g), torch.randn(C, generator=g)
    out = torch.empty(T_out, C, device="cuda", dtype=torch.bfloat16)
    nv.interp_layernorm(x.cuda(), T_out, gam.cuda(), bet.cuda(), 1e-5, out)
    y = F.interpolate(x.t().unsqueeze(0), size=T_out, mode="linear", align_corners=True)[0].t()
    ref = F.layer_norm(y, (C,), gam, bet, 1e-5)
    err = (out.float().cpu() - ref).abs()
    assert (err <= 1e-2 * ref.abs() + 2e-2).all(), err.max()


def _model(cfg, seed):
    from diffsynth.models.wav2vec2 import Wav2Vec2Model
    sd = _bf(SA.make_state_dict(cfg, seed=seed))
    m = Wav2Vec2Model(cfg).eval()
    m.load_state_dict(sd)
    return m, sd


def _run(cfg, seconds, seed, bf16_bar=None):
    from oracle import wav2vec2_oracle as O
    m, sd = _model(cfg, seed)
    speech = SA.make_waveform(seconds, seed=seed + 1)
    iv = O.normalize(speech)
    T = O.seq_len_for(len(speech))
    out = m.engine("cuda").forward(torch.from_numpy(iv), T)
    got = out.stacked.cpu()
    torch.set_num_threads(8)
    ref = torch.stack(O.forward(sd, cfg, iv, T))
    rel, inside = _rel(got, ref)
    res = {"fp32": (rel, inside)}
    if bf16_bar is not None:
        refb = torch.stack(O.forward(sd, cfg, iv, T, bf16_points=True, split_conv0=True))
        res["bf16_points"] = _rel(got, refb)
    print(f"wav2vec2 {cfg['hidden_size']}x{cfg['num_hidden_layers']} {seconds}s: {res}")
    return res


def test_tiny_model_matches_oracle():
    """H100: fp32 oracle 0.39 % of the std; bf16-point oracle 0.30 %, 84 % inside rtol 1e-2 / atol 1e-3."""
    r = _run(SA.TINY_ENGINE, 3.3, 1, bf16_bar=True)
    assert r["fp32"][0] < 1.5e-2
    assert r["bf16_points"][0] < 6e-3 and r["bf16_points"][1] > 0.75


def test_base_model_matches_oracle_3s():
    """H100: fp32 oracle 0.30 % of the std (83 % inside); bf16-point oracle 0.38 %."""
    r = _run(SA.BASE, 3.0, 2, bf16_bar=True)
    assert r["fp32"][0] < 1.5e-2
    assert r["bf16_points"][0] < 6e-3


@pytest.mark.slow
def test_base_model_matches_oracle_61s():
    """H100: fp32 oracle 0.29 % of the std over 1525 frames x 13 hidden states."""
    r = _run(SA.BASE, 61.0, 3)
    assert r["fp32"][0] < 1.5e-2


# --------------------------------------------------------------------------------------------- SVI-Talk from an audio file
H, W, FRAMES, STEPS, CTX = 64, 96, 9, 2, 24


class _ClipStub:
    def __init__(self):
        self.proj = torch.randn(3, 257 * 1280, generator=torch.Generator().manual_seed(99)) * 0.5

    def encode_image(self, images):
        return (images[0].float().cpu().mean(dim=(0, 2, 3)) @ self.proj).reshape(1, 257, 1280)


def test_talk_pipeline_from_audio_path(tmp_path):
    """pipe(audio_path=...) as test_svi_talk.py calls it: a 44.1 kHz stereo WAV and a base-size wav2vec2 checkpoint
    directory; tiny talk DiT.  The windows match the oracle's, the second clip reuses the cached features, two extractions
    are bit-identical, and the frames made from the audio file differ from those made from the oracle's windows by less
    than 0.1 of what silent audio changes.  H100: windows 0.32 % of the std from the fp32 oracle's; frames 0.60 levels
    from the oracle-window clip against 39.6 levels for silent audio."""
    from diffsynth import ModelManager, SVITalkVideoPipeline
    from diffsynth.models.wan_video_dit import WanModel
    from diffsynth.models.wan_video_vae import WanVideoVAE
    from oracle import wav2vec2_oracle as O
    from PIL import Image
    from tools import synth, synth_vae
    from utils.audio_process import audio_prepare_single
    cfg = SA.BASE
    m, sd = _model(cfg, 4)
    ck = SA.write_checkpoint(str(tmp_path / "chinese-wav2vec2-base"), cfg, m.state_dict())
    wav = SA.write_wav(str(tmp_path / "talk.wav"), SA.make_waveform(4.0, sr=44100, seed=6, channels=2), 44100, "int16")
    dcfg = synth.CFG_TINY_TALK
    dit = WanModel(**dcfg).eval()
    dit.load_state_dict({k: v.to(torch.bfloat16).float() for k, v in synth.make_dit_state_dict(dcfg, seed=5).items()})
    vae = WanVideoVAE().eval()
    vae.load_state_dict({k: v.to(torch.bfloat16).float() for k, v in synth_vae.make_vae_state_dict(seed=0).items()})
    mm = ModelManager(torch_dtype=torch.bfloat16, device="cuda")
    mm.add_model("wan_video_dit", dit.to("cuda"))
    mm.add_model("wan_video_vae", vae.to("cuda"))
    pipe = SVITalkVideoPipeline.from_model_manager(mm, torch_dtype=torch.bfloat16, device="cuda", is_test=True, wav2vec_path=ck)
    pipe.prompter = lambda prompt, positive=True: torch.randn(1, CTX, dcfg["text_dim"], generator=torch.Generator().manual_seed(11 if positive else 12))
    pipe.image_encoder = _ClipStub()
    img = Image.fromarray(np.random.default_rng(5).integers(0, 255, size=(H, W, 3), dtype=np.uint8))
    # windows against the oracle (fp32, same prepared waveform)
    w0 = pipe.get_audio_embedding(wav, FRAMES, audio_start_idx=0)
    w1 = pipe.get_audio_embedding(wav, FRAMES, audio_start_idx=95)
    assert pipe.audio_extractions == 1 and w0.shape == (1, FRAMES, 5, 12, 768) and w0.is_cuda
    torch.set_num_threads(8)
    emb = O.embedding(sd, cfg, audio_prepare_single(wav))
    for w, s in ((w0, 0), (w1, 95)):
        rel, _ = _rel(w.cpu(), O.windows(emb, FRAMES, s))
        print(f"windows at {s}: mean|err|/std = {rel:.4e}")
        assert rel < 1.5e-2
    first = pipe.audio_hidden_states(wav).clone()
    pipe._audio_cache = None
    assert torch.equal(pipe.audio_hidden_states(wav), first) and pipe.audio_extractions == 2
    # one clip from the file, from the oracle's windows and from silence
    args = types.SimpleNamespace(ref_pad_cfg=False, ref_pad_num=-1, sequential_cfg="none")
    kw = dict(prompt="p", negative_prompt="n", input_image=img, num_inference_steps=STEPS, cfg_scale={"text": 5.0, "audio": 4.0},
              seed=42, tiled=False, random_ref_frame=torch.from_numpy(np.array(img)), height=H, width=W, num_frames=FRAMES,
              args=args, progress_bar_cmd=lambda x: x)
    clip = lambda **extra: np.stack([np.array(f) for f in pipe(**kw, **extra)]).astype(np.float32)
    from_file = clip(audio_path=wav, audio_start_idx=0)
    assert pipe.audio_extractions == 2
    from_oracle = clip(audio_embed=O.windows(emb, FRAMES, 0))
    silent = clip(audio_embed=torch.zeros(1, FRAMES, 5, 12, 768))
    d_audio, d_silent = np.abs(from_file - from_oracle).mean(), np.abs(silent - from_oracle).mean()
    print(f"talk clip: |file - oracle windows| = {d_audio:.3f} levels, |silent - oracle windows| = {d_silent:.3f} levels")
    assert d_silent > 0.5 and d_audio < 0.1 * d_silent
