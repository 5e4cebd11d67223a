"""GPU: UniAnimate-DiT — the window kernels against their torch stand-ins, the reference-pose stem against the oracle, and
one short clip and one long video (three windows, the last realigned) through the public pipelines against the same
video computed by the CPU oracles."""
import numpy as np
import pytest
import torch
from PIL import Image

from tools import synth, synth_unianimate as SU, synth_vae

pytestmark = pytest.mark.gpu

H, W, STEPS = 32, 48, 3


def test_window_kernels_equal_torch_stand_ins():
    import nv_emulation_unianimate as E
    from diffsynth import _native as nv
    from diffsynth.pipelines.wan_video import context_windows, window_counts
    g = torch.Generator(device="cuda").manual_seed(0)
    for n_lat, cs, ov, h, w in ((9, 5, 2, 4, 6), (41, 21, 4, 60, 104)):
        wins = context_windows(n_lat, cs, ov)
        assert wins[-1][0] == n_lat - cs
        count = torch.tensor(window_counts(wins, n_lat), dtype=torch.int32, device="cuda")
        outs = []
        for _ in range(2):
            acc, ref = torch.zeros(1, 16, n_lat, h, w, device="cuda"), torch.zeros(1, 16, n_lat, h, w, device="cuda")
            gen = torch.Generator(device="cuda").manual_seed(1)
            for k, win in enumerate(wins):
                x = torch.randn(1, 16, cs, h, w, device="cuda", generator=gen)
                nv.window_accumulate(x, 0 if k == 0 else 2, acc, win[0])
                E.window_accumulate(x, 0 if k == 0 else 2, ref, win[0])
            assert torch.equal(acc, ref)
            out, want = torch.empty_like(acc), torch.empty_like(acc)
            nv.window_normalize(acc, count, out)
            E.window_normalize(ref, count, want)
            assert torch.equal(out, want)
            nv.window_normalize(acc, count, acc)             # in place
            assert torch.equal(acc, want)
            outs.append(out)
        assert torch.equal(outs[0], outs[1])
    x = torch.randn(1, 16, 5, 4, 6, device="cuda", generator=g)
    acc = torch.zeros(1, 16, 9, 4, 6, device="cuda")
    with pytest.raises(RuntimeError, match="skip"):
        nv.window_accumulate(x, 5, acc, 0)
    with pytest.raises(RuntimeError, match="outside"):
        nv.window_accumulate(x, 0, acc, 5)
    with pytest.raises(RuntimeError, match="overlap"):
        nv.window_accumulate(acc, 0, acc, 0)


@pytest.mark.parametrize("h,w", [(64, 96), (80, 112)])
def test_ref_stem_matches_oracle(h, w):
    from diffsynth.models.dwpose_embedding import RandomRefEmbeddingEngine, make_randomref_embedding_pose
    from oracle import unianimate_oracle as U
    sd = SU.ref_stem_sd(seed=h)
    seq = make_randomref_embedding_pose()
    seq.load_state_dict(sd)
    img = SU.ref_pose(h, w, seed=w)
    got = RandomRefEmbeddingEngine(seq, "cuda").forward(img.permute(2, 0, 1).cuda() / 255.0).cpu()
    want = U.ref_stem(sd, img)
    err = (got - want).abs()
    rel = err.mean().item() / want.std().item()
    print(f"reference-pose stem {h}x{w}: max={err.max().item():.4e} mean/std={rel:.4e}")
    assert got.shape == want.shape and rel < 1e-2


def _bf(t):
    return t.to(torch.bfloat16).float()


def _pipe(cls):
    import test_dance_gpu as D
    from diffsynth import ModelManager
    from diffsynth.models.wan_video_dit import WanModel
    from diffsynth.models.wan_video_vae import WanVideoVAE
    cfg = synth.CFG_TINY_I2V
    dit_sd = {k: _bf(v) for k, v in synth.make_dit_state_dict(cfg, seed=2).items()}
    vae_sd = {k: _bf(v) for k, v in synth_vae.make_vae_state_dict(seed=0).items()}
    pose_sd, ref_sd = SU.pose_stem_sd(cfg["dim"], seed=7), SU.ref_stem_sd(seed=8)
    dit = WanModel(**cfg).eval()
    dit.load_state_dict(dit_sd)
    vae = WanVideoVAE().eval()
    vae.load_state_dict(vae_sd)
    mm = ModelManager(torch_dtype=torch.bfloat16, device="cuda")
    mm.add_model("wan_video_dit", dit.to("cuda"))
    mm.add_model("wan_video_vae", vae.to("cuda"))
    mm.state_dict_new_module = {"pipe.dwpose_embedding." + k: v for k, v in pose_sd.items()}
    mm.state_dict_new_module.update({"pipe.randomref_embedding_pose." + k: v for k, v in ref_sd.items()})
    pipe = cls.from_model_manager(mm, torch_dtype=torch.bfloat16, device="cuda")
    pipe.prompter = D._prompter
    pipe.image_encoder = D._ClipStub()
    return pipe, dict(cfg=cfg, dit=dit_sd, vae=vae_sd, pose=pose_sd, ref=ref_sd)


def _image():
    return Image.fromarray(np.random.default_rng(5).integers(0, 255, size=(H, W, 3), dtype=np.uint8))


def _oracle_conditioning(m, img, n_frames):
    """What the pipeline builds before its loop, on the CPU oracles: prompts, CLIP feature, y (+ reference pose)."""
    import test_dance_gpu as D
    from oracle import unianimate_oracle as U
    from oracle import wan_vae_oracle as V
    x = torch.from_numpy(np.array(img, dtype=np.float32) * (2 / 255) - 1).permute(2, 0, 1).unsqueeze(0)
    clip = _bf(D._ClipStub().encode_image([x]))
    msk = torch.zeros(1, n_frames, H // 8, W // 8)
    msk[:, 0] = 1
    msk = torch.cat([torch.repeat_interleave(msk[:, 0:1], 4, dim=1), msk[:, 1:]], dim=1)
    msk = msk.view(1, msk.shape[1] // 4, 4, H // 8, W // 8).transpose(1, 2)[0]
    vae_in = torch.cat([x.transpose(0, 1), torch.zeros(3, n_frames - 1, H, W)], dim=1)
    y = torch.cat([msk, V.vae_encode(m["vae"], vae_in.unsqueeze(0))[0]]).unsqueeze(0).to(torch.bfloat16)
    y = (y + U.ref_stem(m["ref"], SU.ref_pose(H, W, seed=11)).to(torch.bfloat16)).float()
    return _bf(D._prompter("p", True)), _bf(D._prompter("n", False)), clip, y


def _frames_close(frames, vid, what):
    got = np.stack([np.array(f) for f in frames]).astype(np.float32)
    ref = ((vid[0].permute(1, 2, 3, 0) + 1) * 127.5).clip(0, 255).numpy().astype(np.uint8).astype(np.float32)
    diff = np.abs(got - ref)
    print(f"{what} parity: mean {diff.mean():.3f} levels, p99 {np.percentile(diff, 99):.1f}")
    assert diff.mean() < 2.0 and np.percentile(diff, 99) < 12


def test_short_clip_matches_oracle():
    from diffsynth import WanUniAnimateVideoPipeline
    from oracle import dwpose_oracle as DO
    from oracle import unianimate_oracle as U
    from oracle import wan_vae_oracle as V
    nf = 9
    pipe, m = _pipe(WanUniAnimateVideoPipeline)
    img, pose = _image(), SU.pose_video(nf, H, W, seed=10)
    frames = pipe(prompt="p", negative_prompt="n", input_image=img, seed=42, height=H, width=W, num_frames=nf,
                  num_inference_steps=STEPS, tiled=False, progress_bar_cmd=lambda x: x, dwpose_data=pose,
                  random_ref_dwpose=SU.ref_pose(H, W, seed=11))
    noise = _bf(torch.randn(1, 16, (nf - 1) // 4 + 1, H // 8, W // 8, generator=torch.Generator().manual_seed(42)))
    with torch.no_grad():
        pos, neg, clip, y = _oracle_conditioning(m, img, nf)
        lat = U.short_loop(m["dit"], m["cfg"], noise, pos, neg, clip, y, _bf(DO.pose_condition(m["pose"], pose)), STEPS)
        _frames_close(frames, V.vae_decode(m["vae"], lat), "UniAnimate clip")


def _long_call(pipe, img, pose, seed):
    return pipe(prompt="p", negative_prompt="n", input_image=img, seed=seed, height=H, width=W, num_frames=33,
                num_inference_steps=STEPS, tiled=False, progress_bar_cmd=lambda x: x, dwpose_data=pose,
                random_ref_dwpose=SU.ref_pose(H, W, seed=11), context_size=5, context_overlap=2)


def test_long_video_matches_oracle_and_repeats(monkeypatch):
    """9 latent frames in windows of 5 overlapping by 2: starts 0, 3 and 4 (the last window realigned)."""
    from diffsynth import WanUniAnimateLongVideoPipeline
    from oracle import dwpose_oracle as DO
    from oracle import unianimate_oracle as U
    from oracle import wan_vae_oracle as V
    pipe, m = _pipe(WanUniAnimateLongVideoPipeline)
    img, pose = _image(), SU.pose_video(33, H, W, seed=10)
    draws = []
    orig = torch.randn_like

    def rec(t, *a, **k):
        r = orig(t, *a, **k)
        draws.append(r.clone())
        return r
    monkeypatch.setattr(torch, "randn_like", rec)
    torch.cuda.manual_seed(3)
    frames = _long_call(pipe, img, pose, seed=42)
    assert len(draws) == 3 and all(d.is_cuda and d.dtype == torch.bfloat16 for d in draws)
    torch.cuda.manual_seed(3)
    again = _long_call(pipe, img, pose, seed=42)
    assert all(np.array_equal(np.array(a), np.array(b)) for a, b in zip(frames, again)), "same seed, different bytes"
    wins = U.windows(9, 5, 2)
    assert [w[0] for w in wins] == [0, 3, 4]
    noise = _bf(torch.randn(1, 16, 9, H // 8, W // 8, generator=torch.Generator().manual_seed(42)))
    with torch.no_grad():
        pos, neg, clip, y = _oracle_conditioning(m, img, 4 * 5 - 3)
        conds = [_bf(DO.pose_condition(m["pose"], pose[:, 4 * w[0]:4 * w[-1] + 1])) for w in wins]
        lat = U.long_loop(m["dit"], m["cfg"], noise, pos, neg, clip, y, conds, wins, [d.float().cpu() for d in draws[:3]], STEPS)
        _frames_close(frames, V.vae_decode(m["vae"], lat), "UniAnimate long video")
