"""GPU: UniAnimate-DiT Replace-Anyone — svi_replace_mask_stage against torch's formula bit for bit, both stems against
the f32 oracle, and one clip through the public pipeline against the same clip computed by the CPU oracles."""
import numpy as np
import pytest
import torch

from tools import synth_replace_anyone as SR, synth_unianimate as SU

pytestmark = pytest.mark.gpu

H, W, STEPS = 32, 48, 3


def _bits(t):
    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int16)


@pytest.mark.parametrize("seg_dtype", [torch.uint8, torch.float32])
@pytest.mark.parametrize("T,h,w", [(3, 5, 7), (9, 48, 80)])
def test_mask_stage_equals_torch(seg_dtype, T, h, w):
    """HW = 35 is not a multiple of any vector width; the video has negative values, -0.0, inf and NaN; the
    segmentation has 0, 1 and 255 (and, in f32, fractions, a negative value and NaN)."""
    from diffsynth import _native as nv
    g = torch.Generator().manual_seed(T * 1000 + h)
    video = torch.rand(3, T, h, w, generator=g) * 2 - 1
    video.view(-1)[:4] = torch.tensor([-0.0, float("nan"), float("inf"), -3.0])
    seg = SR.segmentation(T, h, w, seed=h, dtype=torch.float32).view(T, h, w)
    seg.view(-1)[:3] = torch.tensor([0.0, 1.0, 255.0])
    seg[0, 0, 3:6] = 0                              # the special video values of channel 0 are kept
    if seg_dtype == torch.float32:
        seg.view(-1)[-4:] = torch.tensor([0.25, -1.0, float("nan"), 1e-30])
    vd, sd = video.cuda(), seg.to(seg_dtype).cuda()
    keep = ~(sd / 255. > 0)                         # on the device, where NaN results are the same canonical NaN
    want = (vd * keep).cpu()
    want_ring = torch.cat([want.permute(1, 2, 3, 0), keep.float().cpu().unsqueeze(-1)], dim=-1).to(torch.bfloat16)
    for with_masked in (True, False):
        masked = torch.full_like(vd, 7.0) if with_masked else None
        ring = torch.full((T, h, w, 64), 3.0, device="cuda", dtype=torch.bfloat16)
        nv.replace_mask_stage(vd, sd, masked, ring)
        torch.cuda.synchronize()
        if with_masked:
            assert torch.equal(_bits(masked.cpu()), _bits(want)), "masked video differs from video * ~seg"
        got = ring.cpu()
        finite = ~torch.isnan(want_ring.float())
        assert torch.equal(_bits(got[..., :4])[finite], _bits(want_ring)[finite])
        assert torch.isnan(got[..., :4].float()[~finite]).all()
        assert (got[..., 4:].float() == 3.0).all(), "padding channels were written"
    with pytest.raises(RuntimeError, match="ldr"):
        nv.replace_mask_stage(vd, sd, None, torch.zeros(T, h, w, 6, device="cuda", dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="uint8 or float32"):
        nv.replace_mask_stage(vd, sd.double(), None, torch.zeros(T, h, w, 64, device="cuda", dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="overlap"):
        nv.replace_mask_stage(vd, sd, vd, torch.zeros(T, h, w, 64, device="cuda", dtype=torch.bfloat16))


def _rel(got, want):
    return (got - want).abs().mean().item() / want.std().item()


@pytest.mark.parametrize("T,h,w", [(9, 48, 80), (17, 64, 96)])
def test_learn_in_stem_matches_oracle(T, h, w):
    from diffsynth.models.dwpose_embedding import LearnInEmbeddingEngine, make_learn_in_embedding
    from oracle import replace_anyone_oracle as R
    sd = SR.learn_in_sd(seed=T)
    seq = make_learn_in_embedding()
    seq.load_state_dict(sd)
    video, seg = SR.video(T, h, w, seed=1), SR.segmentation(T, h, w, seed=2)
    masked = torch.empty(3, T, h, w, device="cuda")
    got = LearnInEmbeddingEngine(seq, "cuda").forward(video.cuda(), seg[0].cuda(), masked).cpu()
    want = R.learn_in(sd, R.learn_in_input(video, seg))
    rel = _rel(got, want)
    print(f"learn-in stem T={T} {h}x{w}: mean|err|/std = {100 * rel:.3f} %")
    assert got.shape == want.shape == (1, 16, (T - 1) // 4 + 1, h // 8, w // 8)
    assert rel <= 5e-3
    assert torch.equal(masked.cpu(), R.masked_video(video, seg))


@pytest.mark.parametrize("f,h,w", [(3, 6, 10), (21, 60, 104)])
def test_inpaint_stem_matches_oracle(f, h, w):
    from diffsynth.models.dwpose_embedding import InpaintEmbeddingEngine, make_inpaint_embedding
    from oracle import replace_anyone_oracle as R
    sd = SR.inpaint_sd(seed=f)
    seq = make_inpaint_embedding()
    seq.load_state_dict(sd)
    lat = SR.masked_latents(f, h, w, seed=3)
    got = InpaintEmbeddingEngine(seq, "cuda").forward(lat.cuda()).cpu()
    want = R.inpaint(sd, lat)
    rel = _rel(got, want)
    print(f"inpaint stem f={f} {h}x{w}: mean|err|/std = {100 * rel:.3f} %")
    assert got.shape == want.shape and rel <= 5e-3


def _pipe():
    import test_unianimate_gpu as U
    from diffsynth import WanRepalceAnyoneVideoPipeline
    pipe, m = U._pipe(WanRepalceAnyoneVideoPipeline)
    m["learn_in"], m["inpaint"] = SR.learn_in_sd(seed=20), SR.inpaint_sd(seed=21)
    pipe.load_replace_stems({"pipe.learn_in_embedding." + k: v for k, v in m["learn_in"].items()} |
                            {"pipe.inpaint_embedding." + k: v for k, v in m["inpaint"].items()})
    return pipe, m


def _call(pipe, img, pose, batch, cfg_scale):
    return pipe(prompt="p", negative_prompt="n", input_image=img, seed=42, height=H, width=W, num_frames=9,
                cfg_scale=cfg_scale, num_inference_steps=STEPS, tiled=False, progress_bar_cmd=lambda x: x,
                dwpose_data=pose, random_ref_dwpose=SU.ref_pose(H, W, seed=11), batch=batch)


@pytest.mark.parametrize("cfg_scale", [5.0, 1.0])
def test_clip_matches_oracle_and_repeats(cfg_scale):
    import test_unianimate_gpu as U
    from oracle import dwpose_oracle as DO
    from oracle import replace_anyone_oracle as R
    from oracle import wan_vae_oracle as V
    nf = 9
    pipe, m = _pipe()
    img, pose = U._image(), SU.pose_video(nf, H, W, seed=10)
    video, seg = SR.video(nf, H, W, seed=30), SR.segmentation(nf, H, W, seed=31)
    batch = {"video": video.cuda().to(torch.bfloat16), "segmentation_data": seg}
    frames = _call(pipe, img, pose, batch, cfg_scale)
    again = _call(pipe, img, pose, batch, cfg_scale)
    assert all(np.array_equal(np.array(a), np.array(b)) for a, b in zip(frames, again)), "same seed, different bytes"
    noise = U._bf(torch.randn(1, 16, (nf - 1) // 4 + 1, H // 8, W // 8, generator=torch.Generator().manual_seed(42)))
    vid = video.to(torch.bfloat16).float()
    with torch.no_grad():
        pos, neg, clip, y = U._oracle_conditioning(m, img, nf)
        lat_m = V.vae_encode(m["vae"], R.masked_video(vid, seg).unsqueeze(0))
        off = R.offset(m["learn_in"], m["inpaint"], vid, seg, lat_m)
        lat = R.replace_loop(m["dit"], m["cfg"], noise, off, pos, neg, clip, y, U._bf(DO.pose_condition(m["pose"], pose)),
                             STEPS, cfg_scale)
        U._frames_close(frames, V.vae_decode(m["vae"], lat), f"Replace-Anyone clip (cfg {cfg_scale})")
