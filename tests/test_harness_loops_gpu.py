"""GPU: the multi-clip loops of the SVI-Dance and SVI-Talk scripts (test_svi_dance.py, test_svi_talk.py) through the
public pipelines, with the scripts' own helpers from utils.image_process / utils.video_process, on tiny random-init
models.  Clip 2 of each loop is checked against the CPU oracles fed the SAME recycled motion frame and the same pose
tensor or audio window, so only clip 2's own arithmetic is compared (as in test_pipeline_gpu.py's chain test)."""
import types

import numpy as np
import pytest
import torch
from PIL import Image

from tools import synth, synth_vae

pytestmark = pytest.mark.gpu

H, W, FRAMES, CTX = 64, 96, 9, 24
MOTION = 1                              # --num_motion_frames, the default of both scripts


def _bf(t):
    return t.to(torch.bfloat16).float()


def _prep(im):
    return torch.from_numpy(np.array(im, dtype=np.float32) * (2 / 255) - 1).permute(2, 0, 1).unsqueeze(0)   # [1,3,H,W]


def _models(cfg, dit_seed):
    from diffsynth import ModelManager
    from diffsynth.models.wan_video_dit import WanModel
    from diffsynth.models.wan_video_vae import WanVideoVAE
    dit_sd = {k: _bf(v) for k, v in synth.make_dit_state_dict(cfg, seed=dit_seed).items()}
    vae_sd = {k: _bf(v) for k, v in synth_vae.make_vae_state_dict(seed=0).items()}
    dit = WanModel(**cfg).eval()
    dit.load_state_dict(dit_sd)
    vae = WanVideoVAE().eval()
    vae.load_state_dict(vae_sd)
    mm = ModelManager(torch_dtype=torch.bfloat16, device="cuda")
    mm.add_model("wan_video_dit", dit.to("cuda"))
    mm.add_model("wan_video_vae", vae.to("cuda"))
    return mm, dit_sd, vae_sd


def _oracle_conditioning(vae_sd, ref_img, motion_frame):
    """clip feature and y of a clip conditioned on one motion frame with the reference image repeated
    after it (ref_pad_num=-1) and the mask on the first frame only (ref_pad_cfg=False)."""
    from oracle import wan_vae_oracle as V
    from test_dance_gpu import _ClipStub
    x, f = _prep(ref_img), _prep(motion_frame)
    clip = _bf(_ClipStub().encode_image([f]))
    msk = torch.zeros(1, FRAMES, H // 8, W // 8)
    msk[:, 0] = 1
    msk = torch.cat([torch.repeat_interleave(msk[:, 0:1], 4, dim=1), msk[:, 1:]], dim=1)
    msk = msk.view(1, msk.shape[1] // 4, 4, H // 8, W // 8).transpose(1, 2)[0]
    vae_in = torch.cat([f.transpose(0, 1), x.transpose(0, 1).repeat(1, FRAMES - 1, 1, 1)], dim=1)
    y = _bf(torch.cat([msk, V.vae_encode(vae_sd, vae_in.unsqueeze(0))[0]]).unsqueeze(0))
    return clip, y


def _noise(seed):
    return _bf(torch.randn((1, 16, (FRAMES - 1) // 4 + 1, H // 8, W // 8), generator=torch.Generator().manual_seed(seed)))


def _frames(vid):
    return ((vid[0].permute(1, 2, 3, 0) + 1) * 127.5).clip(0, 255).numpy().astype(np.uint8)


def _grey_error(label, got, want):
    diff = np.abs(np.stack([np.array(f) for f in got]).astype(np.float32) - want.astype(np.float32))
    mean, p99 = diff.mean(), np.percentile(diff, 99)
    print(f"{label}: mean {mean:.3f} levels, p99 {p99:.1f}")
    return mean, p99


def test_dance_script_loop_matches_oracle():
    """test_svi_dance.py's loop: the pose video is fitted to the clip size with resize_and_pad_to_target, repeated when
    shorter than a clip, and clip 2 takes the last motion frame's pose followed by wrapped indices into the pose video.
    H100: clip 2 0.457 grey levels mean, p99 2.0."""
    from diffsynth import SVIDanceVideoPipeline
    from oracle import dwpose_oracle as DO
    from oracle import wan_dit_oracle as O
    from oracle import wan_vae_oracle as V
    from test_dance_gpu import _ClipStub, _prompter, _stem_sd
    from utils.image_process import resize_and_pad_to_target, tensor2pil
    from utils.video_process import image_compose_width
    cfg, steps, scale = synth.CFG_TINY_I2V, 3, {"audio": 1.0, "text": 5.0}
    mm, dit_sd, vae_sd = _models(cfg, dit_seed=2)
    stem_sd = _stem_sd(cfg["dim"], seed=7)
    mm.state_dict_new_module = {"pipe.dwpose_embedding." + k: v for k, v in stem_sd.items()}
    pipe = SVIDanceVideoPipeline.from_model_manager(mm, torch_dtype=torch.bfloat16, device="cuda", is_test=True)
    pipe.prompter = _prompter
    pipe.image_encoder = _ClipStub()
    img = Image.fromarray(np.random.default_rng(5).integers(0, 255, size=(H, W, 3), dtype=np.uint8))
    ref = torch.from_numpy(np.array(img))
    # a 4-frame uint8 pose video at 40 x 50, as the script stacks it from pose.mp4: [N, 3, h, w]
    g = torch.Generator().manual_seed(3)
    pose_video = torch.randint(0, 256, (4, 3, 40, 50), dtype=torch.uint8, generator=g)
    pose_all = resize_and_pad_to_target(pose_video, (H, W), pad_value=0).permute(1, 0, 2, 3)          # [3, N, H, W]
    assert pose_all.dtype == torch.uint8 and pose_all.shape == (3, 4, H, W)
    assert pose_all.shape[1] < FRAMES                                                                   # repeat-padding
    pose_all = torch.cat([pose_all] * (FRAMES // pose_all.shape[1] + 1), dim=1)
    pose = pose_all[:, :FRAMES]
    sampled_idx = FRAMES - 1
    args = types.SimpleNamespace(ref_pad_cfg=False, ref_pad_num=-1, sequential_cfg="none")
    kw = dict(prompt="p", negative_prompt="n", num_inference_steps=steps, cfg_scale=scale, tiled=False,
              random_ref_frame=ref, height=H, width=W, num_frames=FRAMES, use_controlnet=False, cond_wo_pose=True,
              args=args, progress_bar_cmd=lambda x: x)
    cond = img
    for k, seed in enumerate((0, 42)):
        video = pipe(input_image=cond, seed=seed, humanpose_data=pose, **kw)
        assert len(video) == FRAMES
        if k == 1:
            clip, y = _oracle_conditioning(vae_sd, img, cond[0])
            pc = _bf(DO.pose_condition(stem_sd, pose))
            sig, lat = O.flow_match_sigmas(steps, 5.0), _noise(seed)
            with torch.no_grad():
                for i in range(steps):
                    ts = (sig[i] * 1000).reshape(1)
                    vc = O.dit_forward(dit_sd, cfg, lat, ts, _bf(_prompter("p", True)), clip, y, add_condition=pc)
                    vu = O.dit_forward(dit_sd, cfg, lat, ts, _bf(_prompter("n", False)), clip, y, add_condition=pc)
                    lat = O.flow_match_step(sig, i, O.cfg_combine(vc, vu, scale["text"]), lat)
                want = _frames(V.vae_decode(vae_sd, lat))
            mean, p99 = _grey_error("dance loop clip 2 (1 motion frame, recycled pose)", video, want)
            assert mean < 2.0 and p99 < 12
        cond = video[-MOTION:]
        kept = video[:-MOTION] if k == 0 else video
        # the script's side-by-side frame: reference | pose | generated
        for ii in (0, len(kept) - 1):
            pose_im = tensor2pil(pose[:, ii].permute(1, 2, 0).to(torch.uint8))
            out = image_compose_width(image_compose_width(tensor2pil(ref.permute(2, 0, 1)), pose_im), kept[ii])
            want = np.concatenate([np.array(img), pose[:, ii].permute(1, 2, 0).numpy(), np.array(kept[ii])], axis=1)
            assert out.size == (3 * W, H) and np.array_equal(np.array(out), want)
        # clip k+1's pose: the last motion frames' poses, then the pose video from where the clip stopped, wrapped
        new = torch.zeros(3, FRAMES, H, W)
        new[:, :MOTION] = pose[:, -MOTION:]
        for i in range(MOTION, FRAMES):
            sampled_idx = sampled_idx % pose_all.shape[1]
            new[:, i] = pose_all[:, sampled_idx]
            sampled_idx += 1
        if k == 0:
            assert torch.equal(new[:, 0], pose[:, -1].float())
            assert torch.equal(new[:, 1:], pose_all[:, [8, 9, 10, 11, 0, 1, 2, 3]].float())
        pose = new


def test_talk_script_loop_matches_oracle(tmp_path):
    """test_svi_talk.py's loop: clip k's audio windows start at k * 81 - num_motion_frames; clip 2 is run from
    audio_path= (features extracted on the GPU once) and from audio_embed= windows of the same cached features, and is
    checked against the oracle given that window.  The wav2vec2 is base-sized: the talk DiT's audio projection takes
    12 x 768 features.  H100: clip 2 0.458 grey levels mean, p99 2.0; latents 4.7e-3 of the std, 68 % inside."""
    from diffsynth import SVITalkVideoPipeline
    from diffsynth.pipelines.svi_video_talk import preprocess_audio
    from oracle import wan_dit_oracle as O
    from oracle import wan_vae_oracle as V
    from oracle import wav2vec2_oracle as WO
    from test_audio_gpu import _model
    from test_dance_gpu import _ClipStub
    from tools import synth_audio as SA
    cfg, steps, st, sa = synth.CFG_TINY_TALK, 2, 5.0, 4.0
    m, _ = _model(SA.BASE, 4)
    ck = SA.write_checkpoint(str(tmp_path / "chinese-wav2vec2-base"), SA.BASE, m.state_dict())
    wav = SA.write_wav(str(tmp_path / "talk.wav"), SA.make_waveform(4.0, sr=16000, seed=6), 16000, "int16")
    mm, dit_sd, vae_sd = _models(cfg, dit_seed=5)
    pipe = SVITalkVideoPipeline.from_model_manager(mm, torch_dtype=torch.bfloat16, device="cuda", is_test=True, wav2vec_path=ck)
    prompter = lambda prompt, positive=True: torch.randn(1, CTX, cfg["text_dim"], generator=torch.Generator().manual_seed(11 if positive else 12))
    pipe.prompter = prompter
    pipe.image_encoder = _ClipStub()
    img = Image.fromarray(np.random.default_rng(5).integers(0, 255, size=(H, W, 3), dtype=np.uint8))
    feats = pipe.audio_hidden_states(wav).float().cpu()                                   # [T, 12, 768] at 25 fps
    assert feats.shape[0] >= 81 + FRAMES + 1                                             # clip 2's window is inside
    latents = []
    decode = pipe.decode_video
    pipe.decode_video = lambda lat, **kw: (latents.append(lat.float().cpu().clone()), decode(lat, **kw))[1]
    args = types.SimpleNamespace(ref_pad_cfg=False, ref_pad_num=-1, sequential_cfg="none")
    kw = dict(prompt="p", negative_prompt="n", num_inference_steps=steps, cfg_scale={"audio": sa, "text": st}, tiled=False,
              random_ref_frame=torch.from_numpy(np.array(img)), height=H, width=W, num_frames=FRAMES, use_controlnet=False,
              args=args, progress_bar_cmd=lambda x: x)

    def loop(route):
        cond, out = img, []
        for k, seed in enumerate((0, 42)):
            start = k * 81 - MOTION if k > 0 else 0
            audio = dict(audio_path=wav) if route == "path" else dict(audio_embed=WO.windows(feats, FRAMES, start))
            video = pipe(input_image=cond, seed=seed, audio_start_idx=start, **audio, **kw)
            assert len(video) == FRAMES
            out.append((cond, start, video, latents[-1]))
            cond = video[-MOTION:]
        return out

    by_embed = loop("embed")
    by_path = loop("path")
    assert pipe.audio_extractions == 1
    cond, start, video, lat_got = by_embed[1]
    assert start == 81 - MOTION
    for (_, _, a, _), (_, _, b, _) in zip(by_embed, by_path):
        assert all(np.array_equal(np.array(x), np.array(y)) for x, y in zip(a, b)), "audio_path= and audio_embed= differ"
    # clip 2 on the oracle: the same recycled frame, the same window of features (rounded to bf16 as the pipeline does)
    clip, y = _oracle_conditioning(vae_sd, img, cond[0])
    window = WO.windows(feats, FRAMES, start)
    tup = tuple(_bf(t) for t in preprocess_audio(window))
    null = tuple(_bf(t) for t in preprocess_audio(torch.zeros_like(window)))
    cp, cn = _bf(prompter("p", True)), _bf(prompter("n", False))
    sig, lat = O.flow_match_sigmas(steps, 5.0), _noise(42)
    with torch.no_grad():
        for i in range(steps):
            ts = (sig[i] * 1000).reshape(1)
            vc = O.dit_forward(dit_sd, cfg, lat, ts, cp, clip, y, audio_embed_tuple=tup)
            vu = O.dit_forward(dit_sd, cfg, lat, ts, cn, clip, y, audio_embed_tuple=null)
            vd = O.dit_forward(dit_sd, cfg, lat, ts, cn, clip, y, audio_embed_tuple=tup)
            lat = O.flow_match_step(sig, i, vu + st * (vc - vd) + sa * (vd - vu), lat)
        want = _frames(V.vae_decode(vae_sd, lat))
    err = (lat_got - lat).abs()
    inside = (err <= 1e-3 + 1e-2 * lat.abs()).float().mean().item()
    rel = err.mean().item() / lat.std().item()
    print(f"talk loop clip 2 latents (audio_start_idx={start}): inside={inside:.4f} mean/std={rel:.4e}")
    mean, p99 = _grey_error(f"talk loop clip 2 (1 motion frame, audio_start_idx={start})", video, want)
    assert inside > 0.5 and rel < 2e-2
    assert mean < 2.0 and p99 < 12
