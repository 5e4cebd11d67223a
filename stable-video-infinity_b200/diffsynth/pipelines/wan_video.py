"""The Wan pipelines of reference diffsynth/pipelines/wan_video.py.

* ``WanVideoPipeline`` (:25-286), the plain T2V/I2V surface.  Same hot loop as SVIVideoPipeline (shared
  implementation); differences follow the reference: scalar ``cfg_scale`` and ``encode_image`` (single first frame, zero
  padding) instead of ``encode_images_adaptive``.
* ``WanUniAnimateVideoPipeline`` (:411-757), UniAnimate-DiT pose animation of one clip: a pose video through the
  ``dwpose_embedding`` stem conditions the conditional branch in token space, a reference-pose image through the
  ``randomref_embedding_pose`` stem is added to the image condition ``y``.
* ``WanUniAnimateLongVideoPipeline`` (:762-1202), the same model over a video longer than one clip: every step denoises
  overlapping windows of ``context_size`` latent frames and averages them per frame (``svi_window_accumulate`` /
  ``svi_window_normalize``).

* ``WanRepalceAnyoneVideoPipeline`` (:1207-1584, also exported as ``WanReplaceAnyoneVideoPipeline``), UniAnimate-DiT
  Replace-Anyone: re-animates the person masked out of ``batch["video"]`` by ``batch["segmentation_data"]`` (the
  ``batch`` keyword of its ``__call__``, :1488) with the identity of ``input_image`` and the pose of ``dwpose_data``.
"""
import numpy as np
import torch
from tqdm import tqdm

from .. import _native as nv
from ..models.dwpose_embedding import (DWPoseEmbeddingEngine, InpaintEmbeddingEngine, LearnInEmbeddingEngine,
                                       RandomRefEmbeddingEngine, make_dwpose_embedding, make_inpaint_embedding,
                                       make_learn_in_embedding, make_randomref_embedding_pose, pose_condition)
from .svi_video import SVIVideoPipeline, TeaCache, model_fn_wan_video  # noqa: F401  (re-exported like the reference)


class WanVideoPipeline(SVIVideoPipeline):
    @staticmethod
    def from_model_manager(model_manager, torch_dtype=None, device=None, use_usp=False):
        device = model_manager.device if device is None else device
        torch_dtype = model_manager.torch_dtype if torch_dtype is None else torch_dtype
        pipe = WanVideoPipeline(device=device, torch_dtype=torch_dtype)
        pipe.fetch_models(model_manager)
        if use_usp:
            pipe.enable_usp()
        return pipe

    def encode_image(self, image, num_frames, height, width):
        """reference wan_video.py:157-172: mask of the first frame + VAE latents of [image, zeros...]."""
        dev = self.device
        im = self.preprocess_image(image.resize((width, height))).to(device=dev, dtype=torch.float32)
        clip_context = self.image_encoder.encode_image([im])
        msk = torch.ones(1, num_frames, height // 8, width // 8, device=dev)
        msk[:, 1:] = 0
        msk = torch.concat([torch.repeat_interleave(msk[:, 0:1], repeats=4, dim=1), msk[:, 1:]], dim=1)
        msk = msk.view(1, msk.shape[1] // 4, 4, height // 8, width // 8).transpose(1, 2)[0]
        vae_input = torch.concat([im.transpose(0, 1), torch.zeros(3, num_frames - 1, height, width, device=dev)], dim=1)
        y = self.vae.encode([vae_input], device=dev)[0]
        y = torch.concat([msk, y.to(torch.float32)]).unsqueeze(0)
        return {"clip_feature": clip_context.to(self.torch_dtype), "y": y.to(self.torch_dtype)}

    @torch.no_grad()
    def __call__(self, prompt, negative_prompt="", input_image=None, input_video=None, denoising_strength=1.0, seed=None,
                 rand_device="cpu", height=480, width=832, num_frames=81, cfg_scale=5.0, num_inference_steps=50,
                 sigma_shift=5.0, tiled=True, tile_size=(30, 52), tile_stride=(15, 26), tea_cache_l1_thresh=None,
                 tea_cache_model_id="", progress_bar_cmd=tqdm, progress_bar_st=None):
        height, width = self.check_resize_height_width(height, width)
        if num_frames % 4 != 1:
            num_frames = (num_frames + 2) // 4 * 4 + 1
            print(f"Only `num_frames % 4 != 1` is acceptable. We round it up to {num_frames}.")
        tiler_kwargs = {"tiled": tiled, "tile_size": tile_size, "tile_stride": tile_stride}
        self.scheduler.set_timesteps(num_inference_steps, denoising_strength=denoising_strength, shift=sigma_shift)
        noise = self.generate_noise((1, 16, (num_frames - 1) // 4 + 1, height // 8, width // 8), seed=seed,
                                    device=rand_device, dtype=torch.float32)
        latents = noise.to(dtype=self.torch_dtype, device=self.device).to(torch.float32)
        if input_video is not None:
            vid = torch.stack(self.preprocess_images(input_video), dim=2).to(dtype=torch.float32, device=self.device)
            latents = self.scheduler.add_noise(self.encode_video(vid, **tiler_kwargs).to(torch.float32), latents,
                                               timestep=self.scheduler.timesteps[0])
        pos = self.encode_prompt(prompt, positive=True)
        neg = self.encode_prompt(negative_prompt, positive=False) if cfg_scale != 1.0 else pos
        image_emb = {}
        if input_image is not None and self.image_encoder is not None:
            image_emb = self.encode_image(input_image, num_frames, height, width)
        bar = (lambda r: progress_bar_cmd(r)) if progress_bar_cmd is not None else (lambda r: r)
        from .svi_video import TeaCache
        mk = lambda: (TeaCache(num_inference_steps, rel_l1_thresh=tea_cache_l1_thresh, model_id=tea_cache_model_id)
                      if tea_cache_l1_thresh is not None else None)     # reference wan_video.py:261-262
        latents = self.denoise_latents(latents, pos["context"], neg["context"], image_emb.get("clip_feature"),
                                       image_emb.get("y"), cfg_scale, bar, self.sp_group(), tea_cache_posi=mk(),
                                       tea_cache_nega=mk())
        frames = self.decode_video(latents, **tiler_kwargs)
        return self.tensor2video(frames[0])


def _stem_keys(state_dict_new_module, tag):
    """The keys of one extra module with everything up to `tag` removed ('pipe.dwpose_embedding.0.weight' -> '0.weight')."""
    return {k.split(tag)[1]: v for k, v in state_dict_new_module.items() if tag in k}


class WanUniAnimateVideoPipeline(WanVideoPipeline):
    """UniAnimate-DiT on one clip (reference wan_video.py:411-757)."""

    def __init__(self, device="cuda", torch_dtype=torch.float16, tokenizer_path=None):
        super().__init__(device=device, torch_dtype=torch_dtype, tokenizer_path=tokenizer_path)
        self.dwpose_embedding = None
        self.randomref_embedding_pose = None
        self._pose_engine = None
        self._ref_engine = None

    def fetch_models(self, model_manager):
        super().fetch_models(model_manager)
        self.load_pose_stems(model_manager.state_dict_new_module)

    def load_pose_stems(self, state_dict_new_module):
        """Build both stems from the extra-module keys load_lora_v2 keeps (`...dwpose_embedding.N.*`,
        `...randomref_embedding_pose.N.*`; strict, like the reference :559-570).  A stem whose keys are absent stays
        None.  The pose stem's output width is the checkpoint's (the reference hard-codes 5120, :541)."""
        sd = _stem_keys(state_dict_new_module, "dwpose_embedding.")
        if sd:
            self.dwpose_embedding = make_dwpose_embedding(dim=sd["12.weight"].shape[0])
            self.dwpose_embedding.load_state_dict(sd, strict=True)
            self._pose_engine = None
        sd = _stem_keys(state_dict_new_module, "randomref_embedding_pose.")
        if sd:
            self.randomref_embedding_pose = make_randomref_embedding_pose(randomref_dim=sd["10.weight"].shape[0])
            self.randomref_embedding_pose.load_state_dict(sd, strict=True)
            self._ref_engine = None

    @staticmethod
    def from_model_manager(model_manager, torch_dtype=None, device=None, use_usp=False):
        device = model_manager.device if device is None else device
        torch_dtype = model_manager.torch_dtype if torch_dtype is None else torch_dtype
        pipe = WanUniAnimateVideoPipeline(device=device, torch_dtype=torch_dtype)
        pipe.fetch_models(model_manager)
        if use_usp:
            pipe.enable_usp()
        return pipe

    def encode_pose(self, dwpose_data):
        """dwpose_data [3, T, H, W] in 0..255 -> tokens f32 [1, L, dim], rounded to bf16 as the reference does (:731)."""
        if self.dwpose_embedding is None:
            raise RuntimeError("svi_b200: no pose stem loaded (dwpose_embedding.* keys of the UniAnimate-DiT checkpoint)")
        if self._pose_engine is None:
            self._pose_engine = DWPoseEmbeddingEngine(self.dwpose_embedding, self.device)
        return pose_condition(self._pose_engine, dwpose_data).to(torch.bfloat16).to(torch.float32)

    def encode_ref_pose(self, random_ref_dwpose):
        """random_ref_dwpose [H, W, 3] in 0..255 -> bf16 [1, 20, 1, H/8, W/8] (reference :732)."""
        if self.randomref_embedding_pose is None:
            raise RuntimeError("svi_b200: no reference-pose stem loaded (randomref_embedding_pose.* keys of the "
                               "UniAnimate-DiT checkpoint)")
        if self._ref_engine is None:
            self._ref_engine = RandomRefEmbeddingEngine(self.randomref_embedding_pose, self.device)
        x = random_ref_dwpose.to(device=self.device, dtype=torch.float32).permute(2, 0, 1) / 255.0
        return self._ref_engine.forward(x).to(torch.bfloat16)

    def _check_inputs(self, input_image, dwpose_data, random_ref_dwpose, num_frames, height, width):
        if input_image is None or self.image_encoder is None:
            raise ValueError("UniAnimate needs input_image and an image encoder: the reference-pose term is added to "
                             "the image condition y")
        if dwpose_data is None or random_ref_dwpose is None:
            raise ValueError("UniAnimate needs dwpose_data ([3, num_frames, H, W]) and random_ref_dwpose ([H, W, 3])")
        if tuple(dwpose_data.shape) != (3, num_frames, height, width):
            raise ValueError(f"dwpose_data must be [3, num_frames, height, width] = {(3, num_frames, height, width)} "
                             f"(num_frames after rounding to 4k+1), got {tuple(dwpose_data.shape)}")
        if tuple(random_ref_dwpose.shape) != (height, width, 3):
            raise ValueError(f"random_ref_dwpose must be [height, width, 3] = {(height, width, 3)}, "
                             f"got {tuple(random_ref_dwpose.shape)}")

    def _initial_latents(self, num_frames, height, width, seed, rand_device, input_video, tiler_kwargs):
        noise = self.generate_noise((1, 16, (num_frames - 1) // 4 + 1, height // 8, width // 8), seed=seed,
                                    device=rand_device, dtype=torch.float32)
        latents = noise.to(dtype=self.torch_dtype, device=self.device).to(torch.float32)
        if input_video is not None:
            vid = torch.stack(self.preprocess_images(input_video), dim=2).to(dtype=torch.float32, device=self.device)
            latents = self.scheduler.add_noise(self.encode_video(vid, **tiler_kwargs).to(torch.float32), latents,
                                               timestep=self.scheduler.timesteps[0])
        return latents

    @torch.no_grad()
    def __call__(self, prompt, negative_prompt="", input_image=None, input_video=None, denoising_strength=1.0, seed=None,
                 rand_device="cpu", height=480, width=832, num_frames=81, cfg_scale=5.0, num_inference_steps=50,
                 sigma_shift=5.0, tiled=True, tile_size=(30, 52), tile_stride=(15, 26), tea_cache_l1_thresh=None,
                 tea_cache_model_id="", progress_bar_cmd=tqdm, progress_bar_st=None, dwpose_data=None,
                 random_ref_dwpose=None):
        height, width = self.check_resize_height_width(height, width)
        if num_frames % 4 != 1:
            num_frames = (num_frames + 2) // 4 * 4 + 1
            print(f"Only `num_frames % 4 != 1` is acceptable. We round it up to {num_frames}.")
        self._check_inputs(input_image, dwpose_data, random_ref_dwpose, num_frames, height, width)
        tiler_kwargs = {"tiled": tiled, "tile_size": tile_size, "tile_stride": tile_stride}
        self.scheduler.set_timesteps(num_inference_steps, denoising_strength=denoising_strength, shift=sigma_shift)
        latents = self._initial_latents(num_frames, height, width, seed, rand_device, input_video, tiler_kwargs)
        pos = self.encode_prompt(prompt, positive=True)
        neg = self.encode_prompt(negative_prompt, positive=False) if cfg_scale != 1.0 else pos
        image_emb = self.encode_image(input_image, num_frames, height, width)
        condition = self.encode_pose(dwpose_data)
        y = image_emb["y"] + self.encode_ref_pose(random_ref_dwpose)        # reference :734, in the operands' dtypes
        bar = (lambda r: progress_bar_cmd(r)) if progress_bar_cmd is not None else (lambda r: r)
        mk = lambda: (TeaCache(num_inference_steps, rel_l1_thresh=tea_cache_l1_thresh, model_id=tea_cache_model_id)
                      if tea_cache_l1_thresh is not None else None)
        latents = self.denoise_latents(latents, pos["context"], neg["context"], image_emb["clip_feature"], y, cfg_scale,
                                       bar, self.sp_group(), tea_cache_posi=mk(), tea_cache_nega=mk(),
                                       add_condition_posi=condition, add_condition_nega=None)
        frames = self.decode_video(latents, **tiler_kwargs)
        return self.tensor2video(frames[0])


def ordered_halving(val):
    """Bit-reversed fraction of `val` (reference wan_video.py:762-767)."""
    return int(f"{val:064b}"[::-1], 2) / (1 << 64)


def context_scheduler(step=..., num_steps=None, num_frames=..., context_size=None, context_stride=3, context_overlap=4,
                      closed_loop=False):
    """Windows of `context_size` frame indices (reference wan_video.py:769-797, same results)."""
    if num_frames <= context_size:
        yield list(range(num_frames))
        return
    context_stride = min(context_stride, int(np.ceil(np.log2(num_frames / context_size))) + 1)
    for context_step in 1 << np.arange(context_stride):
        pad = int(round(num_frames * ordered_halving(step)))
        for j in range(int(ordered_halving(step) * context_step) + pad,
                       num_frames + pad + (0 if closed_loop else -context_overlap),
                       (context_size * context_step - context_overlap)):
            yield [e % num_frames for e in range(j, j + context_size * context_step, context_step)]


def context_windows(num_frames, context_size, context_overlap):
    """The long pipeline's window list (reference :1070-1097): the schedule at step 0 with stride 1, the last window
    moved to end at the last frame."""
    queue = list(context_scheduler(0, 31, num_frames, context_size=context_size, context_stride=1,
                                   context_overlap=context_overlap))
    step = min(1, int(np.ceil(np.log2(num_frames / context_size))) + 1)
    queue[-1] = [e % num_frames for e in range(num_frames - context_size * step, num_frames, step)]
    return queue


def window_counts(windows, num_frames):
    """How many windows add to each frame: window 0 all of its frames, every later window all but its first two."""
    counts = [0] * num_frames
    for i, w in enumerate(windows):
        for f in (w if i == 0 else w[2:]):
            counts[f] += 1
    return counts


class WanUniAnimateLongVideoPipeline(WanUniAnimateVideoPipeline):
    """UniAnimate-DiT over a video longer than one clip, in overlapping sliding windows (reference wan_video.py:800-1202).

    Per step and window w (start s_w): gather latents s_w .. s_w+cs-1 with the first two frames replaced by the window's
    carried state, the conditional forward with the window's pose tokens and the unconditional one without, one fused
    CFG + Euler step (svi_cfg_euler_step), the stepped frames 0..1 become the new carry, and the stepped window is added
    into an f32 per-frame sum (svi_window_accumulate).  After the last window every frame is sum / count
    (svi_window_normalize).  Latents, sum and division are f32; the reference keeps them in the pipeline dtype."""

    @staticmethod
    def from_model_manager(model_manager, torch_dtype=None, device=None):
        device = model_manager.device if device is None else device
        torch_dtype = model_manager.torch_dtype if torch_dtype is None else torch_dtype
        pipe = WanUniAnimateLongVideoPipeline(device=device, torch_dtype=torch_dtype)
        pipe.fetch_models(model_manager)
        return pipe

    @torch.no_grad()
    def __call__(self, prompt, negative_prompt="", input_image=None, input_video=None, denoising_strength=1.0, seed=None,
                 rand_device="cpu", height=480, width=832, num_frames=81, cfg_scale=5.0, num_inference_steps=50,
                 sigma_shift=5.0, tiled=True, tile_size=(30, 52), tile_stride=(15, 26), tea_cache_l1_thresh=None,
                 tea_cache_model_id="", progress_bar_cmd=tqdm, progress_bar_st=None, dwpose_data=None,
                 random_ref_dwpose=None, context_size=21, context_overlap=4):
        height, width = self.check_resize_height_width(height, width)
        if num_frames % 4 != 1:
            num_frames = (num_frames - 1) // 4 * 4 + 1           # rounds down, as the reference does (:1045-1047)
            print(f"Only `num_frames % 4 != 1` is acceptable. We round it down to {num_frames}.")
        cs = context_size
        n_lat = (num_frames - 1) // 4 + 1
        if context_overlap < 2:
            raise ValueError(f"context_overlap must be at least 2 (got {context_overlap}): every window after the first "
                             "skips its first two frames, so a smaller overlap leaves frames no window adds to")
        if context_overlap >= cs:
            raise ValueError(f"context_overlap ({context_overlap}) must be smaller than context_size ({cs})")
        if n_lat < cs:
            raise ValueError(f"num_frames = {num_frames} gives {n_lat} latent frames, fewer than context_size = {cs}: "
                             f"the windows would wrap around the video")
        self._check_inputs(input_image, dwpose_data, random_ref_dwpose, num_frames, height, width)
        tiler_kwargs = {"tiled": tiled, "tile_size": tile_size, "tile_stride": tile_stride}
        self.scheduler.set_timesteps(num_inference_steps, denoising_strength=denoising_strength, shift=sigma_shift)
        latents = self._initial_latents(num_frames, height, width, seed, rand_device, input_video, tiler_kwargs)
        windows = context_windows(n_lat, cs, context_overlap)
        starts = [w[0] for w in windows]
        counts = window_counts(windows, n_lat)
        pos = self.encode_prompt(prompt, positive=True)
        neg = self.encode_prompt(negative_prompt, positive=False) if cfg_scale != 1.0 else None
        image_emb = self.encode_image(input_image, 4 * cs - 3, height, width)
        mk = lambda: (TeaCache(num_inference_steps, rel_l1_thresh=tea_cache_l1_thresh, model_id=tea_cache_model_id)
                      if tea_cache_l1_thresh is not None else None)
        tea = [(mk(), mk()) for _ in windows]
        conditions = [self.encode_pose(dwpose_data[:, 4 * s:4 * (s + cs - 1) + 1]) for s in starts]
        # the carries' initial noise: one draw per window in window order, in the pipeline dtype on its device (:1139)
        lat_dt = latents.to(self.torch_dtype)
        carries = [torch.randn_like(lat_dt[:, :, s:s + 2]).to(torch.float32) for s in starts]
        y = image_emb["y"] + self.encode_ref_pose(random_ref_dwpose)
        bar = (lambda r: progress_bar_cmd(r)) if progress_bar_cmd is not None else (lambda r: r)
        latents = self.denoise_windows(latents, pos["context"], None if neg is None else neg["context"],
                                       image_emb["clip_feature"], y, cfg_scale, starts, cs, counts, conditions, carries,
                                       tea, bar)
        frames = self.decode_video(latents, **tiler_kwargs)
        return self.tensor2video(frames[0])

    def denoise_windows(self, latents, context_posi, context_nega, clip_feature, y, cfg_scale, starts, cs, counts,
                        conditions, carries, tea, progress_bar_cmd=lambda x: x):
        """The sliding-window loop (reference :1146-1192).  latents f32 [1, 16, F, h, w]; starts: first frame of each
        window; counts: windows adding to each frame; conditions / carries / tea: per window (carries f32
        [1, 16, 2, h, w], updated in place).  Returns the denoised f32 latents."""
        eng = self.dit.engine(self.device)
        dev = self.device
        lat = latents.to(device=dev, dtype=torch.float32).contiguous()
        y = y.to(device=dev, dtype=torch.float32).contiguous()
        cp = eng.context_state(context_posi, clip_feature)
        cn = eng.context_state(context_nega, clip_feature) if cfg_scale != 1.0 else None
        _, C, _, h, w = lat.shape
        win = torch.empty(1, C, cs, h, w, device=dev, dtype=torch.float32)
        v_c = torch.empty_like(win)
        v_u = torch.empty_like(win) if cn is not None else None
        acc = torch.empty_like(lat)
        count = torch.tensor(counts, dtype=torch.int32).to(dev)
        sig = self.scheduler.sigmas
        ts = self.scheduler.timesteps
        n = len(ts)
        for i in progress_bar_cmd(range(n)):
            nxt = float(sig[i + 1]) if i + 1 < n else 0.0
            nv.zero_(acc)
            for k, s in enumerate(starts):
                win.copy_(lat[:, :, s:s + cs])
                win[:, :, :2].copy_(carries[k])
                self.denoise_step(eng, win, float(ts[i]), float(sig[i]), nxt, cp, cn, v_c, v_u, cfg_scale, y=y,
                                  tea=tea[k], add_condition=(conditions[k], None))
                carries[k].copy_(win[:, :, :2])
                nv.window_accumulate(win, 0 if k == 0 else 2, acc, s)
            nv.window_normalize(acc, count, lat)
        return lat


class WanRepalceAnyoneVideoPipeline(WanUniAnimateVideoPipeline):
    """UniAnimate-DiT Replace-Anyone (reference wan_video.py:1207-1584; the class name keeps the reference's spelling,
    ``WanReplaceAnyoneVideoPipeline`` is the same class).

    ``batch = {"video": [3, num_frames, height, width] float in [-1, 1], "segmentation_data": [1, num_frames, height,
    width] uint8 or float, > 0 on the person to replace}``.  Once per call the video with the person cut out,
    ``video * keep`` with ``keep = !(segmentation_data / 255 > 0)``, goes through the VAE encoder and the inpaint stem, and
    together with ``keep`` through the learn-in stem (svi_replace_mask_stage stages both); the sum of the two results,
    each rounded to bf16 as the reference does, is the offset of the conditional branch.  Every step the conditional
    forward sees latents + offset and the pose tokens, the unconditional forward the plain latents and no pose tokens.
    That asymmetry is the reference's (:1566, :1569).  Latents, the offset and latents + offset are f32; the reference
    keeps them in the pipeline dtype."""

    def __init__(self, device="cuda", torch_dtype=torch.float16, tokenizer_path=None):
        super().__init__(device=device, torch_dtype=torch_dtype, tokenizer_path=tokenizer_path)
        self.learn_in_embedding = None
        self.inpaint_embedding = None
        self._learn_in_engine = None
        self._inpaint_engine = None

    def fetch_models(self, model_manager):
        super().fetch_models(model_manager)
        self.load_replace_stems(model_manager.state_dict_new_module)

    def load_replace_stems(self, state_dict_new_module):
        """Build the learn-in and inpaint stems from the extra-module keys load_lora_v2 keeps (`...learn_in_embedding.N.*`,
        `...inpaint_embedding.N.*`; strict, like the reference :1384-1395).  A stem whose keys are absent stays None."""
        sd = _stem_keys(state_dict_new_module, "learn_in_embedding.")
        if sd:
            self.learn_in_embedding = make_learn_in_embedding()
            self.learn_in_embedding.load_state_dict(sd, strict=True)
            self._learn_in_engine = None
        sd = _stem_keys(state_dict_new_module, "inpaint_embedding.")
        if sd:
            self.inpaint_embedding = make_inpaint_embedding()
            self.inpaint_embedding.load_state_dict(sd, strict=True)
            self._inpaint_engine = None

    @staticmethod
    def from_model_manager(model_manager, torch_dtype=None, device=None):
        device = model_manager.device if device is None else device
        torch_dtype = model_manager.torch_dtype if torch_dtype is None else torch_dtype
        pipe = WanRepalceAnyoneVideoPipeline(device=device, torch_dtype=torch_dtype)
        pipe.fetch_models(model_manager)
        return pipe

    @staticmethod
    def _check_batch(batch, num_frames, height, width):
        if batch is None or "video" not in batch or "segmentation_data" not in batch:
            raise ValueError('Replace-Anyone needs batch={"video": [3, num_frames, height, width], '
                             '"segmentation_data": [1, num_frames, height, width]}')
        video, seg = batch["video"], batch["segmentation_data"]
        if not torch.is_tensor(video) or tuple(video.shape) != (3, num_frames, height, width):
            raise ValueError(f'batch["video"] must be a tensor [3, num_frames, height, width] = '
                             f'{(3, num_frames, height, width)} (num_frames after rounding to 4k+1, height and width '
                             f'after rounding to multiples of 16), got {tuple(getattr(video, "shape", ()))}')
        if not torch.is_tensor(seg) or tuple(seg.shape) != (1, num_frames, height, width):
            raise ValueError(f'batch["segmentation_data"] must be a tensor [1, num_frames, height, width] = '
                             f'{(1, num_frames, height, width)}, got {tuple(getattr(seg, "shape", ()))}')
        return video, seg

    def encode_masked_video(self, video, segmentation_data, tiler_kwargs):
        """video [3, T, H, W], segmentation_data [1, T, H, W] -> the conditional branch's offset, f32 [1, 16, f, h, w]:
        bf16(learn_in_embedding(...)) + bf16(inpaint_embedding(VAE(video * keep))) (reference :1545-1555)."""
        if self.learn_in_embedding is None or self.inpaint_embedding is None:
            raise RuntimeError("svi_b200: no learn-in or inpaint stem loaded (learn_in_embedding.* and inpaint_embedding.* "
                               "keys of the UniAnimate-DiT Replace-Anyone checkpoint)")
        if self._learn_in_engine is None:
            self._learn_in_engine = LearnInEmbeddingEngine(self.learn_in_embedding, self.device)
        if self._inpaint_engine is None:
            self._inpaint_engine = InpaintEmbeddingEngine(self.inpaint_embedding, self.device)
        dev = self.device
        video = video.to(device=dev, dtype=torch.float32).contiguous()
        seg = segmentation_data[0].to(dev)
        if seg.dtype not in (torch.uint8, torch.float32):
            seg = seg.to(torch.float32)
        masked = torch.empty_like(video)
        learn_in = self._learn_in_engine.forward(video, seg.contiguous(), masked)
        lat_masked = self.encode_video(masked.unsqueeze(0), **tiler_kwargs).to(torch.float32)
        inpaint = self._inpaint_engine.forward(lat_masked)
        return nv.axpby(learn_in.to(torch.bfloat16).to(torch.float32), 1.0,
                        inpaint.to(torch.bfloat16).to(torch.float32), 1.0, learn_in)

    @torch.no_grad()
    def __call__(self, prompt, negative_prompt="", input_image=None, input_video=None, denoising_strength=1.0, seed=None,
                 rand_device="cpu", height=480, width=832, num_frames=81, cfg_scale=5.0, num_inference_steps=50,
                 sigma_shift=5.0, tiled=True, tile_size=(30, 52), tile_stride=(15, 26), tea_cache_l1_thresh=None,
                 tea_cache_model_id="", progress_bar_cmd=tqdm, progress_bar_st=None, dwpose_data=None,
                 random_ref_dwpose=None, batch=None):
        height, width = self.check_resize_height_width(height, width)
        if num_frames % 4 != 1:
            num_frames = (num_frames + 2) // 4 * 4 + 1
            print(f"Only `num_frames % 4 != 1` is acceptable. We round it up to {num_frames}.")
        self._check_inputs(input_image, dwpose_data, random_ref_dwpose, num_frames, height, width)
        video, seg = self._check_batch(batch, num_frames, height, width)
        tiler_kwargs = {"tiled": tiled, "tile_size": tile_size, "tile_stride": tile_stride}
        self.scheduler.set_timesteps(num_inference_steps, denoising_strength=denoising_strength, shift=sigma_shift)
        latents = self._initial_latents(num_frames, height, width, seed, rand_device, input_video, tiler_kwargs)
        pos = self.encode_prompt(prompt, positive=True)
        neg = self.encode_prompt(negative_prompt, positive=False) if cfg_scale != 1.0 else None
        image_emb = self.encode_image(input_image, num_frames, height, width)
        condition = self.encode_pose(dwpose_data)
        y = image_emb["y"] + self.encode_ref_pose(random_ref_dwpose)
        offset = self.encode_masked_video(video, seg, tiler_kwargs)
        bar = (lambda r: progress_bar_cmd(r)) if progress_bar_cmd is not None else (lambda r: r)
        mk = lambda: (TeaCache(num_inference_steps, rel_l1_thresh=tea_cache_l1_thresh, model_id=tea_cache_model_id)
                      if tea_cache_l1_thresh is not None else None)
        latents = self.denoise_replace(latents, offset, pos["context"], None if neg is None else neg["context"],
                                       image_emb["clip_feature"], y, cfg_scale, condition, (mk(), mk()), bar)
        frames = self.decode_video(latents, **tiler_kwargs)
        return self.tensor2video(frames[0])

    def denoise_replace(self, latents, offset, context_posi, context_nega, clip_feature, y, cfg_scale, condition,
                        tea=(None, None), progress_bar_cmd=lambda x: x):
        """The loop of :1562-1575.  latents f32 [1, 16, f, h, w]; offset f32 of the same shape.  Per step: x_c = latents +
        offset (svi_axpby), the conditional forward on x_c with the pose tokens, the unconditional forward on the
        latents without them, one fused CFG + Euler step on the latents.  Returns the denoised f32 latents."""
        eng = self.dit.engine(self.device)
        dev = self.device
        lat = latents.to(device=dev, dtype=torch.float32).contiguous()
        offset = offset.to(device=dev, dtype=torch.float32).contiguous()
        y = y.to(device=dev, dtype=torch.float32).contiguous()
        cp = eng.context_state(context_posi, clip_feature)
        cn = eng.context_state(context_nega, clip_feature) if cfg_scale != 1.0 else None
        x_c = torch.empty_like(lat)
        v_c = torch.empty_like(lat)
        v_u = torch.empty_like(lat) if cn is not None else None
        sig = self.scheduler.sigmas
        ts = self.scheduler.timesteps
        n = len(ts)
        for i in progress_bar_cmd(range(n)):
            nxt = float(sig[i + 1]) if i + 1 < n else 0.0
            eng.k.axpby(lat, 1.0, offset, 1.0, x_c)
            eng.forward(x_c, float(ts[i]), cp, y=y, out=v_c, tea_cache=tea[0], add_condition=condition)
            if cn is not None:
                eng.forward(lat, float(ts[i]), cn, y=y, out=v_u, tea_cache=tea[1])
            eng.k.cfg_euler_step(lat, v_c, v_u, cfg_scale, float(sig[i]), nxt)
        return lat


WanReplaceAnyoneVideoPipeline = WanRepalceAnyoneVideoPipeline
