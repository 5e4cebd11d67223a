"""SVIVideoPipeline — one clip of the SVI rolling loop on the H100-native kernels.

Public surface follows the reference (``diffsynth/pipelines/svi_video.py``: ``SVIVideoPipeline`` :140-520,
``model_fn_wan_video`` :74-137) so ``test_svi.py`` can drive it unchanged.  Differences are internal:

* the 50-step CFG/Euler loop keeps fp32 latents on the device, reuses step-invariant conditioning
  (embedded prompts and all cross-attention K/V, ``WanDiTEngine.context_state``) and finishes every step with
  one fused CFG+Euler kernel (reference: 2 sequential forwards + 4 elementwise launches, :392-421);
* nothing is offloaded or copied through the CPU (reference VAE round trip, wan_video_vae.py:761-786).
"""
from typing import Optional

import numpy as np
import torch
from PIL import Image
from tqdm import tqdm

from .. import _native as nv
from ..models.wan_video_dit import WanModel
from ..schedulers.flow_match import FlowMatchScheduler
from .base import BasePipeline


class TeaCache:
    """Step skipping of the reference (svi_video.py:23-72): the relative L1 change of the timestep modulation between
    consecutive steps, passed through a model-specific fitted polynomial, is accumulated; while the sum stays below
    `rel_l1_thresh` the block stack is skipped and the token residual (output - input of the block stack) of the last
    computed step is added instead.  First and last step always compute.  One instance per CFG branch.

    The residual bookkeeping runs on the native kernels (svi_axpby); the decision needs one scalar on the host per
    step, exactly as in the reference (`.cpu().item()`, :52)."""

    # fitted rescaling polynomials, highest power first (numeric constants of the TeaCache release, reference :34-39)
    coefficients_dict = {
        "Wan2.1-T2V-1.3B": [-5.21862437e+04, 9.23041404e+03, -5.28275948e+02, 1.36987616e+01, -4.99875664e-02],
        "Wan2.1-T2V-14B": [-3.03318725e+05, 4.90537029e+04, -2.65530556e+03, 5.87365115e+01, -3.15583525e-01],
        "Wan2.1-I2V-14B-480P": [2.57151496e+05, -3.54229917e+04, 1.40286849e+03, -1.35890334e+01, 1.32517977e-01],
        "Wan2.1-I2V-14B-720P": [8.10705460e+03, 2.13393892e+03, -3.72934672e+02, 1.66203073e+01, -4.17769401e-02],
    }

    def __init__(self, num_inference_steps, rel_l1_thresh, model_id):
        if model_id not in self.coefficients_dict:
            raise ValueError(f"{model_id} is not a supported TeaCache model id. Please choose a valid model id in "
                             f"({', '.join(self.coefficients_dict)}).")
        self.num_inference_steps = num_inference_steps
        self.rel_l1_thresh = rel_l1_thresh
        self.coefficients = self.coefficients_dict[model_id]
        self.step = 0
        self.accumulated_rel_l1_distance = 0
        self.previous_modulated_input = None
        self.previous_hidden_states = None
        self.previous_residual = None
        self.skipped = []                 # step indices that re-used the residual (diagnostics / tests)

    def _rescale(self, v):
        acc = 0.0
        for c in self.coefficients:       # Horner, same polynomial as np.poly1d(coefficients)(v)
            acc = acc * v + c
        return acc

    def check(self, dit, x, t_mod):
        """True when this step may skip the block stack.  x: token stream entering the blocks; t_mod: [6, d] modulation."""
        cur = t_mod.detach().clone()
        if self.step == 0 or self.step == self.num_inference_steps - 1:
            compute = True
            self.accumulated_rel_l1_distance = 0
        else:
            prev = self.previous_modulated_input
            rel = ((cur - prev).abs().mean() / prev.abs().mean()).cpu().item()
            self.accumulated_rel_l1_distance += self._rescale(rel)
            compute = not (self.accumulated_rel_l1_distance < self.rel_l1_thresh)
            if compute:
                self.accumulated_rel_l1_distance = 0
        self.previous_modulated_input = cur
        if not compute:
            self.skipped.append(self.step)
        self.step = (self.step + 1) % self.num_inference_steps
        if compute:
            self.previous_hidden_states = x.clone()
        return not compute

    def store(self, hidden_states):
        """After a computed step: residual = block-stack output - its input."""
        if self.previous_residual is None or self.previous_residual.shape != hidden_states.shape:
            self.previous_residual = torch.empty_like(hidden_states)
        if hidden_states.is_cuda:
            from .. import _native as nv
            nv.axpby(hidden_states, 1.0, self.previous_hidden_states, -1.0, self.previous_residual)
        else:
            torch.sub(hidden_states, self.previous_hidden_states, out=self.previous_residual)
        self.previous_hidden_states = None

    def update(self, hidden_states):
        """Skipped step: hidden_states += residual (in place; also returned, as the reference returns the sum)."""
        if hidden_states.is_cuda:
            from .. import _native as nv
            nv.axpby(hidden_states, 1.0, self.previous_residual, 1.0, hidden_states)
        else:
            hidden_states.add_(self.previous_residual)
        return hidden_states


def model_fn_wan_video(dit: WanModel, x: torch.Tensor, timestep: torch.Tensor, context, clip_feature: Optional[torch.Tensor] = None,
                       y: Optional[torch.Tensor] = None, tea_cache=None, add_condition=None,
                       use_unified_sequence_parallel: bool = False, **kwargs):
    """Drop-in for reference svi_video.py:74-137: one DiT forward, result in x.dtype.  `context` may also be
    a ContextState (pre-projected conditioning)."""
    sp = None
    if use_unified_sequence_parallel:
        from ..distributed.sequence_parallel import get_sp_group
        sp = get_sp_group()
    eng = dit.engine(x.device if x.is_cuda else None)
    out = eng.forward(x, timestep, context, clip_feature, y, sp=sp, tea_cache=tea_cache, add_condition=add_condition)
    return out.to(x.dtype)


class SVIVideoPipeline(BasePipeline):
    OTHER_RANK = object()      # stands for the ContextState of a CFG branch that another rank group computes (denoise_step)

    def __init__(self, device="cuda", torch_dtype=torch.float16, tokenizer_path=None, is_test=False, num_train_timesteps=1000):
        super().__init__(device=device, torch_dtype=torch_dtype)
        self.scheduler = FlowMatchScheduler(shift=5, sigma_min=0.0, extra_one_step=True, num_train_timesteps=num_train_timesteps)
        self.prompter = None          # WanPrompter once a text encoder is loaded; any callable(prompt, positive=bool) ->
        self.text_encoder = None      # [1,512,4096] works too (precomputed embeddings)
        self.image_encoder = None     # WanImageEncoder (or any object with encode_image([f32 1x3xHxW]) -> [1,257,1280])
        self.dit: WanModel = None
        self.vae = None
        self.model_names = ["text_encoder", "dit", "vae"]
        self.height_division_factor = 16
        self.width_division_factor = 16
        self.use_unified_sequence_parallel = False
        self.is_test = is_test

    # ------------------------------------------------------------------ construction
    def enable_vram_management(self, num_persistent_param_in_dit=None):
        """Reference svi_video.py:156-241 wraps every Linear for CPU offload under a 6e9-parameter budget.  On an
        80 GB H100 the whole 14B model (32 GB bf16) plus umT5-XXL, CLIP and the VAE are resident: the all-resident
        policy.  The reference harness builds its ModelManager on the CPU (test_svi.py:316-318), so every model the
        pipeline holds is moved here (and in fetch_models): the engines exist for CUDA devices only."""
        for name in ("dit", "vae", "text_encoder", "image_encoder"):
            m = getattr(self, name, None)
            if isinstance(m, torch.nn.Module):
                m.to(self.device)
                m.vram_management_enabled = False

    def fetch_models(self, model_manager):
        self.dit = model_manager.fetch_model("wan_video_dit")
        self.vae = model_manager.fetch_model("wan_video_vae")
        te = model_manager.fetch_model("wan_video_text_encoder", require_model_path=True)
        if te is not None:        # reference :246-249: the tokenizer lives next to the T5 checkpoint
            import os
            from ..prompters import WanPrompter
            self.text_encoder, te_path = te
            self.prompter = WanPrompter()
            self.prompter.fetch_models(self.text_encoder)
            tok_dir = os.path.join(os.path.dirname(str(te_path)), "google/umt5-xxl")
            if os.path.isdir(tok_dir):
                self.prompter.fetch_tokenizer(tok_dir)
        self.image_encoder = model_manager.fetch_model("wan_video_image_encoder")
        for name in ("dit", "vae", "text_encoder", "image_encoder"):       # a CPU-resident ModelManager is the reference flow
            m = getattr(self, name, None)
            if isinstance(m, torch.nn.Module) and torch.device(self.device).type == "cuda":
                m.to(self.device).eval()

    @staticmethod
    def from_model_manager(model_manager, torch_dtype=None, device=None, use_usp=False, is_test=False, num_train_timesteps=1000):
        device = model_manager.device if device is None else device
        torch_dtype = model_manager.torch_dtype if torch_dtype is None else torch_dtype
        pipe = SVIVideoPipeline(device=device, torch_dtype=torch_dtype, is_test=is_test, num_train_timesteps=num_train_timesteps)
        pipe.fetch_models(model_manager)
        if use_usp:
            pipe.enable_usp()
        return pipe

    def enable_usp(self):
        """`use_usp=True` (reference :265-273 patches in xfuser USP): install the native multi-GPU plan — the two guidance branches
        on two halves of the ranks x token-axis sequence parallelism inside a branch for the denoise loop, row bands over ALL
        ranks with a halo exchange per convolution for the VAE.  Shared by every pipeline of this package."""
        from ..distributed.sequence_parallel import get_sp_group
        self.sp_size = get_sp_group().world
        self.use_unified_sequence_parallel = True
        if self.vae is not None and hasattr(self.vae, "enable_spatial_sharding"):
            self.vae.enable_spatial_sharding()

    def sp_group(self):
        """The multi-GPU plan of this pipeline (None on one GPU)."""
        if not self.use_unified_sequence_parallel:
            return None
        from ..distributed.sequence_parallel import get_sp_group
        return get_sp_group()

    def denoising_model(self):
        return self.dit

    def prepare_unified_sequence_parallel(self):
        return {"use_unified_sequence_parallel": self.use_unified_sequence_parallel}

    def prepare_extra_input(self, latents=None):
        return {}

    # ------------------------------------------------------------------ conditioning
    def encode_prompt(self, prompt, positive=True):
        if self.prompter is None:
            raise RuntimeError("svi_b200: no prompt encoder attached: load a wan_video_text_encoder checkpoint through the "
                               "ModelManager or set pipe.prompter = callable(prompt, positive) -> [1,512,4096].")
        emb = self.prompter(prompt, positive=positive)
        return {"context": emb.to(self.device)}

    def encode_images_adaptive(self, first_frames, random_ref_frame, num_frames, height, width, use_first_aug=False,
                               ref_pad_cfg=False, ref_pad_num=None):
        """reference svi_video.py:291-364: CLIP feature of the first frame, the 4-channel first-frame mask and
        the VAE latents of [condition frames ++ padding]; everything in fp32 then cast to the pipeline dtype."""
        dev = self.device
        def prep(im):
            x = self._device_frame(im, width, height)           # recycled motion frames are already on the device
            return x if x is not None else self.preprocess_image(im.resize((width, height))).to(device=dev, dtype=torch.float32)
        ref = prep(random_ref_frame)
        first = prep(first_frames[0])
        clip_context = self.image_encoder.encode_image([first])
        msk = torch.ones(1, num_frames, height // 8, width // 8, device=dev, dtype=torch.float32)
        msk[:, (len(first_frames) if ref_pad_cfg else 1):] = 0
        msk = torch.concat([torch.repeat_interleave(msk[:, 0:1], repeats=4, dim=1), msk[:, 1:]], dim=1)
        msk = msk.view(1, msk.shape[1] // 4, 4, height // 8, width // 8).transpose(1, 2)[0]
        if len(first_frames) > 1:
            cond = torch.cat([prep(fr) for fr in first_frames], dim=0).permute(1, 0, 2, 3)
        else:
            cond = first.transpose(0, 1)
        remaining = num_frames - len(first_frames)
        if ref_pad_num == 0:
            pad = torch.zeros(3, remaining, height, width, device=dev, dtype=torch.float32)
        elif ref_pad_num == -1:
            pad = ref.transpose(0, 1).repeat(1, remaining, 1, 1)
        elif ref_pad_num is not None and ref_pad_num > 0:
            pads = [ref.transpose(0, 1)] * ref_pad_num
            if remaining > ref_pad_num:
                pads += [torch.zeros(3, 1, height, width, device=dev, dtype=torch.float32)] * (remaining - ref_pad_num)
            pad = torch.cat(pads, dim=1)
        else:
            raise ValueError(f"ref_pad_num must be -1, 0 or positive (got {ref_pad_num})")
        vae_input = torch.concat([cond, pad], dim=1)
        y = self.vae.encode([vae_input], device=dev)[0]
        y = torch.concat([msk, y.to(torch.float32)]).unsqueeze(0)
        return {"clip_feature": clip_context.to(dtype=self.torch_dtype, device=dev), "y": y.to(dtype=self.torch_dtype, device=dev)}

    def tensor2video(self, frames):
        """reference :366-370: [C,T,H,W] in [-1,1] -> list of uint8 PIL frames.  On the device the conversion is one native
        kernel and ONE byte per sample crosses to the host (reference: the fp32 video, 4 bytes); the uint8 frames also stay
        on the device (`_frames_u8`, keyed by the identity of the PIL frames handed out) so that the frames a caller feeds
        back as the next clip's `input_image` (test_svi.py:472) are conditioned on without a host round trip."""
        if frames.is_cuda and frames.shape[0] == 3:
            v = frames.to(torch.float32).contiguous()
            u8 = torch.empty(v.shape[1], v.shape[2], v.shape[3], 3, device=v.device, dtype=torch.uint8)
            nv.frames_to_uint8(v, u8)
            host = u8.cpu().numpy()
            out = [Image.fromarray(f) for f in host]
            self._frames_u8 = {id(im): (im, u8, t) for t, im in enumerate(out)}     # previous clip's entries are dropped here
            return out
        fr = ((frames.float().permute(1, 2, 3, 0) + 1) * 127.5).clip(0, 255).cpu().numpy().astype(np.uint8)
        return [Image.fromarray(f) for f in fr]

    def _device_frame(self, im, width, height):
        """f32 [1,3,H,W] in [-1,1] on the device for a PIL frame this pipeline produced itself (same arithmetic as
        preprocess_image), or None."""
        hit = getattr(self, "_frames_u8", {}).get(id(im))
        if hit is None or hit[0] is not im or im.size != (width, height):
            return None
        _, u8, t = hit
        return (u8[t].to(torch.float32) * (2 / 255) - 1).permute(2, 0, 1).unsqueeze(0)

    def encode_video(self, input_video, tiled=True, tile_size=(34, 34), tile_stride=(18, 16)):
        lat = self.vae.encode(input_video.to(device=self.device, dtype=torch.float32), device=self.device, tiled=tiled,
                              tile_size=tile_size, tile_stride=tile_stride)
        return lat.to(device=self.device, dtype=self.torch_dtype)

    def decode_video(self, latents, tiled=True, tile_size=(34, 34), tile_stride=(18, 16)):
        return self.vae.decode(latents.to(device=self.device, dtype=torch.float32), device=self.device, tiled=tiled,
                               tile_size=tile_size, tile_stride=tile_stride)

    # ------------------------------------------------------------------ denoising
    def denoise_step(self, eng, lat, t, sigma, sigma_next, cp, cn, v_c, v_u, cfg_scale, y=None, sp=None, tea=(None, None),
                     add_condition=(None, None)):
        """ONE flow-matching step of the hot loop (reference :404-420: two forwards, CFG combine, scheduler.step) on the
        device-resident f32 latents `lat` (updated in place).  cp / cn: ContextState of the conditional / unconditional
        prompt (cn None: no guidance).  sp: the multi-GPU plan — with two CFG groups every rank runs ONE branch on its
        token rows and the branches' velocity fields are joined once per step (SequenceParallelGroup.cfg_parallel_step)."""
        if sp is not None and cn is not None:
            return sp.cfg_parallel_step(eng, lat, t, cp, cn, v_c, v_u, cfg_scale, sigma, sigma_next, y=y, tea=tea,
                                        add_condition=add_condition)
        inner = sp if sp is not None and sp.sp_size > 1 else None
        eng.forward(lat, t, cp, y=y, sp=inner, out=v_c, tea_cache=tea[0], add_condition=add_condition[0])
        if cn is not None:
            eng.forward(lat, t, cn, y=y, sp=inner, out=v_u, tea_cache=tea[1], add_condition=add_condition[1])
        eng.k.cfg_euler_step(lat, v_c, v_u if cn is not None else None, cfg_scale, sigma, sigma_next)
        return lat

    def denoise_latents(self, latents, context_posi, context_nega, clip_feature=None, y=None, cfg_scale=5.0,
                        progress_bar_cmd=lambda x: x, sp=None, tea_cache_posi=None, tea_cache_nega=None,
                        add_condition_posi=None, add_condition_nega=None):
        """The hot loop (reference _sample_with_regular_video :392-421).  latents: f32 [1,16,f,h,w] on device,
        updated in place and returned.  Timesteps/sigmas come from self.scheduler (already set)."""
        eng = self.dit.engine(self.device)
        lat = latents
        if lat.dtype != torch.float32 or not lat.is_contiguous():
            lat = lat.to(torch.float32).contiguous()
        if y is not None:
            y = y.to(device=self.device, dtype=torch.float32).contiguous()
        use_cfg = cfg_scale != 1.0
        both = sp is None or not use_cfg          # a CFG-parallel rank projects only its own branch's prompt
        cp = eng.context_state(context_posi, clip_feature) if both or sp.owns_branch(0) else None
        cn = (eng.context_state(context_nega, clip_feature) if both or sp.owns_branch(1) else self.OTHER_RANK) if use_cfg else None
        v_c = torch.empty_like(lat)
        v_u = torch.empty_like(lat) if use_cfg else None
        sig = self.scheduler.sigmas
        ts = self.scheduler.timesteps
        n = len(ts)
        for i in progress_bar_cmd(range(n)):
            nxt = float(sig[i + 1]) if i + 1 < n else 0.0
            self.denoise_step(eng, lat, float(ts[i]), float(sig[i]), nxt, cp, cn, v_c, v_u, cfg_scale, y=y, sp=sp,
                              tea=(tea_cache_posi, tea_cache_nega), add_condition=(add_condition_posi, add_condition_nega))
        return lat

    def _sample_with_regular_video(self, latents, prompt_emb_posi, prompt_emb_nega, image_emb, extra_input, tea_cache_posi,
                                   tea_cache_nega, usp_kwargs, use_controlnet, cfg_scale, progress_bar_cmd):
        sp = self.sp_group() if usp_kwargs.get("use_unified_sequence_parallel") else None
        scale = cfg_scale["text"] if isinstance(cfg_scale, dict) else cfg_scale
        bar = (lambda r: progress_bar_cmd(r)) if progress_bar_cmd is not None else (lambda r: r)
        return self.denoise_latents(latents, prompt_emb_posi["context"], prompt_emb_nega["context"],
                                    image_emb.get("clip_feature"), image_emb.get("y"), scale, bar, sp,
                                    tea_cache_posi.get("tea_cache"), tea_cache_nega.get("tea_cache"))

    @torch.no_grad()
    def __call__(self, prompt, negative_prompt="", input_image=None, input_video=None, denoising_strength=1.0, seed=None,
                 rand_device="cpu", height=480, width=832, num_frames=81, cfg_scale=5.0, num_inference_steps=50,
                 sigma_shift=5.0, tiled=True, tile_size=(30, 52), tile_stride=(15, 26), tea_cache_l1_thresh=None,
                 tea_cache_model_id="", progress_bar_cmd=tqdm, random_ref_frame=None, use_controlnet=False, args=None,
                 last_latent=None):
        height, width = self.check_resize_height_width(height, width)
        if num_frames % 4 != 1:
            num_frames = (num_frames + 2) // 4 * 4 + 1
            print(f"Only `num_frames % 4 != 1` is acceptable. We round it up to {num_frames}.")
        tiler_kwargs = {"tiled": tiled, "tile_size": tile_size, "tile_stride": tile_stride}
        self.scheduler.set_timesteps(num_inference_steps, denoising_strength=denoising_strength, shift=sigma_shift)
        noise = self.generate_noise((1, 16, (num_frames - 1) // 4 + 1, height // 8, width // 8), seed=seed,
                                    device=rand_device, dtype=torch.float32)
        # the reference rounds the initial noise to the pipeline dtype (svi_video.py:465); keep that rounding so
        # identical seeds start from identical latents, then carry fp32 through the loop
        latents = noise.to(dtype=self.torch_dtype, device=self.device).to(torch.float32)
        if input_video is not None:
            vid = torch.stack(self.preprocess_images(input_video), dim=2).to(dtype=torch.float32, device=self.device)
            lat0 = self.encode_video(vid, **tiler_kwargs).to(torch.float32)
            latents = self.scheduler.add_noise(lat0, latents, timestep=self.scheduler.timesteps[0])
        prompt_emb_posi = self.encode_prompt(prompt, positive=True)
        prompt_emb_nega = self.encode_prompt(negative_prompt, positive=False)
        if input_image is not None and self.image_encoder is not None:
            ref_img = Image.fromarray(random_ref_frame.clone().cpu().numpy())
            if not isinstance(input_image, list):
                input_image = [input_image]
            image_emb = self.encode_images_adaptive(input_image, ref_img, num_frames, height, width, use_first_aug=False,
                                                    ref_pad_cfg=args.ref_pad_cfg, ref_pad_num=args.ref_pad_num)
            if last_latent:
                image_emb["y"][:, 0, ...] = last_latent
        else:
            image_emb = {}
        scale = cfg_scale
        usp_kwargs = self.prepare_unified_sequence_parallel()
        mk = lambda: {"tea_cache": TeaCache(num_inference_steps, rel_l1_thresh=tea_cache_l1_thresh, model_id=tea_cache_model_id)
                      if tea_cache_l1_thresh is not None else None}
        latents = self._sample_with_regular_video(latents, prompt_emb_posi, prompt_emb_nega, image_emb, {}, mk(), mk(),
                                                  usp_kwargs, use_controlnet, scale, progress_bar_cmd)
        frames = self.decode_video(latents, **tiler_kwargs)
        frames = self.tensor2video(frames[0])
        if hasattr(args, "sequential_cfg") and args.sequential_cfg == "latent":
            return frames, latents[:, -1, ...]
        return frames
