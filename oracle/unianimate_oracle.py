"""CPU oracle of the UniAnimate-DiT pipelines — TEST INFRASTRUCTURE ONLY (never imported by the product path).

Restates in fp32 what reference diffsynth/pipelines/wan_video.py computes for ``WanUniAnimateVideoPipeline`` (:411-757)
and ``WanUniAnimateLongVideoPipeline`` (:762-1202): the reference-pose stem (six Conv2d, :543-558), the context schedule
(:762-797, :1070-1097) and both denoising loops on ``wan_dit_oracle.dit_forward(..., add_condition=...)``.  The pose
tokens come from ``dwpose_oracle.pose_condition``.  The loops take their conditioning (prompt embeddings, CLIP feature,
``y``, pose tokens) and, for the long loop, the carries' initial noise as inputs.  Pinned to the reference by
tests/golden/unianimate_tiny.npz.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import wan_dit_oracle as O

REF_STRIDES = (1, 1, 1, 2, 2, 2)


def ref_stem(sd, image):
    """sd: keys '0.weight' ... '10.bias'; image [H, W, 3] in 0..255 -> f32 [1, 20, 1, H/8, W/8] (:732, before bf16)."""
    x = (image.float().unsqueeze(0) / 255.0).permute(0, 3, 1, 2)
    for i, s in enumerate(REF_STRIDES):
        x = F.conv2d(x, sd[f"{2 * i}.weight"].float(), sd[f"{2 * i}.bias"].float(), stride=s, padding=1)
        if i < len(REF_STRIDES) - 1:
            x = F.silu(x)
    return x.unsqueeze(2)


def ordered_halving(val):
    """:762-767: the bits of val reversed, as a fraction of 2^64."""
    return int(f"{val:064b}"[::-1], 2) / (1 << 64)


def context_scheduler(step, num_frames, context_size, context_stride=3, context_overlap=4, closed_loop=False):
    """:769-797 as a list of windows."""
    if num_frames <= context_size:
        return [list(range(num_frames))]
    out = []
    context_stride = min(context_stride, int(np.ceil(np.log2(num_frames / context_size))) + 1)
    for context_step in 1 << np.arange(context_stride):
        pad = int(round(num_frames * ordered_halving(step)))
        stop = num_frames + pad + (0 if closed_loop else -context_overlap)
        for j in range(int(ordered_halving(step) * context_step) + pad, stop, context_size * context_step - context_overlap):
            out.append([e % num_frames for e in range(j, j + context_size * context_step, context_step)])
    return out


def windows(num_frames, context_size, context_overlap):
    """:1070-1087: step 0, stride 1, the last window realigned to end at the last frame."""
    q = context_scheduler(0, num_frames, context_size, 1, context_overlap)
    step = min(1, int(np.ceil(np.log2(num_frames / context_size))) + 1)
    q[-1] = [e % num_frames for e in range(num_frames - context_size * step, num_frames, step)]
    return q


def short_loop(sd, cfg, latents, ctx_pos, ctx_neg, clip, y, condition, steps, cfg_scale=5.0, shift=5.0):
    """:736-749: the conditional forward with the pose tokens, the unconditional one without."""
    sig = O.flow_match_sigmas(steps, shift)
    x = latents.float()
    for i in range(steps):
        ts = (sig[i] * 1000).reshape(1)
        v = O.dit_forward(sd, cfg, x, ts, ctx_pos, clip, y, add_condition=condition)
        if cfg_scale != 1.0:
            v = O.cfg_combine(v, O.dit_forward(sd, cfg, x, ts, ctx_neg, clip, y), cfg_scale)
        x = O.flow_match_step(sig, i, v, x)
    return x


def long_loop(sd, cfg, latents, ctx_pos, ctx_neg, clip, y, conditions, wins, carries, steps, cfg_scale=5.0, shift=5.0):
    """:1146-1192.  conditions / carries: per window (carries [1, C, 2, h, w], the initial noise of :1139)."""
    sig = O.flow_match_sigmas(steps, shift)
    x = latents.float()
    carries = [c.float() for c in carries]
    for i in range(steps):
        ts = (sig[i] * 1000).reshape(1)
        counter = torch.zeros(1, 1, x.shape[2], 1, 1)
        total = torch.zeros_like(x)
        for k, win in enumerate(wins):
            xin = x[:, :, win].clone()
            xin[:, :, :2] = carries[k]
            v = O.dit_forward(sd, cfg, xin, ts, ctx_pos, clip, y, add_condition=conditions[k])
            if cfg_scale != 1.0:
                v = O.cfg_combine(v, O.dit_forward(sd, cfg, xin, ts, ctx_neg, clip, y), cfg_scale)
            out = O.flow_match_step(sig, i, v, xin)
            keep = win if k == 0 else win[2:]
            counter[:, :, keep] += 1
            total[:, :, keep] += out[:, :, len(win) - len(keep):]
            carries[k] = out[:, :, :2]
        x = total / counter
    return x
