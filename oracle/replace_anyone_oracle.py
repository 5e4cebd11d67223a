"""CPU oracle of the UniAnimate-DiT Replace-Anyone pipeline — TEST INFRASTRUCTURE ONLY (never imported by the product
path).

Restates in fp32 what reference diffsynth/pipelines/wan_video.py computes for ``WanRepalceAnyoneVideoPipeline``
(:1207-1584): the mask (:1546, :1550-1551), the learn-in stem on the masked video and its keep mask with the first frame
repeated three more times in front (:1353-1361, :1554), the inpaint stem on the VAE latents of the masked video
(:1363-1369, :1555), and the denoising loop whose conditional forward sees latents + both stem outputs and the pose tokens
while the unconditional forward sees the plain latents (:1562-1575), on ``wan_dit_oracle``.  The loop takes its
conditioning and the offset as inputs.  Pinned to the reference by tests/golden/replace_anyone_tiny.npz.
"""
import torch
import torch.nn.functional as F

from oracle import wan_dit_oracle as O

LEARN_IN_STRIDES = ((1, 1, 1), (1, 2, 2), (2, 2, 2), (2, 2, 2))
INPAINT_STRIDES = ((1, 1, 1),) * 3


def keep_mask(segmentation_data):
    """segmentation_data [1, T, H, W] (any real dtype) -> float [1, T, H, W]: 1 where seg / 255 is not > 0."""
    return (~(segmentation_data / 255. > 0)).float()


def masked_video(video, segmentation_data):
    """The VAE encoder's input: video [3, T, H, W] * keep, f32."""
    return video.float() * keep_mask(segmentation_data)


def learn_in_input(video, segmentation_data):
    """[1, 4, T + 3, H, W] f32: (masked video, keep) with the first frame in front three more times."""
    m = torch.cat([masked_video(video, segmentation_data), keep_mask(segmentation_data)], dim=0)
    return torch.cat([m[:, :1]] * 3 + [m], dim=1).unsqueeze(0)


def _stem(sd, x, strides):
    for i, s in enumerate(strides):
        x = F.conv3d(x, sd[f"{2 * i}.weight"].float(), sd[f"{2 * i}.bias"].float(), stride=s, padding=1)
        if i < len(strides) - 1:
            x = F.silu(x)
    return x


def learn_in(sd, x):
    """sd: keys '0.weight' ... '6.bias'; x [1, 4, T', H, W] -> [1, 16, f, H/8, W/8]."""
    return _stem(sd, x.float(), LEARN_IN_STRIDES)


def inpaint(sd, x):
    """sd: keys '0.weight' ... '4.bias'; x [1, 16, f, h, w] -> [1, 16, f, h, w]."""
    return _stem(sd, x.float(), INPAINT_STRIDES)


def offset(learn_in_sd, inpaint_sd, video, segmentation_data, latents_masked):
    """What the conditional branch adds to the latents: both stems on bf16 inputs, outputs rounded to bf16 (the
    reference runs both stems in bf16), summed in f32."""
    bf = lambda t: t.to(torch.bfloat16).float()
    a = bf(learn_in(learn_in_sd, bf(learn_in_input(video, segmentation_data))))
    b = bf(inpaint(inpaint_sd, bf(latents_masked)))
    return a + b


def replace_loop(sd, cfg, latents, offset, ctx_pos, ctx_neg, clip, y, condition, steps, cfg_scale=5.0, shift=5.0):
    """:1562-1575: the conditional forward on latents + offset with the pose tokens, the unconditional one on the
    latents without them."""
    sig = O.flow_match_sigmas(steps, shift)
    x = latents.float()
    for i in range(steps):
        ts = (sig[i] * 1000).reshape(1)
        v = O.dit_forward(sd, cfg, x + offset, ts, ctx_pos, clip, y, add_condition=condition)
        if cfg_scale != 1.0:
            v = O.cfg_combine(v, O.dit_forward(sd, cfg, x, ts, ctx_neg, clip, y), cfg_scale)
        x = O.flow_match_step(sig, i, v, x)
    return x
