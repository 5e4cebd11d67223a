"""CPU fp32 restatement of ESRGAN's RRDBNet and of ESRGAN.upscale (reference diffsynth/extensions/ESRGAN/__init__.py),
in plain functional torch.  Line numbers cite that file.

`rnd` (optional) is applied where the native engine stores bf16: every convolution's input and weight, while the
residual streams and the epilogues stay f32.  With rnd = bf16 rounding the oracle predicts the error the engine's storage
precision causes (the rounding study in DESIGN).  `rnd_first` overrides `rnd` for conv_first's input (the image) alone.
"""
import numpy as np
import torch
import torch.nn.functional as F


def _ident(t):
    return t


def num_blocks(sd):
    return 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("body."))


def rrdbnet(sd, x, rnd=_ident, rnd_first=None):
    """RRDBNet.forward (:56-67): x f32 [N, 3, H, W] -> f32 [N, 3, 4H, 4W]."""
    def conv(t, name, r=rnd):
        return F.conv2d(r(t), rnd(sd[name + ".weight"]), sd[name + ".bias"], padding=1)

    def lrelu(t):
        return F.leaky_relu(t, 0.2)

    def rdb(x, pre):
        # ResidualDenseBlock.forward (:18-24)
        x1 = lrelu(conv(x, pre + "conv1"))
        x2 = lrelu(conv(torch.cat((x, x1), 1), pre + "conv2"))
        x3 = lrelu(conv(torch.cat((x, x1, x2), 1), pre + "conv3"))
        x4 = lrelu(conv(torch.cat((x, x1, x2, x3), 1), pre + "conv4"))
        x5 = conv(torch.cat((x, x1, x2, x3, x4), 1), pre + "conv5")
        return x5 * 0.2 + x

    feat = conv(x, "conv_first", rnd if rnd_first is None else rnd_first)
    body = feat
    for i in range(num_blocks(sd)):
        # RRDB.forward (:35-39)
        out = body
        for r in (1, 2, 3):
            out = rdb(out, f"body.{i}.rdb{r}.")
        body = out * 0.2 + body
    feat = feat + conv(body, "conv_body")
    # repeat(feat, "B C H W -> B C (H 2) (W 2)"): nearest x2
    feat = lrelu(conv(feat.repeat_interleave(2, 2).repeat_interleave(2, 3), "conv_up1"))
    feat = lrelu(conv(feat.repeat_interleave(2, 2).repeat_interleave(2, 3), "conv_up2"))
    return conv(lrelu(conv(feat, "conv_hr")), "conv_last")


def to_tensor(frames):
    """process_image / process_images (:94-101): uint8 RGB [F, H, W, 3] -> f32 [F, 3, H, W] / 255."""
    return torch.from_numpy(np.asarray(frames, dtype=np.float32) / 255).permute(0, 3, 1, 2)


def to_uint8(t):
    """decode_images (:103-106): f32 [F, 3, H, W] -> uint8 [F, H, W, 3] of (x * 255).clip(0, 255), truncated."""
    return (t.permute(0, 2, 3, 1) * 255).clip(0, 255).numpy().astype(np.uint8)


def upscale(sd, frames, batch_size=4, rnd=_ident):
    """ESRGAN.upscale (:109-137) on uint8 RGB frames [F, H, W, 3] -> uint8 [F, 4H, 4W, 3]."""
    x = to_tensor(frames)
    dev = sd["conv_first.weight"].device
    outs = [rrdbnet(sd, x[b:b + batch_size].to(dev), rnd).cpu() for b in range(0, x.shape[0], batch_size)]
    return to_uint8(torch.cat(outs, 0))
