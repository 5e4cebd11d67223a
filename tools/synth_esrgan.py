"""Seeded ESRGAN (RRDBNet) weights.

basicsr's initialisation: kaiming-normal (fan_in, gain sqrt(2)) for every conv, scaled by 0.1 in the residual dense
blocks, with small random biases so that every bias path is exercised.  Left at that, the output has an std of about 10
and nearly every uint8 pixel clips to 0 or 255, so byte comparisons would say nothing.  conv_last is therefore rescaled,
from one calibration run of the fp32 oracle, so that the output is about 0.5 +- 0.2 in every channel.  Test frames come
from tools/synth_rife.make_frames (a smooth texture).
"""
import torch

from oracle import esrgan_oracle as O

CALIB_H, CALIB_W = 12, 16
OUT_MEAN, OUT_STD = 0.5, 0.2


def param_shapes(num_block=23, num_feat=64, num_grow_ch=32, num_in_ch=3, num_out_ch=3):
    """RRDBNet's parameters in the reference's module names (702 tensors for the default config)."""
    s = {"conv_first": (num_feat, num_in_ch)}
    for i in range(num_block):
        for r in (1, 2, 3):
            for k in range(1, 6):
                s[f"body.{i}.rdb{r}.conv{k}"] = (num_grow_ch if k < 5 else num_feat, num_feat + (k - 1) * num_grow_ch)
    for name in ("conv_body", "conv_up1", "conv_up2", "conv_hr"):
        s[name] = (num_feat, num_feat)
    s["conv_last"] = (num_out_ch, num_feat)
    out = {}
    for name, (o, i) in s.items():
        out[name + ".weight"] = (o, i, 3, 3)
        out[name + ".bias"] = (o,)
    return out


def make_state_dict(num_block=23, seed=0):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in param_shapes(num_block).items():
        if len(shape) == 4:
            t = torch.randn(shape, generator=g) * (2.0 / (shape[1] * 9)) ** 0.5
            if ".rdb" in name:
                t = t * 0.1
        else:
            t = 0.01 * torch.randn(shape, generator=g)
        sd[name] = t.float()
    calib = torch.rand(1, 3, CALIB_H, CALIB_W, generator=g)
    sd["conv_last.bias"] = torch.zeros(3)
    with torch.no_grad():
        y = O.rrdbnet(sd, calib)
    k = OUT_STD / y.std().item()
    sd["conv_last.weight"] = (sd["conv_last.weight"] * k).float()
    sd["conv_last.bias"] = (OUT_MEAN - k * y.mean(dim=(0, 2, 3))).float()
    return sd


def weight_checksum(sd):
    """sum over tensors (sorted by name) of sum(w) + 1e-3 * sum(w^2), in fp64"""
    return float(sum(v.double().sum() + 1e-3 * (v.double() ** 2).sum() for _, v in sorted(sd.items())))
