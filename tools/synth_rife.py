"""Seeded RIFE (IFNet) weights and structured test frames.

Default initialisation gives an almost trivial network (flows below a pixel, mask logits with an std of ~3e-3), which
would leave the warps and the blend untested.  So the final layer of each block's flow head is scaled until flows reach
several pixels (some of them pointing off the image) and that of the mask head until the mask logits have an std of
about 1.  The frames are a smooth texture and a shifted, rotated copy of it, so the flows have something to find.
"""
import numpy as np
import torch
from PIL import Image

FLOW_GAIN = 24.0
MASK_GAIN = 80.0


def _block_shapes(in_planes, c=90):
    s = {}
    for i, (ci, co) in enumerate([(in_planes, c // 2), (c // 2, c)]):
        s[f"conv0.{i}.0.weight"] = (co, ci, 3, 3)
        s[f"conv0.{i}.0.bias"] = (co,)
        s[f"conv0.{i}.1.weight"] = (co,)
    for r in range(4):
        for j in range(2):
            s[f"convblock{r}.{j}.0.weight"] = (c, c, 3, 3)
            s[f"convblock{r}.{j}.0.bias"] = (c,)
            s[f"convblock{r}.{j}.1.weight"] = (c,)
    for head, out in (("conv1", 4), ("conv2", 1)):
        s[f"{head}.0.weight"] = (c, c // 2, 4, 4)
        s[f"{head}.0.bias"] = (c // 2,)
        s[f"{head}.1.weight"] = (c // 2,)
        s[f"{head}.2.weight"] = (c // 2, out, 4, 4)
        s[f"{head}.2.bias"] = (out,)
    return s


def param_shapes():
    """IFNet's 160 parameter tensors: block0..2 (11 input channels) and block_tea (14)."""
    out = {}
    for name, cin in (("block0", 11), ("block1", 11), ("block2", 11), ("block_tea", 14)):
        out.update({f"{name}.{k}": v for k, v in _block_shapes(cin).items()})
    return out


def make_state_dict(seed=0, prefix=""):
    """f32 weights: PyTorch's default conv init (uniform, bound 1 / sqrt(fan_in)), PReLU slopes 0.25 +- 0.1, and the
    flow / mask heads' last layers scaled by FLOW_GAIN / MASK_GAIN.  prefix="module." gives the checkpoint's key names."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in param_shapes().items():
        if name.endswith(".1.weight") and len(shape) == 1:                  # PReLU
            t = 0.25 + 0.1 * (2 * torch.rand(shape, generator=g) - 1)
        else:
            bound = (shape[1] * shape[2] * shape[3] if len(shape) == 4 else 90 * 9) ** -0.5
            t = bound * (2 * torch.rand(shape, generator=g) - 1)
            if ".conv1.2." in name:
                t = t * FLOW_GAIN
            elif ".conv2.2." in name:
                t = t * MASK_GAIN
        sd[prefix + name] = t.float()
    return sd


def make_frames(n, H, W, seed=0, shift=(3.0, -2.0), angle=1.5):
    """n uint8 RGB PIL frames: a smooth random texture, each next frame shifted by `shift` pixels and rotated by
    `angle` degrees about the centre relative to the previous one."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    comps = [(rng.uniform(0.02, 0.12, 2), rng.uniform(0, 2 * np.pi), rng.uniform(0.2, 0.5, 3)) for _ in range(6)]
    cy, cx = (H - 1) / 2, (W - 1) / 2

    def texture(y, x):
        img = np.full((H, W, 3), 0.5)
        for (fy, fx), ph, amp in comps:
            v = np.sin(fy * y + fx * x + ph)
            img += 0.25 * amp * v[..., None]
        return img

    frames = []
    for k in range(n):
        a = np.deg2rad(angle * k)
        y0, x0 = yy - cy - shift[1] * k, xx - cx - shift[0] * k
        y = cy + np.cos(a) * y0 - np.sin(a) * x0
        x = cx + np.sin(a) * y0 + np.cos(a) * x0
        frames.append(Image.fromarray((np.clip(texture(y, x), 0, 1) * 255).astype(np.uint8)))
    return frames


def weight_checksum(sd):
    """sum over tensors (sorted by name) of sum(w) + 1e-3 * sum(w^2), in fp64"""
    return float(sum(v.double().sum() + 1e-3 * (v.double() ** 2).sum() for _, v in sorted(sd.items())))
