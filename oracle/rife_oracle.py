"""CPU fp32 restatement of RIFE's IFNet and of RIFEInterpolater / RIFESmoother (reference
diffsynth/extensions/RIFE/__init__.py), in plain functional torch.  Line numbers cite that file.

`rnd` (optional) is applied where the native engine stores bf16: every convolution's input and weight.  With
rnd = bf16 rounding the oracle predicts the error the engine's storage precision causes (the rounding study in DESIGN).
"""
import numpy as np
import torch
import torch.nn.functional as F


def _ident(t):
    return t


def warp(img, flow):
    """:8-23: grid_sample(bilinear, border, align_corners=True) at linspace(-1, 1) + flow / ((size - 1) / 2)."""
    N, _, H, W = flow.shape
    gx = torch.linspace(-1.0, 1.0, W, device=flow.device).view(1, 1, 1, W).expand(N, -1, H, -1)
    gy = torch.linspace(-1.0, 1.0, H, device=flow.device).view(1, 1, H, 1).expand(N, -1, -1, W)
    f = torch.cat([flow[:, 0:1] / ((img.shape[3] - 1.0) / 2.0), flow[:, 1:2] / ((img.shape[2] - 1.0) / 2.0)], 1)
    g = (torch.cat([gx, gy], 1) + f).permute(0, 2, 3, 1)
    return F.grid_sample(img, g, mode="bilinear", padding_mode="border", align_corners=True)


def _interp(x, factor):
    return F.interpolate(x, scale_factor=factor, mode="bilinear", align_corners=False, recompute_scale_factor=False)


def block(sd, pre, x, flow, s, rnd=_ident):
    """IFBlock.forward (:43-57) with the parameters under `pre` (e.g. "block0.")."""
    def conv(t, name, stride=1):
        y = F.conv2d(rnd(t), rnd(sd[pre + name + ".0.weight"]), sd[pre + name + ".0.bias"], stride=stride, padding=1)
        return F.prelu(y, sd[pre + name + ".1.weight"])

    x = _interp(x, 1.0 / s)
    flow = _interp(flow, 1.0 / s) * (1.0 / s)
    feat = conv(conv(torch.cat((x, flow), 1), "conv0.0", 2), "conv0.1", 2)
    for r in range(4):
        feat = conv(conv(feat, f"convblock{r}.0"), f"convblock{r}.1") + feat

    def head(name):
        y = F.conv_transpose2d(rnd(feat), rnd(sd[pre + name + ".0.weight"]), sd[pre + name + ".0.bias"], stride=2, padding=1)
        y = F.prelu(y, sd[pre + name + ".1.weight"])
        return F.conv_transpose2d(rnd(y), rnd(sd[pre + name + ".2.weight"]), sd[pre + name + ".2.bias"], stride=2, padding=1)

    f, m = head("conv1"), head("conv2")
    return _interp(f, s) * s, _interp(m, s)


def ifnet(sd, x, scale_list=(4, 2, 1), rnd=_ident):
    """IFNet.forward (:68-96): x f32 [N, 6, H, W] -> (flow_list, sigmoid(mask), merged list)."""
    img0, img1 = x[:, :3], x[:, 3:6]
    flow = x[:, :4] * 0
    mask = x[:, :1] * 0
    w0, w1 = img0, img1
    flows, masks, merged = [], [], []
    for i in range(3):
        pre = f"block{i}."
        f0, m0 = block(sd, pre, torch.cat((w0[:, :3], w1[:, :3], mask), 1), flow, scale_list[i], rnd)
        f1, m1 = block(sd, pre, torch.cat((w1[:, :3], w0[:, :3], -mask), 1), torch.cat((flow[:, 2:4], flow[:, :2]), 1),
                       scale_list[i], rnd)
        flow = flow + (f0 + torch.cat((f1[:, 2:4], f1[:, :2]), 1)) / 2
        mask = mask + (m0 + (-m1)) / 2
        masks.append(mask)
        flows.append(flow)
        w0, w1 = warp(img0, flow[:, :2]), warp(img1, flow[:, 2:4])
        merged.append((w0, w1))
    out = []
    for i in range(3):
        sg = torch.sigmoid(masks[i])
        out.append(merged[i][0] * sg + merged[i][1] * (1 - sg))
    return flows, torch.sigmoid(masks[2]), out


def to_tensor(frames):
    """uint8 RGB [F, H, W, 3] -> f32 [F, 3, H, W] BGR / 255 (process_image, :130-137, for sides that are multiples of 32)."""
    a = np.asarray(frames, dtype=np.float32)[..., [2, 1, 0]] / 255
    return torch.from_numpy(a).permute(0, 3, 1, 2)


def to_uint8(t):
    """decode_images (:139-142): f32 [F, 3, H, W] BGR -> uint8 RGB [F, H, W, 3], truncating."""
    return (t[:, [2, 1, 0]].permute(0, 2, 3, 1) * 255).clip(0, 255).numpy().astype(np.uint8)


def _batched(sd, inp, scale, batch_size, rnd):
    outs = [ifnet(sd, inp[b:b + batch_size], [4 / scale, 2 / scale, 1 / scale], rnd)[2][2]
            for b in range(0, inp.shape[0], batch_size)]
    return torch.cat(outs, 0)


def interpolate(sd, frames, scale=1.0, batch_size=4, num_iter=1, rnd=_ident):
    """RIFEInterpolater.interpolate (:167-194) on uint8 RGB frames [F, H, W, 3] -> uint8 [2^num_iter (F - 1) + 1, H, W, 3]."""
    x = to_tensor(frames)
    for _ in range(num_iter):
        out = _batched(sd, torch.cat((x[:-1], x[1:]), 1), scale, batch_size, rnd).clip(0, 1)
        y = torch.empty(2 * x.shape[0] - 1, *x.shape[1:])
        y[0::2], y[1::2] = x, out
        x = y
    return to_uint8(x)


def smooth(sd, frames, scale=1.0, batch_size=4, num_iter=1, rnd=_ident):
    """RIFESmoother.__call__ (:218-239): every inner frame becomes IFNet(frame, IFNet(prev, next))."""
    x = to_tensor(frames)
    for _ in range(num_iter):
        mid = _batched(sd, torch.cat((x[:-2], x[2:]), 1), scale, batch_size, rnd)
        x[1:-1] = _batched(sd, torch.cat((x[1:-1], mid), 1), scale, batch_size, rnd)
    return to_uint8(x)
