"""Restatement of FastBlend's PatchMatch and fast-mode blending (reference diffsynth/extensions/FastBlend:
patch_match.py, cupy_kernels.py, runners/fast.py, __init__.py), in vectorised torch with the kernels' rounding.
Line numbers cite those files.

Every float operation is one torch op on whole arrays, so each result is rounded on its own (no FMA), in the order the
reference's loops take; a division is by a tensor of the same device (torch's CUDA division by a host scalar multiplies
by the reciprocal).  The same code therefore gives the same bits on the CPU (where tests/golden pins it to the reference)
and on the GPU (where the full-size tests use it, minutes faster).  Levels whose size ratio is not an integer go through
cv2 on the host, as the reference does.

The reference draws from CuPy's unseeded global RNG; here draw k of the stream below replaces its k-th call of
cp.random.randint / cp.random.permutation, counted from the PyramidPatchMatcher's construction.
"""
import functools

import cv2
import numpy as np
import torch

RANDOM_SEARCH_STEPS, RANDOM_SEARCH_RANGE = 3, 4      # patch_match.py:11 (PatchMatcher defaults)


# ------------------------------------------------------------------------------------------------ the random stream
def lowbias32(x):
    x = np.asarray(x, dtype=np.uint32)
    with np.errstate(over="ignore"):                    # uint32 products wrap around, by definition
        x = x ^ (x >> np.uint32(16))
        x = x * np.uint32(0x7feb352d)
        x = x ^ (x >> np.uint32(15))
        x = x * np.uint32(0x846ca68b)
        return x ^ (x >> np.uint32(16))


def stream_u(k, i):
    """u(k, i) = lowbias32(lowbias32(k ^ 0x9e3779b9) ^ i), uint32 with wrap-around"""
    return lowbias32(lowbias32(np.uint32(k) ^ np.uint32(0x9e3779b9)) ^ np.asarray(i, dtype=np.uint32))


def randint(k, lo, hi, size):
    """draw k as cp.random.randint(lo, hi, size): element i (flat C order) is lo + u(k, i) % (hi - lo)"""
    n = int(np.prod(size))
    u = stream_u(k, np.arange(n, dtype=np.uint32)) % np.uint32(hi - lo)
    return (lo + u.astype(np.int64)).reshape(size)


def permutation4(k):
    """draw k as cp.random.permutation(4): j = u(k, 0) % 24, Lehmer digits (j // 6, (j // 2) % 3, j % 2, 0)"""
    j = int(stream_u(k, 0))
    j %= 24
    rest, out = [0, 1, 2, 3], []
    for digit in (j // 6, (j // 2) % 3, j % 2, 0):
        out.append(rest.pop(digit))
    return out


# ------------------------------------------------------------------------------------------------ resampling
def box_down(x, k):
    """cv2.resize(INTER_AREA) at the integer ratio k of f32 [n, H, W, C]: cv2's resizeAreaFast_ order (row-major over the
    cell, sum += ((a + b) + c) + d per group of four, a scalar tail, then sum * (1 / k^2))."""
    n, H, W, C = x.shape
    h, w = H // k, W // k
    cells = x.reshape(n, h, k, w, k, C)
    taps = [cells[:, :, sy, :, sx] for sy in range(k) for sx in range(k)]
    s = torch.zeros((n, h, w, C), dtype=torch.float32, device=x.device)
    t = 0
    while t <= len(taps) - 4:
        s = s + (((taps[t] + taps[t + 1]) + taps[t + 2]) + taps[t + 3])
        t += 4
    while t < len(taps):
        s = s + taps[t]
        t += 1
    return s * torch.tensor(np.float32(1.0) / np.float32(k * k), device=x.device)


def integer_ratio(H, W, h, w):
    """the ratio k when cv2 takes its integer-ratio path for H x W -> h x w (both sides exact multiples), else None"""
    k = H // h
    return k if h * k == H and w * k == W and W // w == k else None


def resample(x, h, w):
    """patch_match.py:234-242: each frame of f32 [n, H, W, C] to h x w by cv2.resize(INTER_AREA)"""
    n, H, W, C = x.shape
    if (H, W) == (h, w):
        return x
    k = integer_ratio(H, W, h, w)
    if k is not None:
        return box_down(x, k)
    host = x.cpu().numpy()
    out = np.stack([cv2.resize(f, (w, h), interpolation=cv2.INTER_AREA) for f in host]).astype(np.float32)
    return torch.from_numpy(out.reshape(n, h, w, C)).to(x.device)


# ------------------------------------------------------------------------------------------------ fields
def identity_nnf(B, H, W, device):
    """patch_match.py:251-257"""
    y = torch.arange(H, device=device).view(H, 1).expand(H, W)
    x = torch.arange(W, device=device).view(1, W).expand(H, W)
    return torch.stack([y, x], -1).to(torch.int32).unsqueeze(0).expand(B, H, W, 2).contiguous()


def clamp_nnf(nnf, H, W):
    """patch_match.py:89-92"""
    return torch.stack([nnf[..., 0].clamp(0, H - 1), nnf[..., 1].clamp(0, W - 1)], -1)


def upscale_nnf(nnf, H, W):
    """patch_match.py:262-274: repeat x2, x2, times 2; +1 on the row / column of the odd indices below the batch size
    (the list ranges over nnf.shape[0], the batch); cv2 INTER_LINEAR, truncation and clamp when the level is not exactly
    twice the one before (the branch of :269 is an exact copy otherwise)."""
    B, h, w, _ = nnf.shape
    odd = [i for i in range(B) if i & 1]
    if odd and (odd[-1] >= 2 * h or odd[-1] >= 2 * w):
        raise IndexError("batch larger than the upscaled level")             # what :265-266 raise
    up = nnf.repeat_interleave(2, 1).repeat_interleave(2, 2) * 2
    rows = torch.zeros(2 * h, dtype=torch.int32, device=nnf.device)
    cols = torch.zeros(2 * w, dtype=torch.int32, device=nnf.device)
    rows[odd] = 1
    cols[odd] = 1
    up = torch.stack([up[..., 0] + rows.view(1, -1, 1), up[..., 1] + cols.view(1, 1, -1)], -1)
    if (2 * h, 2 * w) != (H, W):
        host = up.cpu().numpy().astype(np.float32)
        host = np.stack([cv2.resize(f, (W, H), interpolation=cv2.INTER_LINEAR) for f in host]).astype(np.int32)
        up = torch.from_numpy(host).to(nnf.device)
    return clamp_nnf(up, H, W).to(torch.int32)


def neighbour_nnf(nnf, d):
    """patch_match.py:100-114 (edge rows / columns take their own entry)"""
    B, H, W, _ = nnf.shape
    if d == 0:
        u = torch.cat([nnf[:, :1], nnf[:, :-1]], 1) + torch.tensor([1, 0], dtype=nnf.dtype, device=nnf.device)
    elif d == 1:
        u = torch.cat([nnf[:, :, :1], nnf[:, :, :-1]], 2) + torch.tensor([0, 1], dtype=nnf.dtype, device=nnf.device)
    elif d == 2:
        u = torch.cat([nnf[:, 1:], nnf[:, -1:]], 1) - torch.tensor([1, 0], dtype=nnf.dtype, device=nnf.device)
    else:
        u = torch.cat([nnf[:, :, 1:], nnf[:, :, -1:]], 2) - torch.tensor([0, 1], dtype=nnf.dtype, device=nnf.device)
    return clamp_nnf(u, H, W)


def random_nnf(nnf, k, r=RANDOM_SEARCH_RANGE):
    """patch_match.py:94-98 with draw k"""
    B, H, W, _ = nnf.shape
    step = torch.from_numpy(randint(k, -r, r + 1, (B, H, W, 2))).to(nnf.device)
    return clamp_nnf(nnf + step.to(nnf.dtype), H, W)


# ------------------------------------------------------------------------------------------------ the three kernels
def remap(style, nnf, patch_size):
    """cupy_kernels.py:3-43 (remapping_kernel, unpadded): per pixel the mean over the taps (px, py), px-major, whose
    neighbour (y + px, x + py) and source nnf(neighbour) - (px, py) are inside the frame."""
    B, H, W, C = style.shape
    r = (patch_size - 1) // 2
    dev = style.device
    y = torch.arange(H, device=dev).view(1, H, 1)
    x = torch.arange(W, device=dev).view(1, 1, W)
    b = torch.arange(B, device=dev).view(B, 1, 1)
    s = torch.zeros((B, H, W, C), dtype=torch.float32, device=dev)
    num = torch.zeros((B, H, W), dtype=torch.int32, device=dev)
    for px in range(-r, r + 1):
        for py in range(-r, r + 1):
            ny, nx = y + px, x + py
            inside = (ny >= 0) & (ny < H) & (nx >= 0) & (nx < W)
            m = nnf[b, ny.clamp(0, H - 1), nx.clamp(0, W - 1)].long()
            sy, sx = m[..., 0] - px, m[..., 1] - py
            ok = inside & (sy >= 0) & (sx >= 0) & (sy < H) & (sx < W)
            v = style[b, sy.clamp(0, H - 1), sx.clamp(0, W - 1)]
            s = torch.where(ok.unsqueeze(-1), s + v, s)
            num = num + ok.to(torch.int32)
    return s / num.to(torch.float32).unsqueeze(-1).expand_as(s)


def _pad(x, r):
    return torch.nn.functional.pad(x, (0, 0, r, r, r, r))


def patch_errors(src_guide, tgt_guide, src_style, tgt_style, nnf, patch_size):
    """cupy_kernels.py:46-79 (patch_error_kernel) for the guide and the style pair at once: per pixel the sum over
    px, py in [-r, r] and the channels of (target(pixel + (px, py)) - source(nnf + (px, py)))^2, zero outside the frame;
    each square and each addition rounded (the reference's compiler may contract them into FMAs)."""
    B, H, W, C = src_guide.shape
    r = (patch_size - 1) // 2
    dev = src_guide.device
    Hp, Wp = H + 2 * r, W + 2 * r
    src = _pad(torch.cat([src_guide, src_style], -1), r).reshape(-1, 2 * C)
    tg, ts = _pad(tgt_guide, r), _pad(tgt_style, r)
    b = torch.arange(B, device=dev).view(B, 1, 1)
    base = (b * Hp + nnf[..., 0].long() + r) * Wp + nnf[..., 1].long() + r
    eg = torch.zeros((B, H, W), dtype=torch.float32, device=dev)
    es = torch.zeros_like(eg)
    for px in range(-r, r + 1):
        for py in range(-r, r + 1):
            s = src[base + (px * Wp + py)]
            t_g = tg[:, r + px:r + px + H, r + py:r + py + W]
            t_s = ts[:, r + px:r + px + H, r + py:r + py + W]
            for c in range(C):
                d = t_g[..., c] - s[..., c]
                eg = eg + d * d
            for c in range(C):
                d = t_s[..., c] - s[..., C + c]
                es = es + d * d
    return eg, es


def error(src_guide, tgt_guide, src_style, tgt_style, nnf, patch_size, guide_weight):
    """patch_match.py:76-87: error_guide * guide_weight + error_style, f32"""
    eg, es = patch_errors(src_guide, tgt_guide, src_style, tgt_style, nnf, patch_size)
    return eg * torch.tensor(np.float32(guide_weight), device=eg.device) + es


# ------------------------------------------------------------------------------------------------ PyramidPatchMatcher
class PyramidPatchMatcher:
    """patch_match.py:205-298 with the identity initialisation and no tracking (the smoother's path)."""

    def __init__(self, image_height, image_width, minimum_patch_size=5, num_iter=5, guide_weight=10.0):
        maximum_patch_size = minimum_patch_size + (num_iter - 1) * 2
        self.pyramid_level = int(np.log2(min(image_height, image_width) / maximum_patch_size))
        self.sizes = [(image_height // 2 ** (self.pyramid_level - 1 - l), image_width // 2 ** (self.pyramid_level - 1 - l))
                      for l in range(self.pyramid_level)]
        self.patch_size_list = [minimum_patch_size + i * 2 for i in range(num_iter)][::-1]
        self.guide_weight = guide_weight
        self.draws = 0

    def _draw(self):
        self.draws += 1
        return self.draws - 1

    def _update(self, sg, tg, ss, ts, nnf, err, cand, patch):
        """patch_match.py:158-163"""
        e = error(sg, tg, ss, ts, cand, patch, self.guide_weight)
        better = e < err
        return torch.where(better.unsqueeze(-1), cand, nnf), torch.where(better, e, err)

    def level(self, sg, tg, ss, nnf):
        """patch_match.py:191-202 (PatchMatcher.estimate_nnf)"""
        for patch in self.patch_size_list:
            ts = remap(ss, nnf, patch)
            err = error(sg, tg, ss, ts, nnf, patch, self.guide_weight)
            for d in permutation4(self._draw()):                                # :165-169
                nnf, err = self._update(sg, tg, ss, ts, nnf, err, neighbour_nnf(nnf, d), patch)
            for _ in range(RANDOM_SEARCH_STEPS):                                # :171-175
                nnf, err = self._update(sg, tg, ss, ts, nnf, err, random_nnf(nnf, self._draw()), patch)
        return nnf, remap(ss, nnf, self.patch_size_list[-1])                     # :201, the last iteration's patch

    def estimate_nnf(self, source_guide, target_guide, source_style):
        """f32 [B, H, W, C] tensors (any device) -> (nnf int32 [B, H, W, 2], target_style f32 [B, H, W, C])"""
        if self.pyramid_level < 1:
            raise ValueError("frames too small for one pyramid level")
        nnf = ts = None
        for lv, (h, w) in enumerate(self.sizes):
            nnf = identity_nnf(source_guide.shape[0], h, w, source_guide.device) if lv == 0 else upscale_nnf(nnf, h, w)
            nnf, ts = self.level(resample(source_guide, h, w), resample(target_guide, h, w), resample(source_style, h, w), nnf)
        return nnf, ts


# ------------------------------------------------------------------------------------------------ TableManager
def task_list(n):
    """runners/fast.py:12-32: for each frame i and each bit level it has clear, the task i -> (i with the bits up to
    that level set), stopping past the end; sorted (stably) by level."""
    out = []
    levels = max(1, n.bit_length()) if n > 0 else 1
    for i in range(n):
        j = i
        for lv in range(levels):
            if i >> lv & 1:
                continue
            j |= 1 << lv
            if j >= n:
                break
            out.append({"source": i, "target": j, "level": lv + 1})
    return sorted(out, key=functools.cmp_to_key(lambda u, v: u["level"] - v["level"]))


def tree_query(leftbound, rightbound):
    """runners/fast.py:66-75: the nodes (index, level) covering [leftbound, rightbound], from the right."""
    nodes, i = [], rightbound
    while i >= leftbound:
        lv = 0
        while (i >> lv) & 1 and i - (1 << (lv + 1)) + 1 >= leftbound:
            lv += 1
        nodes.append((i, lv))
        i -= 1 << lv
    return nodes


def _f32(x, ref):
    return torch.tensor(np.float32(x), device=ref.device)


def scaled(frame, s):
    """numpy's `frame * s` for a Python float s: f64 for uint8 and f64 frames, f32 (s rounded to f32) for f32 frames"""
    if frame.dtype == torch.float32:
        return frame * _f32(s, frame)
    return frame.double() * s


def promoted_add(a, b):
    return a + b if a.dtype == b.dtype else a.double() + b.double()


def _stack(frames):
    """np.stack of uint8 / f32 frames, then cp.array(dtype=float32)"""
    return torch.stack([f.to(torch.float32) for f in frames])


def build_remapping_table(frames_guide, frames_style, engine, batch_size):
    """runners/fast.py:34-54"""
    n = len(frames_guide)
    tasks = task_list(n)
    table = [[(frames_style[i], 1)] for i in range(n)]
    for s in range(0, len(tasks), batch_size):
        batch = tasks[s:s + batch_size]
        _, ts = engine.estimate_nnf(_stack([frames_guide[t["source"]] for t in batch]),
                                    _stack([frames_guide[t["target"]] for t in batch]),
                                    _stack([frames_style[t["source"]] for t in batch]))
        for t, result in zip(batch, ts):
            target, lv = t["target"], t["level"]
            if len(table[target]) == lv:
                table[target].append((result, 1))
            else:
                frame, weight = table[target][lv]
                mean = frame * _f32(weight / (weight + 1), frame) + result / torch.full_like(result, np.float32(weight + 1))
                table[target][lv] = (mean, weight + 1)
    return table


def remapping_table_to_blending_table(table):
    """runners/fast.py:56-64: (f1 + f2) / 2 in f32 (uint8 + f32 promotes to f32)"""
    for row in table:
        for j in range(1, len(row)):
            (f1, w1), (f2, w2) = row[j - 1], row[j]
            row[j] = ((f1.to(torch.float32) + f2) / torch.full_like(f2, 2.0), w1 + w2)
    return table


def process_window_sum(frames_guide, table, engine, window_size, batch_size):
    """runners/fast.py:77-106: the accumulator is f64 when the target's own node is a uint8 (level-0) frame"""
    n = len(table)
    tasks, result = [], []
    for target in range(n):
        for source, lv in tree_query(max(target - window_size, 0), target):
            if source != target:
                tasks.append({"source": source, "target": target, "level": lv})
            else:
                result.append(table[target][lv])
    for s in range(0, len(tasks), batch_size):
        batch = tasks[s:s + batch_size]
        _, ts = engine.estimate_nnf(_stack([frames_guide[t["source"]] for t in batch]),
                                    _stack([frames_guide[t["target"]] for t in batch]),
                                    _stack([table[t["source"]][t["level"]][0] for t in batch]))
        for t, f2 in zip(batch, ts):
            f1, w1 = result[t["target"]]
            w2 = table[t["source"]][t["level"]][1]
            w = w1 + w2
            result[t["target"]] = (promoted_add(scaled(f1, w1 / w), scaled(f2, w2 / w)), w)
    return result


def merge(table_l, frames_style, table_r):
    """__init__.py:45-51: weight_m = -1, f64 sums, clip(0, 255), truncating uint8 cast"""
    out = []
    for (fl, wl), fm, (fr, wr) in zip(table_l, frames_style, table_r):
        w = wl - 1 + wr
        v = promoted_add(promoted_add(scaled(fl, wl / w), scaled(fm, -1 / w)), scaled(fr, wr / w))
        out.append(v.clamp(0, 255).to(torch.uint8))
    return out


def run(frames_guide, frames_style, batch_size=8, window_size=64, minimum_patch_size=5, num_iter=5, guide_weight=10.0,
        device="cpu"):
    """FastBlendSmoother.run (__init__.py:26-52): uint8 [H, W, 3] frames -> uint8 [n, H, W, 3] (numpy)"""
    guide = [torch.from_numpy(np.ascontiguousarray(f)).to(device) for f in frames_guide]
    style = [torch.from_numpy(np.ascontiguousarray(f)).to(device) for f in frames_style]
    H, W = style[0].shape[:2]
    engine = PyramidPatchMatcher(H, W, minimum_patch_size, num_iter, guide_weight)
    tl = build_remapping_table(guide, style, engine, batch_size)
    tl = process_window_sum(guide, remapping_table_to_blending_table(tl), engine, window_size, batch_size)
    tr = build_remapping_table(guide[::-1], style[::-1], engine, batch_size)
    tr = process_window_sum(guide[::-1], remapping_table_to_blending_table(tr), engine, window_size, batch_size)[::-1]
    return torch.stack(merge(tl, style, tr)).cpu().numpy()
