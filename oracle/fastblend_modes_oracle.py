"""Restatement of FastBlend's balanced and accurate modes and keyframe interpolation (reference
diffsynth/extensions/FastBlend: patch_match.py with its three options, runners/balanced.py, runners/accurate.py,
runners/interpolation.py), in vectorised torch with the kernels' rounding, on top of oracle/fastblend_oracle.py.
Line numbers cite those files.

As in fastblend_oracle, every float operation is one torch op on whole arrays, rounded on its own, in the reference's
order, so the same code gives the same bits on the CPU (where tests/golden/fastblend_modes_tiny.npz pins it to the
reference) and on the GPU.  Each runner returns (uint8 [n, H, W, 3] numpy frames in frame order, the matcher's draws).
"""
import numpy as np
import torch

from oracle import fastblend_oracle as O


# ------------------------------------------------------------------------------------------------ the three options
def track_nnf(nnf, d, pairwise):
    """patch_match.py:116-132: entry b takes entry clamp(b + d, 0, B - 1)'s field; with the pairwise error, within the
    even and the odd entries separately"""
    B = nnf.shape[0]
    if not pairwise:
        return nnf[torch.arange(B, device=nnf.device).add(d).clamp(0, B - 1)]
    out = torch.zeros_like(nnf)
    for parity in (0, 1):
        sub = nnf[parity::2]
        out[parity::2] = sub[torch.arange(sub.shape[0], device=nnf.device).add(d).clamp(0, sub.shape[0] - 1)]
    return out


def batch_mean(x):
    """numpy's f32 mean(axis=0): the sum in b order, then / f32(B)"""
    s = x[0]
    for b in range(1, x.shape[0]):
        s = s + x[b]
    return s / torch.full_like(s, np.float32(x.shape[0]))


def guide_error(src_guide, tgt_guide, nnf, patch_size):
    return O.patch_errors(src_guide, tgt_guide, src_guide, tgt_guide, nnf, patch_size)[0]


def pairwise_style_error(src_style, nnf, patch_size):
    """cupy_kernels.py:82-119 and patch_match.py:63-74: per pair k the sum over px, py, c of
    (style[2k][nnf(2k) + (px, py)] - style[2k + 1][nnf(2k + 1) + (px, py)])^2, zero outside the frame, repeated for both
    members of the pair"""
    B, H, W, C = src_style.shape
    r = (patch_size - 1) // 2
    dev = src_style.device
    Hp, Wp = H + 2 * r, W + 2 * r
    src = torch.nn.functional.pad(src_style, (0, 0, r, r, r, r)).reshape(-1, C)
    b = torch.arange(B, device=dev).view(B, 1, 1)
    base = (b * Hp + nnf[..., 0].long() + r) * Wp + nnf[..., 1].long() + r
    ba, bb = base[0::2], base[1::2]
    e = torch.zeros((B // 2, H, W), dtype=torch.float32, device=dev)
    for px in range(-r, r + 1):
        for py in range(-r, r + 1):
            a, s = src[ba + (px * Wp + py)], src[bb + (px * Wp + py)]
            for c in range(C):
                d = a[..., c] - s[..., c]
                e = e + d * d
    return e.repeat_interleave(2, 0)


class PyramidPatchMatcher(O.PyramidPatchMatcher):
    """patch_match.py:205-298 with use_mean_target_style, use_pairwise_patch_error and tracking_window_size."""

    def __init__(self, image_height, image_width, minimum_patch_size=5, num_iter=5, guide_weight=10.0,
                 use_mean_target_style=False, use_pairwise_patch_error=False, tracking_window_size=0):
        super().__init__(image_height, image_width, minimum_patch_size, num_iter, guide_weight)
        self.mean, self.pairwise, self.tracking = use_mean_target_style, use_pairwise_patch_error, tracking_window_size

    def _error(self, sg, tg, ss, ts, nnf, patch):
        """patch_match.py:76-87"""
        gw = torch.tensor(np.float32(self.guide_weight), device=sg.device)
        if self.pairwise:
            return guide_error(sg, tg, nnf, patch) * gw + pairwise_style_error(ss, nnf, patch)
        if self.mean:
            ts = batch_mean(O.remap(ss, nnf, patch)).unsqueeze(0).expand_as(ss).contiguous()
        return O.error(sg, tg, ss, ts, nnf, patch, self.guide_weight)

    def _update(self, sg, tg, ss, ts, nnf, err, cand, patch):
        """patch_match.py:158-163"""
        e = self._error(sg, tg, ss, ts, cand, patch)
        better = e < err
        return torch.where(better.unsqueeze(-1), cand, nnf), torch.where(better, e, err)

    def level(self, sg, tg, ss, nnf):
        """patch_match.py:185-202"""
        for patch in self.patch_size_list:
            ts = O.remap(ss, nnf, patch)
            err = self._error(sg, tg, ss, ts, nnf, patch)
            for d in O.permutation4(self._draw()):
                nnf, err = self._update(sg, tg, ss, ts, nnf, err, O.neighbour_nnf(nnf, d), patch)
            for _ in range(O.RANDOM_SEARCH_STEPS):
                nnf, err = self._update(sg, tg, ss, ts, nnf, err, O.random_nnf(nnf, self._draw()), patch)
            for d in range(1, self.tracking + 1):
                nnf, err = self._update(sg, tg, ss, ts, nnf, err, track_nnf(nnf, d, self.pairwise), patch)
                nnf, err = self._update(sg, tg, ss, ts, nnf, err, track_nnf(nnf, -d, self.pairwise), patch)
        return nnf, O.remap(ss, nnf, self.patch_size_list[-1])


# ------------------------------------------------------------------------------------------------ runners
def _frames(frames, device):
    return [torch.from_numpy(np.ascontiguousarray(f)).to(device) for f in frames]


def _u8(x):
    return x.clamp(0, 255).to(torch.uint8)


def _result(out):
    return torch.stack(out).cpu().numpy()


def balanced(frames_guide, frames_style, batch_size, window_size, device="cpu", **config):
    """runners/balanced.py: the running mean f64(frame) * (w / (w + 1)) + f64(result / f32(w + 1)); each frame is saved
    as the blend before its last neighbour (the reference clips the `frame` it read)"""
    guide, style = _frames(frames_guide, device), _frames(frames_style, device)
    n = len(style)
    engine = PyramidPatchMatcher(*style[0].shape[:2], **config)
    tasks = [(s, t) for t in range(n) for s in range(t - window_size, t + window_size + 1) if 0 <= s < n and s != t]
    frames, out = [(None, 1)] * n, [None] * n
    for i in range(0, len(tasks), batch_size):
        batch = tasks[i:i + batch_size]
        _, ts = engine.estimate_nnf(O._stack([guide[s] for s, _ in batch]), O._stack([guide[t] for _, t in batch]),
                                    O._stack([style[s] for s, _ in batch]))
        for (s, t), result in zip(batch, ts):
            frame, w = frames[t]
            if frame is None:
                frame = style[t]
            frames[t] = (frame.double() * (w / (w + 1)) + (result / torch.full_like(result, np.float32(w + 1))).double(),
                         w + 1)
            if w + 1 == min(n, t + window_size + 1) - max(0, t - window_size):
                out[t] = _u8(frame.double())
                frames[t] = (None, 1)
    return _result(out), engine.draws


def accurate(frames_guide, frames_style, batch_size, window_size, device="cpu", **config):
    """runners/accurate.py: the f32 mean of every remapped frame of the window, in order"""
    guide, style = _frames(frames_guide, device), _frames(frames_style, device)
    n = len(style)
    engine = PyramidPatchMatcher(*style[0].shape[:2], use_mean_target_style=True, **config)
    out = []
    for t in range(n):
        l, r = max(t - window_size, 0), min(t + window_size + 1, n)
        remapped = []
        for i in range(l, r, batch_size):
            j = min(i + batch_size, r)
            _, ts = engine.estimate_nnf(O._stack(guide[i:j]), O._stack([guide[t]] * (j - i)), O._stack(style[i:j]))
            remapped.append(ts)
        out.append(_u8(batch_mean(torch.cat(remapped))))
    return _result(out), engine.draws


def _weight(l, m, r):
    wl, wr = abs(m - r), abs(m - l)
    return (0.5, 0.5) if wl + wr == 0 else (wl / (wl + wr), wr / (wl + wr))


def _task_groups(index_style, n):
    index_style = sorted(index_style)
    groups = [[(index_style[0], m, index_style[0]) for m in range(index_style[0])]] if index_style[0] > 0 else []
    groups += [[(l, m, r) for m in range(l, r)] for l, r in zip(index_style[:-1], index_style[1:])]
    return groups + [[(index_style[-1], m, index_style[-1]) for m in range(index_style[-1], n)]]


def interpolation(frames_guide, frames_style, index_style, batch_size, device="cpu", **config):
    """runners/interpolation.py InterpolationModeRunner: f32 frame_l * f32(w_l) + frame_r * f32(w_r)"""
    guide, style = _frames(frames_guide, device), _frames(frames_style, device)
    n = len(guide)
    engine = PyramidPatchMatcher(*style[0].shape[:2], use_pairwise_patch_error=True, **config)
    key = {index: i for i, index in enumerate(index_style)}
    out = [None] * n
    for tasks in _task_groups(index_style, n):
        for i in range(0, len(tasks), batch_size):
            batch = tasks[i:i + batch_size]
            sg = [guide[x] for l, m, r in batch for x in (l, r)]
            tg = [guide[m] for l, m, r in batch for _ in (l, r)]
            ss = [style[key[x]] for l, m, r in batch for x in (l, r)]
            _, ts = engine.estimate_nnf(O._stack(sg), O._stack(tg), O._stack(ss))
            for k, (l, m, r) in enumerate(batch):
                wl, wr = _weight(l, m, r)
                out[m] = _u8(ts[2 * k] * O._f32(wl, ts) + ts[2 * k + 1] * O._f32(wr, ts))
    return _result(out), engine.draws


def single_frame(frames_guide, frames_style, index_style, batch_size, device="cpu", **config):
    """runners/interpolation.py InterpolationModeSingleFrameRunner: overlapping batches of consecutive guide frames,
    each frame taken from the first batch that renders it before the tracking margin"""
    guide, style = _frames(frames_guide, device), _frames(frames_style, device)
    n, T = len(guide), config.get("tracking_window_size", 0)
    engine = PyramidPatchMatcher(*style[0].shape[:2], **config)
    key_guide, key_style = guide[index_style[0]], style[0]
    out, frame_id = [], 0
    for i in range(0, n, batch_size - 2 * T):
        l, r = (max(n - batch_size, 0), n) if i + batch_size > n else (i, i + batch_size)
        _, ts = engine.estimate_nnf(O._stack([key_guide] * (r - l)), O._stack(guide[l:r]), O._stack([key_style] * (r - l)))
        for j, frame in zip(range(l, r), ts):
            if j == frame_id:
                out.append(_u8(frame))
                frame_id += 1
            if r < n and r - frame_id <= T:
                break
    return _result(out), engine.draws
