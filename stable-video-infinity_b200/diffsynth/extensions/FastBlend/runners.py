"""FastBlend's runners (the reference's diffsynth/extensions/FastBlend/runners): the fast, balanced and accurate
deflicker modes and keyframe interpolation, on the native kernels.

Each runner keeps the reference's signature, task order and batching (the batch composition changes the bits: see
PyramidPatchMatcher), writes `%05d.png` into `save_path` when one is given, and returns the frames as PIL images in
frame order (the reference returns None).  Frames go in as PIL images or uint8 [H, W, 3] arrays and cross the bus once
as bytes in each direction; everything between stays on the device.  The fast, balanced and accurate runners also take
the frames as a uint8 [F, H, W, 3] tensor, and then return the output as a uint8 tensor on the device.

Kept from the reference on purpose:
  - Balanced saves each frame's blend as it stood *before* its last neighbour was added (runners/balanced.py clips the
    `frame` it read, not the one it stored), so the last neighbour of every window never reaches the output.
  - Interpolation does not copy a keyframe into the output: it re-renders it as the keyframe PatchMatched onto its own
    guide frame (weight 1; a frame at or after the last keyframe blends 0.5 + 0.5 of the same match), so an output
    keyframe can differ from the input one.
Input the reference would crash on or drop silently raises ValueError instead.
"""
import os

import torch
from PIL import Image

from ... import _native as nv
from . import Frame, PyramidPatchMatcher, fast_mode, frame_size, stage_frames, stage_pair


def _raw(frames):
    """the reference's VideoData (`raw_data()`) or a sequence of frames -> a list of frames; a frame tensor as it is"""
    if torch.is_tensor(frames):
        return frames
    return frames.raw_data() if hasattr(frames, "raw_data") else list(frames)


def _stack(frames):
    return torch.stack([f.data for f in frames])


def _finish(out, save_path, frames_style=None):
    """uint8 [n, H, W, 3] on the device -> PIL images (or `out` itself when frames_style is a tensor), saved as
    %05d.png when save_path is given"""
    if save_path is None and torch.is_tensor(frames_style):
        return out
    images = [Image.fromarray(f) for f in out.cpu().numpy()]
    if save_path is not None:
        for i, image in enumerate(images):
            image.save(os.path.join(save_path, "%05d.png" % i))
    return out if torch.is_tensor(frames_style) else images


def _engine(frames_style, ebsynth_config, **options):
    H, W = frame_size(frames_style[0])
    engine = PyramidPatchMatcher(image_height=H, image_width=W, channel=3, **options, **ebsynth_config)
    nv.require_cuda(engine.device, "FastBlend")
    return engine


class FastModeRunner:
    """runners/fast.py: the fast mode of `FastBlendSmoother`, taking the matcher's options from ebsynth_config."""

    def run(self, frames_guide, frames_style, batch_size, window_size, ebsynth_config, save_path=None):
        frames = fast_mode(_raw(frames_guide), _raw(frames_style), batch_size, window_size, ebsynth_config)
        if save_path is not None:
            for i, image in enumerate(frames if not torch.is_tensor(frames) else _finish(frames, None)):
                image.save(os.path.join(save_path, "%05d.png" % i))
        return frames


class BalancedModeRunner:
    """runners/balanced.py: every frame matched against each frame of its window, blended in a running mean."""

    def run(self, frames_guide, frames_style, batch_size, window_size, ebsynth_config, desc="Balanced Mode",
            save_path=None):
        n = len(frames_style)
        if n < 2 or window_size < 1:
            raise ValueError(f"FastBlend balanced mode: needs at least 2 frames and window_size >= 1 "
                             f"(got {n} frames, window_size {window_size}); there would be nothing to blend")
        engine = _engine(frames_style, ebsynth_config)
        guide, style = stage_pair(frames_guide, frames_style, engine.device)
        H, W = style[0].data.shape[:2]
        tasks = [(source, target) for target in range(n) for source in range(target - window_size, target + window_size + 1)
                 if 0 <= source < n and source != target]
        frames = [(None, 1)] * n
        out = torch.empty(n, H, W, 3, dtype=torch.uint8, device=engine.device)
        for start in range(0, len(tasks), batch_size):
            batch = tasks[start:start + batch_size]
            _, ts = engine.estimate_nnf_device(_stack([guide[s] for s, _ in batch]), _stack([guide[t] for _, t in batch]),
                                               _stack([style[s] for s, _ in batch]))
            for (source, target), result in zip(batch, ts):
                frame, weight = frames[target]
                if frame is None:
                    frame = style[target]
                blend = torch.empty(H, W, 4, dtype=torch.float64, device=engine.device)
                nv.fastblend_running_mean(frame.data, weight / (weight + 1), result, weight + 1, blend,
                                          frame_u8=frame.kind == "uint8")
                frames[target] = (Frame(blend, "float64"), weight + 1)
                if weight + 1 == min(n, target + window_size + 1) - max(0, target - window_size):
                    nv.fastblend_to_u8(frame.data, out[target], a_u8=frame.kind == "uint8")   # the blend before this one
                    frames[target] = (None, 1)
        return _finish(out, save_path, frames_style)


class AccurateModeRunner:
    """runners/accurate.py: every frame matched against its whole window with the mean target style, the remapped
    frames averaged."""

    def run(self, frames_guide, frames_style, batch_size, window_size, ebsynth_config, desc="Accurate Mode",
            save_path=None):
        if window_size < 0:
            raise ValueError(f"FastBlend accurate mode: window_size must be >= 0, got {window_size}")
        engine = _engine(frames_style, ebsynth_config, use_mean_target_style=True)
        guide, style = stage_pair(frames_guide, frames_style, engine.device)
        n = len(style)
        H, W = style[0].data.shape[:2]
        out = torch.empty(n, H, W, 3, dtype=torch.uint8, device=engine.device)
        mean = torch.empty(H, W, 4, dtype=torch.float32, device=engine.device)
        for target in range(n):
            l, r = max(target - window_size, 0), min(target + window_size + 1, n)
            remapped = []
            for i in range(l, r, batch_size):
                j = min(i + batch_size, r)
                _, ts = engine.estimate_nnf_device(_stack(guide[i:j]), _stack([guide[target]] * (j - i)),
                                                   _stack(style[i:j]))
                remapped.append(ts)
            nv.fastblend_batch_mean(torch.cat(remapped), mean)
            nv.fastblend_to_u8(mean, out[target])
        return _finish(out, save_path, frames_style)


def _check_keyframes(index_style, frames_style, n, single):
    index_style = [int(i) for i in index_style]
    if not index_style or (not single and len(index_style) != len(frames_style)) or (single and not len(frames_style)):
        raise ValueError(f"FastBlend interpolation: {len(index_style)} keyframe indices for {len(frames_style)} keyframes")
    if any(i < 0 or i >= n for i in index_style) or len(set(index_style)) != len(index_style):
        raise ValueError(f"FastBlend interpolation: keyframe indices {index_style} must be distinct frames of 0..{n - 1}")
    return index_style


class InterpolationModeRunner:
    """runners/interpolation.py: each frame rendered from the keyframes on either side of it, both PatchMatched onto
    its guide frame with the pairwise patch error, blended by distance."""

    def get_index_dict(self, index_style):
        return {index: i for i, index in enumerate(index_style)}

    def get_weight(self, l, m, r):
        weight_l, weight_r = abs(m - r), abs(m - l)
        if weight_l + weight_r == 0:
            return 0.5, 0.5
        return weight_l / (weight_l + weight_r), weight_r / (weight_l + weight_r)

    def get_task_group(self, index_style, n):
        """(l, m, r) triples: the frames before the first keyframe from it alone, each segment between two keyframes
        from both, the frames from the last keyframe on from it alone"""
        index_style = sorted(index_style)
        groups = []
        if index_style[0] > 0:
            groups.append([(index_style[0], m, index_style[0]) for m in range(index_style[0])])
        for l, r in zip(index_style[:-1], index_style[1:]):
            groups.append([(l, m, r) for m in range(l, r)])
        groups.append([(index_style[-1], m, index_style[-1]) for m in range(index_style[-1], n)])
        return groups

    def run(self, frames_guide, frames_style, index_style, batch_size, ebsynth_config, save_path=None):
        n = len(frames_guide)
        index_style = _check_keyframes(index_style, frames_style, n, single=False)
        engine = _engine(frames_style, ebsynth_config, use_mean_target_style=False, use_pairwise_patch_error=True)
        guide = stage_frames(frames_guide, engine.device)
        style = stage_frames(frames_style, engine.device)
        H, W = style[0].data.shape[:2]
        if guide[0].data.shape != style[0].data.shape:
            raise ValueError("FastBlend interpolation: guide frames and keyframes must be of one size")
        index_dict = self.get_index_dict(index_style)
        out = torch.empty(n, H, W, 3, dtype=torch.uint8, device=engine.device)
        for tasks in self.get_task_group(index_style, n):
            for start in range(0, len(tasks), batch_size):
                batch = tasks[start:start + batch_size]
                sg, tg, ss = [], [], []
                for l, m, r in batch:                                   # l -> m, then r -> m
                    sg += [guide[l], guide[r]]
                    tg += [guide[m], guide[m]]
                    ss += [style[index_dict[l]], style[index_dict[r]]]
                _, ts = engine.estimate_nnf_device(_stack(sg), _stack(tg), _stack(ss))
                for k, (l, m, r) in enumerate(batch):
                    weight_l, weight_r = self.get_weight(l, m, r)
                    nv.fastblend_table(nv.FB_WSUM, out[m], ts[2 * k], weight_l, ts[2 * k + 1], weight_r)
        return _finish(out, save_path)


class InterpolationModeSingleFrameRunner:
    """runners/interpolation.py: one keyframe PatchMatched onto every guide frame, in overlapping batches of
    consecutive frames so that tracking reaches across each batch."""

    def run(self, frames_guide, frames_style, index_style, batch_size, ebsynth_config, save_path=None):
        tracking_window_size = ebsynth_config.get("tracking_window_size", 0)
        if tracking_window_size * 2 >= batch_size:
            raise ValueError("batch_size should be larger than track_window_size * 2")
        n = len(frames_guide)
        index_style = _check_keyframes(index_style, frames_style, n, single=True)
        engine = _engine(frames_style, ebsynth_config)
        guide = stage_frames(frames_guide, engine.device)
        key_style = stage_frames(frames_style[:1], engine.device)[0]
        key_guide = guide[index_style[0]]
        H, W = key_style.data.shape[:2]
        if key_guide.data.shape != key_style.data.shape:
            raise ValueError("FastBlend interpolation: guide frames and keyframes must be of one size")
        out = torch.empty(n, H, W, 3, dtype=torch.uint8, device=engine.device)
        frame_id = 0
        for i in range(0, n, batch_size - tracking_window_size * 2):
            l, r = (max(n - batch_size, 0), n) if i + batch_size > n else (i, i + batch_size)
            _, ts = engine.estimate_nnf_device(_stack([key_guide] * (r - l)), _stack(guide[l:r]),
                                               _stack([key_style] * (r - l)))
            for j, frame in zip(range(l, r), ts):
                if j == frame_id:
                    nv.fastblend_to_u8(frame, out[frame_id])
                    frame_id += 1
                if r < n and r - frame_id <= tracking_window_size:
                    break
        return _finish(out[:frame_id], save_path)
