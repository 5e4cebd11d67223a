"""FastBlend video deflickering on the native sm_90a kernels (include/svi_b200_fastblend.h and
include/svi_b200_fastblend_modes.h).

The reference's names and call semantics (diffsynth/extensions/FastBlend: __init__.py, runners/fast.py,
patch_match.py): `FastBlendSmoother()(frames)` matches every frame against the frames of a window around it with a
coarse-to-fine PatchMatch (`PyramidPatchMatcher`), remaps them onto it and blends them through the tree tables of
`TableManager`.  The whole computation runs on the device; frames cross the bus once as bytes in each direction.
The balanced and accurate modes and keyframe interpolation are the runners of `.runners`.

Exactness: every kernel repeats the reference's arithmetic in its order, each operation rounded on its own, and the host
keeps the reference's task order and batching (batch composition changes results: PyramidPatchMatcher's NNF upscale adds
+1 on the rows and columns whose index is odd and below the batch size).  The reference's unseeded CuPy draws are
replaced by a counter-based stream (draw k = the k-th randint / permutation since the matcher's construction; see
include/svi_b200_fastblend.h), so the same input gives the same bytes.  Blending-table frames keep the dtype numpy's
promotion gives them in the reference: uint8 input frames, f32 remapped frames and means, f64 window sums that start
from a uint8 frame, an f64 final merge.
"""
import collections
import functools

import cv2
import numpy as np
import torch
from PIL import Image

from ... import _native as nv

RANDOM_SEARCH_STEPS, RANDOM_SEARCH_RANGE = 3, 4      # the reference PatchMatcher's defaults (its PyramidPatchMatcher keeps them)
MAX_PATCH = 61                                        # SVI_FASTBLEND_MAX_PATCH: the step kernel's shared-memory windows

# A blending-table frame on the device: `data` f32 [H, W, 4] (f64 for kind "float64"); kind "uint8" is an input frame
# held as its f32 values, which numpy's promotion treats as the uint8 array it stands for.
Frame = collections.namedtuple("Frame", ["data", "kind"])


def _device(gpu_id):
    return torch.device("cuda", int(gpu_id))


def _unsupported(option, value, why):
    return ValueError(f"FastBlend: unsupported config {option}={value!r} ({why})")


class PyramidPatchMatcher:
    """Coarse-to-fine PatchMatch of target frames against source frames (patch_match.py:205).  `gpu_id` selects the
    device; `threads_per_block` is accepted and has no effect (the kernels choose their own launch shape).

    `use_mean_target_style` measures every candidate's style error against the batch mean of the source style remapped
    through that candidate; `use_pairwise_patch_error` gives entries 2k and 2k + 1 one shared style error, the patch
    distance between their source styles (the batch must be even); `tracking_window_size` T adds 2T steps per
    iteration whose candidates are the fields of the batch entries d = 1, -1, ..., T, -T away (within each parity class
    with the pairwise error)."""

    def __init__(self, image_height, image_width, channel, minimum_patch_size, threads_per_block=8, num_iter=5, gpu_id=0,
                 guide_weight=10.0, use_mean_target_style=False, use_pairwise_patch_error=False, tracking_window_size=0,
                 initialize="identity"):
        if initialize != "identity":
            raise _unsupported("initialize", initialize, "only the identity initialisation is implemented")
        if channel != 3:
            raise _unsupported("channel", channel, "frames are RGB")
        maximum_patch_size = minimum_patch_size + (num_iter - 1) * 2
        if minimum_patch_size < 1 or num_iter < 1 or maximum_patch_size > MAX_PATCH:
            raise _unsupported("minimum_patch_size", minimum_patch_size,
                               f"patches of 1 to {MAX_PATCH} pixels, num_iter >= 1")
        self.pyramid_level = int(np.log2(min(image_height, image_width) / maximum_patch_size))
        if self.pyramid_level < 1:
            raise ValueError(f"FastBlend: frames of {image_height}x{image_width} are too small for one pyramid level "
                             f"(the shorter side must be at least 2 x {maximum_patch_size}, twice the largest patch)")
        self.image_height, self.image_width, self.channel = image_height, image_width, channel
        self.pyramid_heights = [image_height // 2 ** (self.pyramid_level - 1 - l) for l in range(self.pyramid_level)]
        self.pyramid_widths = [image_width // 2 ** (self.pyramid_level - 1 - l) for l in range(self.pyramid_level)]
        self.patch_size_list = [minimum_patch_size + i * 2 for i in range(num_iter)][::-1]
        self.minimum_patch_size, self.num_iter = minimum_patch_size, num_iter
        self.gpu_id, self.guide_weight, self.initialize = gpu_id, guide_weight, initialize
        self.use_mean_target_style, self.use_pairwise_patch_error = bool(use_mean_target_style), bool(use_pairwise_patch_error)
        self.tracking_window_size = int(tracking_window_size)
        self.device = _device(gpu_id)
        self.draws = 0        # the random stream's counter: one per randint / permutation the reference would draw

    # -------------------------------------------------------------------------------------------- public interface
    def estimate_nnf(self, source_guide, target_guide, source_style):
        """[B, H, W, 3] frames (arrays or tensors, any dtype) -> host (nnf int32 [B, H, W, 2], target_style f32
        [B, H, W, 3]), as the reference's `.get()` returns them."""
        frames = [self._to_device(x) for x in (source_guide, target_guide, source_style)]
        nnf, ts = self.estimate_nnf_device(*frames)
        return nnf.cpu().numpy(), ts[..., :3].cpu().numpy()

    def check_batch(self, B):
        """The reference indexes the rows and columns of the first upscaled level with the odd numbers below the batch
        size (patch_match.py:265-266); a batch that reaches past them raises IndexError there."""
        odd = B - 1 if B % 2 == 0 else B - 2
        if self.pyramid_level >= 2 and odd >= 1 and odd >= 2 * min(self.pyramid_heights[0], self.pyramid_widths[0]):
            raise ValueError(f"FastBlend: batch_size {B} is too large for frames of {self.image_height}x{self.image_width}: "
                             f"the batch may not exceed the {2 * self.pyramid_heights[0]}x{2 * self.pyramid_widths[0]} "
                             f"second pyramid level")

    def estimate_nnf_device(self, source_guide, target_guide, source_style):
        """f32 [B, H, W, 4] frames on the device -> (nnf int32 [B, H, W, 2], target_style f32 [B, H, W, 4])."""
        B = source_guide.shape[0]
        self.check_batch(B)
        if self.use_pairwise_patch_error and B % 2:
            raise ValueError(f"FastBlend: the pairwise patch error pairs entries 2k and 2k + 1; a batch of {B} is odd")
        nv.require_cuda(self.device, "FastBlend")
        nnf = ts = None
        for level, (h, w) in enumerate(zip(self.pyramid_heights, self.pyramid_widths)):
            if level == 0:
                nnf = nv.fastblend_nnf_identity(torch.empty(B, h, w, 2, dtype=torch.int32, device=self.device))
            else:
                nnf = self._upscale(nnf, h, w)
            nnf, ts = self._level(self._resample(source_guide, h, w), self._resample(target_guide, h, w),
                                  self._resample(source_style, h, w), nnf)
        return nnf, ts

    # -------------------------------------------------------------------------------------------- levels
    def _to_device(self, x):
        t = torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x)
        if t.dim() != 4 or t.shape[-1] != 3 or tuple(t.shape[1:3]) != (self.image_height, self.image_width):
            raise ValueError(f"FastBlend: frames must be [B, {self.image_height}, {self.image_width}, 3], got {tuple(t.shape)}")
        if t.dtype == torch.uint8:
            return nv.fastblend_stage_frames(t.to(self.device).contiguous(),
                                             torch.empty(*t.shape[:3], 4, dtype=torch.float32, device=self.device))
        out = torch.zeros(*t.shape[:3], 4, dtype=torch.float32, device=self.device)
        out[..., :3] = t.to(self.device, torch.float32)      # cp.array(dtype=float32): one rounding of f64 input
        return out

    def _resample(self, x, h, w):
        """cv2.resize(INTER_AREA) of every frame (patch_match.py:234-242): the box kernel at an integer ratio (bit for bit
        cv2's order), cv2 on the host otherwise, as the reference does."""
        n, H, W, _ = x.shape
        if (H, W) == (h, w):
            return x
        k = H // h
        if h * k == H and w * k == W:
            return nv.fastblend_downsample(x, k, torch.empty(n, h, w, 4, dtype=torch.float32, device=self.device))
        host = x[..., :3].cpu().numpy()
        out = torch.zeros(n, h, w, 4, dtype=torch.float32)
        out[..., :3] = torch.from_numpy(np.stack([cv2.resize(f, (w, h), interpolation=cv2.INTER_AREA) for f in host]))
        return out.to(self.device)

    def _upscale(self, nnf, H, W):
        """patch_match.py:262-274: the doubled field with the odd-index-below-batch quirk; then cv2 INTER_LINEAR on the
        host, truncation and clamp when the level is not exactly twice the one below (an exact copy otherwise)."""
        B, h, w, _ = nnf.shape
        up = nv.fastblend_nnf_upscale(nnf, torch.empty(B, 2 * h, 2 * w, 2, dtype=torch.int32, device=self.device))
        if (2 * h, 2 * w) == (H, W):
            return up
        host = up.cpu().numpy().astype(np.float32)
        host = np.stack([cv2.resize(f, (W, H), interpolation=cv2.INTER_LINEAR) for f in host]).astype(np.int32)
        host[..., 0] = host[..., 0].clip(0, H - 1)
        host[..., 1] = host[..., 1].clip(0, W - 1)
        return torch.from_numpy(host).to(self.device)

    def _draw(self):
        self.draws += 1
        return self.draws - 1

    def _level(self, sg, tg, ss, nnf):
        """one level's PatchMatch (patch_match.py:191-202): per iteration the remapped style, the error of the current
        field, four neighbour steps in a drawn order, three random steps and 2T tracking steps; each step reads one
        field / error pair and writes the other.  Without the mean or pairwise error a neighbour or random step is one
        svi_fastblend_step; otherwise, and for tracking, the candidate field is built first and then evaluated
        (svi_fastblend_candidate, then svi_fastblend_select), the mean target style remapped and averaged in between."""
        B, H, W, _ = sg.shape
        plain = not (self.use_mean_target_style or self.use_pairwise_patch_error)
        pairwise = self.use_pairwise_patch_error
        mean_style = self.use_mean_target_style and not pairwise     # with both, the reference's mean goes unused
        ts = torch.empty_like(ss)
        fields = [nnf, torch.empty_like(nnf)]
        errs = [torch.empty(B, H, W, dtype=torch.float32, device=self.device) for _ in range(2)]
        cand = torch.empty_like(nnf) if not plain or self.tracking_window_size > 0 else None
        remapped = torch.empty_like(ss) if mean_style else None
        mean = torch.empty(H, W, 4, dtype=torch.float32, device=self.device) if mean_style else None
        cur = 0

        def step(mode, patch, **kw):
            nonlocal cur
            nv.fastblend_step(sg, ss, tg, ts, fields[cur], None if mode == nv.FB_CURRENT else errs[cur], fields[1 - cur],
                              errs[1 - cur], patch, mode, self.guide_weight, **kw)
            cur = 1 - cur

        def select(candidate, patch, first=False):
            nonlocal cur
            target = ts
            if pairwise:
                target = None
            elif mean_style:                                      # get_error (patch_match.py:76-87)
                nv.fastblend_remap(ss, candidate, patch, remapped)
                target = nv.fastblend_batch_mean(remapped, mean)
            nv.fastblend_select(sg, ss, tg, target, candidate, None if first else fields[cur], None if first else errs[cur],
                                fields[1 - cur], errs[1 - cur], patch, self.guide_weight, pairwise=pairwise)
            cur = 1 - cur

        def propose(mode, patch, **kw):
            if plain and mode != nv.FB_TRACK:
                step(mode, patch, **kw)
            else:
                nv.fastblend_candidate(fields[cur], cand, mode, pairwise=pairwise, **kw)
                select(cand, patch)

        for patch in self.patch_size_list:
            if plain:
                nv.fastblend_remap(ss, fields[cur], patch, ts)
                step(nv.FB_CURRENT, patch)
            else:
                select(fields[cur], patch, first=True)
            perm = self._permutation4()
            for d in perm:
                propose(nv.FB_NEIGHBOUR, patch, dir=d)
            for _ in range(RANDOM_SEARCH_STEPS):
                propose(nv.FB_RANDOM, patch, draw=self._draw(), radius=RANDOM_SEARCH_RANGE)
            for d in range(1, self.tracking_window_size + 1):          # track (patch_match.py:177-183)
                propose(nv.FB_TRACK, patch, shift=d)
                propose(nv.FB_TRACK, patch, shift=-d)
        out = torch.empty_like(ss)
        nv.fastblend_remap(ss, fields[cur], self.patch_size_list[-1], out)
        return fields[cur], out

    def _permutation4(self):
        """cp.random.permutation(4) as draw k: j = u(k, 0) % 24, Lehmer digits (j // 6, (j // 2) % 3, j % 2, 0)"""
        j = stream_u(self._draw(), 0) % 24
        rest = [0, 1, 2, 3]
        return [rest.pop(digit) for digit in (j // 6, (j // 2) % 3, j % 2, 0)]


def _lowbias32(x):
    m = 0xFFFFFFFF
    x ^= x >> 16
    x = (x * 0x7feb352d) & m
    x ^= x >> 15
    x = (x * 0x846ca68b) & m
    return x ^ (x >> 16)


def stream_u(k, i):
    """u(k, i) = lowbias32(lowbias32(k ^ 0x9e3779b9) ^ i), the random stream of include/svi_b200_fastblend.h"""
    return _lowbias32(_lowbias32((k & 0xFFFFFFFF) ^ 0x9e3779b9) ^ (i & 0xFFFFFFFF))


class TableManager:
    """The tree tables of the fast mode (runners/fast.py:8), on the device.  Frames are `Frame`s of the engine's device
    (`stage_frames`); a table is a list per frame of (Frame, weight) pairs."""

    def task_list(self, n):
        """For each frame i and each bit it has clear, from the lowest: the task i -> j (j = i with every bit up to that
        one set) at level bit + 1, until j passes the end; stably sorted by level."""
        tasks = []
        for i in range(n):
            j = i
            for bit in range(max(1, n.bit_length())):
                if i >> bit & 1:
                    continue
                j |= 1 << bit
                if j >= n:
                    break
                tasks.append({"source": i, "target": j, "level": bit + 1})
        tasks.sort(key=functools.cmp_to_key(lambda u, v: u["level"] - v["level"]))
        return tasks

    def tree_query(self, leftbound, rightbound):
        """The (index, level) nodes that cover [leftbound, rightbound], right to left: from index i, the highest level
        whose block (i - 2^level + 1 .. i) lies inside the range and whose lower bits of i are all set."""
        nodes, i = [], rightbound
        while i >= leftbound:
            level = 0
            while (i >> level) & 1 and i - (1 << (level + 1)) + 1 >= leftbound:
                level += 1
            nodes.append((i, level))
            i -= 1 << level
        return nodes

    def _match(self, engine, guide_src, guide_tgt, style_src):
        stack = lambda frames: torch.stack([f.data for f in frames])
        _, ts = engine.estimate_nnf_device(stack(guide_src), stack(guide_tgt), stack(style_src))
        return ts

    def build_remapping_table(self, frames_guide, frames_style, patch_match_engine, batch_size, desc=""):
        """Each task's remapped style frame, averaged per (target, level) in task order (f32 running mean)."""
        n = len(frames_guide)
        tasks = self.task_list(n)
        table = [[(frames_style[i], 1)] for i in range(n)]
        for start in range(0, len(tasks), batch_size):
            batch = tasks[start:start + batch_size]
            ts = self._match(patch_match_engine, [frames_guide[t["source"]] for t in batch],
                             [frames_guide[t["target"]] for t in batch], [frames_style[t["source"]] for t in batch])
            for t, result in zip(batch, ts):
                target, level = t["target"], t["level"]
                if len(table[target]) == level:
                    table[target].append((Frame(result, "float32"), 1))
                else:
                    frame, weight = table[target][level]
                    out = torch.empty_like(result)
                    nv.fastblend_table(nv.FB_MEAN, out, frame.data, weight / (weight + 1), result, weight + 1)
                    table[target][level] = (Frame(out, "float32"), weight + 1)
        return table

    def remapping_table_to_blending_table(self, table):
        """Entry j becomes the f32 mean of entries j - 1 (already blended) and j; the weights add."""
        for row in table:
            for j in range(1, len(row)):
                (f1, w1), (f2, w2) = row[j - 1], row[j]
                out = torch.empty_like(f2.data)
                nv.fastblend_table(nv.FB_HALF, out, f1.data, 0.0, f2.data, 0.0, a_u8=f1.kind == "uint8")
                row[j] = (Frame(out, "float32"), w1 + w2)
        return table

    def process_window_sum(self, frames_guide, blending_table, patch_match_engine, window_size, batch_size, desc=""):
        """Per target, the weighted mean of the blended nodes covering [target - window_size, target], each remapped onto
        it; f64 when the target's own node is an input frame, f32 otherwise (numpy's promotion)."""
        n = len(blending_table)
        tasks, result = [], []
        for target in range(n):
            for source, level in self.tree_query(max(target - window_size, 0), target):
                if source != target:
                    tasks.append({"source": source, "target": target, "level": level})
                else:
                    result.append(blending_table[target][level])
        for start in range(0, len(tasks), batch_size):
            batch = tasks[start:start + batch_size]
            ts = self._match(patch_match_engine, [frames_guide[t["source"]] for t in batch],
                             [frames_guide[t["target"]] for t in batch],
                             [blending_table[t["source"]][t["level"]][0] for t in batch])
            for t, f2 in zip(batch, ts):
                f1, w1 = result[t["target"]]
                w2 = blending_table[t["source"]][t["level"]][1]
                w = w1 + w2
                kind = "float32" if f1.kind == "float32" else "float64"
                out = torch.empty(f2.shape, dtype=torch.float32 if kind == "float32" else torch.float64, device=f2.device)
                nv.fastblend_table(nv.FB_WSUM, out, f1.data, w1 / w, f2, w2 / w, a_u8=f1.kind == "uint8")
                result[t["target"]] = (Frame(out, kind), w)
        return result


def stage_frames(frames, device):
    """uint8 RGB frames (PIL images or [H, W, 3] arrays, or one uint8 [F, H, W, 3] tensor, which stays on the device)
    -> `Frame`s on the device (one upload, one staging launch)."""
    if torch.is_tensor(frames):
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3 or frames.shape[0] == 0:
            raise ValueError("FastBlend: a frame tensor must be uint8 [F, H, W, 3]")
        u8 = frames.to(device).contiguous()
    else:
        arrs = [np.asarray(f.convert("RGB") if isinstance(f, Image.Image) else f) for f in frames]
        if not arrs:
            raise ValueError("FastBlend: no frames")
        H, W = arrs[0].shape[:2]
        if any(a.dtype != np.uint8 or a.shape != (H, W, 3) for a in arrs):
            raise ValueError("FastBlend: frames must be uint8 RGB of one size (PIL images or [H, W, 3] arrays)")
        u8 = torch.from_numpy(np.stack(arrs)).to(device)
    F, H, W, _ = u8.shape
    staged = nv.fastblend_stage_frames(u8, torch.empty(F, H, W, 4, dtype=torch.float32, device=device))
    return [Frame(f, "uint8") for f in staged]


def stage_pair(frames_guide, frames_style, device):
    """stage_frames of the guide and style frames (the guide is the style when they are the same object); both of one
    size and count"""
    style = stage_frames(frames_style, device)
    guide = style if frames_guide is frames_style else stage_frames(frames_guide, device)
    if len(guide) != len(style) or guide[0].data.shape != style[0].data.shape:
        raise ValueError("FastBlend: original and rendered frames must be as many and of one size")
    return guide, style


def frame_size(frame):
    """(H, W) of a PIL image or [H, W, 3] array or tensor"""
    if torch.is_tensor(frame):
        return tuple(frame.shape[:2])
    return np.asarray(frame.convert("RGB") if isinstance(frame, Image.Image) else frame).shape[:2]


def fast_mode(frames_guide, frames_style, batch_size, window_size, ebsynth_config):
    """The fast mode (runners/fast.py, __init__.py): the left and right tree tables and their merge.  Frames (PIL images
    or uint8 [H, W, 3] arrays) -> PIL images; frames_style as a uint8 [F, H, W, 3] tensor -> a tensor on the device."""
    H, W = frame_size(frames_style[0])
    engine = PyramidPatchMatcher(image_height=H, image_width=W, channel=3, **ebsynth_config)
    nv.require_cuda(engine.device, "FastBlend")
    guide, style = stage_pair(frames_guide, frames_style, engine.device)
    tm = TableManager()
    table_l = tm.build_remapping_table(guide, style, engine, batch_size)
    table_l = tm.process_window_sum(guide, tm.remapping_table_to_blending_table(table_l), engine, window_size, batch_size)
    table_r = tm.build_remapping_table(guide[::-1], style[::-1], engine, batch_size)
    table_r = tm.process_window_sum(guide[::-1], tm.remapping_table_to_blending_table(table_r), engine, window_size,
                                    batch_size)[::-1]
    out = torch.empty(len(style), H, W, 3, dtype=torch.uint8, device=engine.device)
    for i, ((fl, wl), fm, (fr, wr)) in enumerate(zip(table_l, style, table_r)):
        w = wl - 1 + wr                                         # the reference's weight_m = -1
        nv.fastblend_table(nv.FB_WSUM, out[i], fl.data, wl / w, fm.data, -1 / w, c=fr.data, sc=wr / w,
                           a_u8=fl.kind == "uint8", b_u8=True, c_u8=fr.kind == "uint8")
    if torch.is_tensor(frames_style):
        return out
    return [Image.fromarray(f) for f in out.cpu().numpy()]


class FastBlendSmoother:
    """FastBlend's fast mode (__init__.py:7): deflickers rendered frames, guided by the original frames or, with
    original_frames=None, by the rendered frames themselves."""

    def __init__(self):
        self.batch_size = 8
        self.window_size = 64
        self.ebsynth_config = {
            "minimum_patch_size": 5,
            "threads_per_block": 8,
            "num_iter": 5,
            "gpu_id": 0,
            "guide_weight": 10.0,
            "initialize": "identity",
            "tracking_window_size": 0,
        }

    @staticmethod
    def from_model_manager(model_manager):
        return FastBlendSmoother()

    def run(self, frames_guide, frames_style, batch_size, window_size, ebsynth_config):
        """Frames (PIL images or uint8 [H, W, 3] arrays) -> PIL images.  The fast mode keeps the reference's per-frame
        target style and plain patch error, without tracking: those options raise ValueError here (the balanced and
        accurate modes and keyframe interpolation, in `.runners`, are where they apply)."""
        for option, why in (("use_mean_target_style", "the accurate mode's option (runners.AccurateModeRunner)"),
                            ("use_pairwise_patch_error", "keyframe interpolation's option (runners.InterpolationModeRunner)"),
                            ("tracking_window_size", "the fast mode does not track")):
            if ebsynth_config.get(option):
                raise _unsupported(option, ebsynth_config[option], why)
        return fast_mode(frames_guide, frames_style, batch_size, window_size, ebsynth_config)

    def __call__(self, rendered_frames, original_frames=None, **kwargs):
        frames = self.run(rendered_frames if original_frames is None else original_frames, rendered_frames,
                          self.batch_size, self.window_size, self.ebsynth_config)
        return frames
