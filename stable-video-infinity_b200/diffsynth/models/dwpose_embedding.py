"""SVI-Dance pose stem: pose video -> token-space condition added to the DiT's patch embedding (SURVEY.md §8f.2).

The reference builds the stem inline (``pipelines/svi_video_dance.py:254-268``): seven ``nn.Conv3d`` with SiLU in
between — three 3x3x3 convs at full resolution (3 -> 16 -> 16 -> 16 channels), one with spatial stride 2, two with
stride 2 in time and space, and a (1,2,2)/(1,2,2) projection to the DiT width — applied to
``cat([first pose frame x3, pose video]) / 255`` (``:526-528``) and flattened to ``[1, f*h*w, dim]``.  The weights arrive
as extra-module keys of the SVI-Dance LoRA file (``dwpose_embedding.N.{weight,bias}``, ``:270-275``).

``make_dwpose_embedding`` returns the same ``nn.Sequential`` (same keys) as a parameter container;
``DWPoseEmbeddingEngine`` runs it on the kernel library: the 3x3x3 convolutions on the implicit-GEMM conv kernel
(``svi_conv3d_causal`` with an explicit frame-slot table: symmetric temporal padding and temporal stride are just a
different table; spatial stride 2 with padding 1 is a 2x2 conv over a space-to-depth input, weights repacked on the
host), SiLU fused into the bf16 staging of the next conv's input, the final projection on ``svi_gemm_bf16``.

UniAnimate-DiT adds a second, 2-D stem on a single reference-pose image (``randomref_embedding_pose``, reference
``pipelines/wan_video.py:543-558``): six ``nn.Conv2d`` 3x3 / padding 1 (3 -> 16 -> 16 -> 16 -> 16 -> 16 -> 20 channels,
strides 1, 1, 1, 2, 2, 2, SiLU after all but the last).  ``RandomRefEmbeddingEngine`` runs it on the same conv launch as
the 3-D stem with one frame and kt = 1.

The Replace-Anyone model of UniAnimate-DiT adds two more 3-D stems (reference ``pipelines/wan_video.py:1353-1369``), both
3x3x3 / padding 1 with SiLU between the convs: ``learn_in_embedding`` (4 -> 16 -> 16 -> 16 -> 16 channels, strides 1,
(1, 2, 2), 2, 2) on the masked video and its keep mask, and ``inpaint_embedding`` (16 -> 16 -> 16 -> 16, stride 1) on the
VAE latents of the masked video.  ``LearnInEmbeddingEngine`` and ``InpaintEmbeddingEngine`` run them on the pose stem's
layer loop (``_StemEngine._layers``).
"""
import torch
import torch.nn as nn

from .. import _native as nv
from .wan_video_vae import _Conv, _Ring, _pick_tile_w


def make_dwpose_embedding(dim=5120, concat_dim=4):
    c = concat_dim * 4
    return nn.Sequential(
        nn.Conv3d(3, c, (3, 3, 3), stride=(1, 1, 1), padding=(1, 1, 1)), nn.SiLU(),
        nn.Conv3d(c, c, (3, 3, 3), stride=(1, 1, 1), padding=(1, 1, 1)), nn.SiLU(),
        nn.Conv3d(c, c, (3, 3, 3), stride=(1, 1, 1), padding=(1, 1, 1)), nn.SiLU(),
        nn.Conv3d(c, c, (3, 3, 3), stride=(1, 2, 2), padding=(1, 1, 1)), nn.SiLU(),
        nn.Conv3d(c, c, 3, stride=(2, 2, 2), padding=1), nn.SiLU(),
        nn.Conv3d(c, c, 3, stride=(2, 2, 2), padding=1), nn.SiLU(),
        nn.Conv3d(c, dim, (1, 2, 2), stride=(1, 2, 2), padding=0))


def slot_table(frames, zero_slot, T_out, t_stride, kt):
    """Ring slots read by output frame t, tap a: input frame t*t_stride + a - (kt-1)//2 (symmetric temporal padding:
    1 for the 3x3x3 convs, 0 for a Conv2d run as kt = 1), the zero slot outside the video.  Pure host logic (CPU-tested
    against nn.Conv3d and nn.Conv2d)."""
    n_in = len(frames)
    pad = (kt - 1) // 2
    table = []
    for t in range(T_out):
        row = []
        for a in range(kt):
            i = t * t_stride + a - pad
            row.append(frames[i] if 0 <= i < n_in else zero_slot)
        table.append(row)
    return table


class StemPlan:
    """Kernel-ready weights of the seven convolutions (device-agnostic packing; the engine needs them on a GPU)."""

    def __init__(self, seq: nn.Sequential, device):
        convs = [m for m in seq if isinstance(m, nn.Conv3d)]
        if len(convs) != 7:
            raise RuntimeError("dwpose_embedding must be the 7-conv stem of svi_video_dance.py:256-268")
        dev = torch.device(device)
        self.c = convs[1].in_channels
        self.full = [_Conv(m.weight, m.bias, dev) for m in convs[:3]]                      # stride 1, padding 1
        self.down = [_Conv(m.weight, m.bias, dev, s2d="before") for m in convs[3:6]]        # spatial stride 2, padding 1
        self.t_stride = [m.stride[0] for m in convs[3:6]]
        last = convs[6]
        k = 4 * self.c
        self.kproj = max(64, (k + 7) // 8 * 8)
        w = torch.zeros(last.out_channels, self.kproj, dtype=torch.float32, device=dev)
        wl = last.weight.detach().to(dev, torch.float32)                                   # [dim, c, 1, 2, 2]
        for dy in range(2):
            for dx in range(2):
                w[:, (dy * 2 + dx) * self.c:(dy * 2 + dx + 1) * self.c] = wl[:, :, 0, dy, dx]
        self.w_proj = w.to(torch.bfloat16).contiguous()
        self.b_proj = last.bias.detach().to(dev, torch.float32).contiguous()


class _StemEngine:
    """The conv launch both pose stems share."""
    MAX_T = 4      # output frames per conv launch (slot table of svi_conv_desc)

    def __init__(self, device, what):
        nv.require_cuda(device, what)
        self.device = torch.device(device)
        self.launches = 0

    def _conv(self, cv, ring, frames, T_out, t_stride, H, W):
        """out[t] = sum_a w[a] * in[t*t_stride + a - (kt-1)//2] (zero outside): symmetric temporal padding, spatial
        padding 1."""
        full_table = slot_table(frames, ring.slots, T_out, t_stride, cv.kt)
        out = torch.empty(T_out, H, W, cv.c_out, device=self.device, dtype=torch.float32)
        for t0 in range(0, T_out, self.MAX_T):
            n = min(self.MAX_T, T_out - t0)
            table = full_table[t0:t0 + n]
            d = nv.ConvDesc()
            d.x_ring = ring.buf.data_ptr()
            d.ring_slots, d.in_H, d.in_W, d.C_in = ring.slots + 1, ring.H, ring.W, ring.C
            d.w_packed, d.w_rows, d.w_ld = cv.w.data_ptr(), cv.w.shape[0], cv.w.shape[1]
            d.kt, d.kh, d.kw, d.pad_h, d.pad_w = cv.kt, cv.kh, cv.kw, 1, 1
            d.H, d.W, d.T = H, W, n
            for t in range(n):
                for a in range(cv.kt):
                    d.slot[t * 3 + a] = table[t][a]
            d.C_out = cv.c_out
            d.tile_w = _pick_tile_w(H, W)
            o = out[t0:t0 + n]
            d.out, d.out_frame_stride, d.out_ld = o.data_ptr(), out.stride(0), cv.c_out
            d.n_split, d.split_offset = 0, 0
            d.bias = cv.b.data_ptr()
            nv.conv3d_causal(d)
            self.launches += 1
        return out

    def _layers(self, full, down, t_strides, stage, frames, H, W):
        """The layer sequence of the 3-D stems: full-resolution convs (stride 1), then convs with spatial stride 2 and
        temporal strides `t_strides`, all 3x3x3 with padding 1 and SiLU between them.  `stage(ring)` writes the first
        conv's input into a ring of max(frames) + 1 frames; `frames` maps that conv's input frames to ring slots, so a
        repeated slot repeats a frame without a copy.  The later full-resolution convs restage frame t into slot t, which
        needs a ring of at least len(frames) frames.  Returns the last conv's f32 output [T, H', W', c_out]."""
        dev = self.device
        # ---- full-resolution convs: one ring holds the input frames (+ the zero slot) and is re-staged layer by layer
        ring = _Ring(max(frames) + 1, H, W, full[0].c_in, dev, history=0)
        stage(ring)
        T = len(frames)
        x = self._conv(full[0], ring, frames, T, 1, H, W)
        for cv in full[1:]:
            for t in range(T):
                xt = x[t]                                                                     # [H, W, c] f32
                nv.vae_norm_act(xt, H * W, xt.shape[-1], xt.stride(1), None, True, ring.buf[t], ring.C)   # SiLU -> bf16
                self.launches += 1
            x = self._conv(cv, ring, list(range(T)), T, 1, H, W)
        del ring
        # ---- strided convs: SiLU + space-to-depth staging, 2x2 spatial taps, temporal stride through the slot table
        for cv, ts in zip(down, t_strides):
            Tn, Hn, Wn, Cn = x.shape
            ring = _Ring(Tn, Hn // 2, Wn // 2, 4 * Cn, dev, history=0)
            for t in range(Tn):
                nv.vae_space_to_depth_act(x[t], Hn, Wn, Cn, nv.ACT_SILU, ring.buf[t])
                self.launches += 1
            T_out = (Tn + 2 - 3) // ts + 1
            x = self._conv(cv, ring, list(range(Tn)), T_out, ts, Hn // 2, Wn // 2)
            del ring
        return x


class DWPoseEmbeddingEngine(_StemEngine):
    def __init__(self, seq: nn.Sequential, device):
        super().__init__(device, "the pose stem")
        plan = StemPlan(seq, self.device)
        self.c, self.full, self.down, self.t_stride = plan.c, plan.full, plan.down, plan.t_stride
        self.kproj, self.w_proj, self.b_proj = plan.kproj, plan.w_proj, plan.b_proj

    def forward(self, pose):
        """pose f32 [3, T, H, W] (already /255 and front-padded as in :527) -> tokens f32 [1, f*h*w, dim]."""
        dev = self.device
        C, T, H, W = pose.shape
        if C != 3 or H % 16 or W % 16:
            raise RuntimeError(f"svi_b200: pose video must be [3, T, H, W] with H, W multiples of 16, got {tuple(pose.shape)}")
        pose = pose.to(device=dev, dtype=torch.float32).contiguous()

        def stage(ring):
            xin = torch.empty(H, W, 8, device=dev, dtype=torch.float32)
            for t in range(T):
                nv.vae_from_planar(pose[:, t], 3, H * W, None, None, xin, 8, False, ldc=T * H * W)
                nv.vae_norm_act(xin, H * W, 8, 8, None, False, ring.buf[t], ring.C)
                self.launches += 2
        x = self._layers(self.full, self.down, self.t_stride, stage, list(range(T)), H, W)
        # ---- projection: SiLU, (1,2,2)/(1,2,2) conv = space-to-depth + GEMM to the DiT width
        Tn, Hn, Wn, Cn = x.shape
        a = torch.zeros(Tn, Hn // 2, Wn // 2, self.kproj, device=dev, dtype=torch.bfloat16)
        if self.kproj == 4 * Cn:
            for t in range(Tn):
                nv.vae_space_to_depth_act(x[t], Hn, Wn, Cn, nv.ACT_SILU, a[t])
        else:
            tmp = torch.empty(Hn // 2, Wn // 2, 4 * Cn, device=dev, dtype=torch.bfloat16)
            for t in range(Tn):
                nv.vae_space_to_depth_act(x[t], Hn, Wn, Cn, nv.ACT_SILU, tmp)
                a[t, :, :, :4 * Cn] = tmp
        self.launches += Tn + 1
        L = Tn * (Hn // 2) * (Wn // 2)
        out = torch.empty(L, self.w_proj.shape[0], device=dev, dtype=torch.float32)
        nv.gemm(a.view(L, self.kproj), self.w_proj, out, bias=self.b_proj)
        return out.unsqueeze(0)


def pose_condition(engine, humanpose_data):
    """humanpose_data [3, T, H, W] in 0..255 -> [1, f*h*w, dim]: the first frame is repeated three more times in front
    and the values are scaled to 0..1 (reference svi_video_dance.py:526-528)."""
    x = humanpose_data.to(torch.float32)
    x = torch.cat([x[:, :1].repeat(1, 3, 1, 1), x], dim=1) / 255.0
    return engine.forward(x)


def make_randomref_embedding_pose(concat_dim=4, randomref_dim=20):
    """The reference-pose stem of UniAnimate-DiT (reference wan_video.py:543-558), keys `0.weight` ... `10.bias`."""
    c = concat_dim * 4
    return nn.Sequential(
        nn.Conv2d(3, c, 3, stride=1, padding=1), nn.SiLU(),
        nn.Conv2d(c, c, 3, stride=1, padding=1), nn.SiLU(),
        nn.Conv2d(c, c, 3, stride=1, padding=1), nn.SiLU(),
        nn.Conv2d(c, c, 3, stride=2, padding=1), nn.SiLU(),
        nn.Conv2d(c, c, 3, stride=2, padding=1), nn.SiLU(),
        nn.Conv2d(c, randomref_dim, 3, stride=2, padding=1))


class RandomRefEmbeddingEngine(_StemEngine):
    """The reference-pose stem on svi_conv3d_causal: one frame, kt = 1; the stride-2 convs as 2x2 convs over a
    space-to-depth input, SiLU fused into each conv's input staging."""

    def __init__(self, seq: nn.Sequential, device):
        super().__init__(device, "the reference-pose stem")
        convs = [m for m in seq if isinstance(m, nn.Conv2d)]
        if len(convs) != 6 or [m.stride[0] for m in convs] != [1, 1, 1, 2, 2, 2]:
            raise RuntimeError("randomref_embedding_pose must be the 6-conv stem of wan_video.py:544-558")
        self.full = [_Conv(m.weight, m.bias, self.device) for m in convs[:3]]
        self.down = [_Conv(m.weight, m.bias, self.device, s2d="before") for m in convs[3:]]
        self.out_channels = convs[-1].out_channels

    def forward(self, image):
        """image f32 [3, H, W] (already /255) -> f32 [1, out_channels, 1, H/8, W/8]."""
        dev = self.device
        C, H, W = image.shape
        if C != 3 or H % 8 or W % 8:
            raise RuntimeError(f"svi_b200: reference pose must be [3, H, W] with H, W multiples of 8, got {tuple(image.shape)}")
        image = image.to(device=dev, dtype=torch.float32).contiguous()
        ring = _Ring(1, H, W, self.full[0].c_in, dev, history=0)
        xin = torch.empty(H, W, 8, device=dev, dtype=torch.float32)
        nv.vae_from_planar(image, 3, H * W, None, None, xin, 8, False)
        nv.vae_norm_act(xin, H * W, 8, 8, None, False, ring.buf[0], ring.C)
        self.launches += 2
        x = self._conv(self.full[0], ring, [0], 1, 1, H, W)
        for cv in self.full[1:]:
            nv.vae_norm_act(x[0], H * W, x.shape[-1], x[0].stride(1), None, True, ring.buf[0], ring.C)   # SiLU -> bf16
            self.launches += 1
            x = self._conv(cv, ring, [0], 1, 1, H, W)
        for cv in self.down:
            _, Hn, Wn, Cn = x.shape
            ring = _Ring(1, Hn // 2, Wn // 2, 4 * Cn, dev, history=0)
            nv.vae_space_to_depth_act(x[0], Hn, Wn, Cn, nv.ACT_SILU, ring.buf[0])
            self.launches += 1
            x = self._conv(cv, ring, [0], 1, 1, Hn // 2, Wn // 2)
        return x[..., :self.out_channels].permute(3, 0, 1, 2).unsqueeze(0).contiguous()


def make_learn_in_embedding(concat_dim=4):
    """The masked-video stem of UniAnimate-DiT Replace-Anyone (reference wan_video.py:1353-1361), keys `0.weight` ...
    `6.bias`."""
    c = concat_dim * 4
    return nn.Sequential(
        nn.Conv3d(4, c, (3, 3, 3), stride=(1, 1, 1), padding=(1, 1, 1)), nn.SiLU(),
        nn.Conv3d(c, c, (3, 3, 3), stride=(1, 2, 2), padding=(1, 1, 1)), nn.SiLU(),
        nn.Conv3d(c, c, 3, stride=(2, 2, 2), padding=1), nn.SiLU(),
        nn.Conv3d(c, 16, 3, stride=2, padding=1))


def make_inpaint_embedding(concat_dim=4):
    """The masked-latent stem of UniAnimate-DiT Replace-Anyone (reference wan_video.py:1363-1369), keys `0.weight` ...
    `4.bias`."""
    c = concat_dim * 4
    return nn.Sequential(
        nn.Conv3d(16, c, (3, 3, 3), stride=(1, 1, 1), padding=(1, 1, 1)), nn.SiLU(),
        nn.Conv3d(c, c, 3, stride=(1, 1, 1), padding=1), nn.SiLU(),
        nn.Conv3d(c, 16, 3, stride=1, padding=1))


def _convs3d(seq, strides, what):
    convs = [m for m in seq if isinstance(m, nn.Conv3d)]
    if [tuple(m.stride) for m in convs] != strides or any(tuple(m.kernel_size) != (3, 3, 3) for m in convs):
        raise RuntimeError(f"{what} must be the {len(strides)}-conv stem of wan_video.py:1353-1369")
    return convs


class LearnInEmbeddingEngine(_StemEngine):
    """The masked-video stem.  Its first ring is written by svi_replace_mask_stage straight from the video and the
    segmentation; the three leading repeats of frame 0 are slot-table entries, not copies."""

    def __init__(self, seq: nn.Sequential, device):
        super().__init__(device, "the learn-in stem")
        convs = _convs3d(seq, [(1, 1, 1), (1, 2, 2), (2, 2, 2), (2, 2, 2)], "learn_in_embedding")
        self.full = [_Conv(convs[0].weight, convs[0].bias, self.device)]
        self.down = [_Conv(m.weight, m.bias, self.device, s2d="before") for m in convs[1:]]
        self.t_stride = [m.stride[0] for m in convs[1:]]
        self.out_channels = convs[-1].out_channels

    def forward(self, video, seg, masked=None):
        """video f32 [3, T, H, W], seg uint8 or f32 [T, H, W] (on the device, contiguous) -> f32
        [1, 16, f, H/8, W/8] of cat([m[:, :1] x3, m]) with m = cat([video * keep, keep]), keep = !(seg / 255 > 0).
        `masked` (f32 [3, T, H, W] or None) receives video * keep, the VAE encoder's input."""
        C, T, H, W = video.shape
        if C != 3 or H % 8 or W % 8:
            raise RuntimeError(f"svi_b200: the learn-in stem needs a [3, T, H, W] video with H, W multiples of 8, "
                               f"got {tuple(video.shape)}")

        def stage(ring):
            nv.replace_mask_stage(video, seg, masked, ring.buf[:T])
            self.launches += 1
        x = self._layers(self.full, self.down, self.t_stride, stage, [0, 0, 0] + list(range(T)), H, W)
        return x[..., :self.out_channels].permute(3, 0, 1, 2).unsqueeze(0).contiguous()


class InpaintEmbeddingEngine(_StemEngine):
    """The masked-latent stem: the f32 planar latents staged to the bf16 ring by svi_vae_from_planar, three stride-1
    convs."""

    def __init__(self, seq: nn.Sequential, device):
        super().__init__(device, "the inpaint stem")
        convs = _convs3d(seq, [(1, 1, 1)] * 3, "inpaint_embedding")
        self.full = [_Conv(m.weight, m.bias, self.device) for m in convs]
        self.in_channels, self.out_channels = convs[0].in_channels, convs[-1].out_channels

    def forward(self, latents):
        """latents f32 [1, C, f, h, w] -> f32 [1, out_channels, f, h, w]."""
        dev = self.device
        lat = latents.to(device=dev, dtype=torch.float32).contiguous()
        _, C, F, h, w = lat.shape
        if C != self.in_channels:
            raise RuntimeError(f"svi_b200: the inpaint stem needs {self.in_channels}-channel latents, got {tuple(lat.shape)}")

        def stage(ring):
            for t in range(F):
                nv.vae_from_planar(lat[0, :, t], C, h * w, None, None, ring.buf[t], ring.C, True, ldc=F * h * w)
                self.launches += 1
        x = self._layers(self.full, [], [], stage, list(range(F)), h, w)
        return x[..., :self.out_channels].permute(3, 0, 1, 2).unsqueeze(0).contiguous()
