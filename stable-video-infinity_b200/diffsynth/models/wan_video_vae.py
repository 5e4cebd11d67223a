"""Wan 3-D causal VAE — host side of the H100-native encode/decode at the clip boundaries.

Module / parameter names follow the reference (``diffsynth/models/wan_video_vae.py``: ``WanVideoVAE`` :599-789,
``VideoVAE_`` :492-596, ``Encoder3d`` :276-376, ``Decoder3d`` :379-481, ``ResidualBlock`` :198-232,
``Resample`` :82-174, ``AttentionBlock`` :235-273, ``CausalConv3d`` :33-52, ``RMS_norm`` :55-70), so Wan VAE
checkpoints load unchanged; the nn.Modules only hold parameters.  ``WanVAEEngine`` runs the arithmetic:

* activations are channels-last; conv inputs are bf16 *frame rings* ``[slots][H][W][C]`` that keep the last two
  input frames of every causal conv in place (the reference clones / concatenates / pads its feature cache on
  every call, :44-52, :214-232);
* every conv (3x3x3 causal, 3x3 spatial, (3,1,1) temporal, 1x1x1) is one launch of the wgmma implicit-GEMM
  kernel ``svi_conv3d_causal`` with bias / residual / channel->frame split fused in its epilogue;
* RMS-norm + SiLU run fused with the fp32 -> bf16 staging of the next conv's input (``svi_vae_norm_act``);
  nearest upsampling and the stride-2 space-to-depth are fused with that staging too;
* the stride-2 Conv2d of ``downsample`` is computed as a 2x2 conv on the space-to-depth input with re-packed
  weights (same arithmetic, zero weights for the 7 unused (tap, phase) pairs);
* the per-frame attention block is 4 GEMM launches + a row softmax (0.4 % of the VAE FLOPs).

The streaming semantics (which conv has which history on which chunk) are those derived and pinned in
``oracle/wan_vae_oracle.py``.  Precision: bf16 conv operands, fp32 accumulation, fp32 activations and norms
(the reference runs the VAE in fp32, svi_video.py:378,386; parity is reported in uint8 levels, DESIGN.md).
"""
import torch
import torch.nn as nn

from .. import _native as nv

CACHE_T = 2


class CausalConv3d(nn.Conv3d):
    """Parameter container (weight [O, I, kt, kh, kw], bias); arithmetic in WanVAEEngine."""


class RMS_norm(nn.Module):
    def __init__(self, dim, channel_first=True, images=True, bias=False):
        super().__init__()
        shape = (dim, 1, 1) if images else (dim, 1, 1, 1)
        self.scale = dim ** 0.5
        self.gamma = nn.Parameter(torch.ones(shape))


class Upsample(nn.Upsample):
    pass


class Resample(nn.Module):
    def __init__(self, dim, mode):
        assert mode in ("none", "upsample2d", "upsample3d", "downsample2d", "downsample3d")
        super().__init__()
        self.dim, self.mode = dim, mode
        if mode in ("upsample2d", "upsample3d"):
            self.resample = nn.Sequential(Upsample(scale_factor=(2.0, 2.0), mode="nearest-exact"),
                                          nn.Conv2d(dim, dim // 2, 3, padding=1))
            if mode == "upsample3d":
                self.time_conv = CausalConv3d(dim, dim * 2, (3, 1, 1), padding=(1, 0, 0))
        elif mode in ("downsample2d", "downsample3d"):
            self.resample = nn.Sequential(nn.ZeroPad2d((0, 1, 0, 1)), nn.Conv2d(dim, dim, 3, stride=(2, 2)))
            if mode == "downsample3d":
                self.time_conv = CausalConv3d(dim, dim, (3, 1, 1), stride=(2, 1, 1), padding=(0, 0, 0))
        else:
            self.resample = nn.Identity()


class ResidualBlock(nn.Module):
    def __init__(self, in_dim, out_dim, dropout=0.0):
        super().__init__()
        self.in_dim, self.out_dim = in_dim, out_dim
        self.residual = nn.Sequential(RMS_norm(in_dim, images=False), nn.SiLU(), CausalConv3d(in_dim, out_dim, 3, padding=1),
                                      RMS_norm(out_dim, images=False), nn.SiLU(), nn.Dropout(dropout),
                                      CausalConv3d(out_dim, out_dim, 3, padding=1))
        self.shortcut = CausalConv3d(in_dim, out_dim, 1) if in_dim != out_dim else nn.Identity()


class AttentionBlock(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.dim = dim
        self.norm = RMS_norm(dim)
        self.to_qkv = nn.Conv2d(dim, dim * 3, 1)
        self.proj = nn.Conv2d(dim, dim, 1)
        nn.init.zeros_(self.proj.weight)


class Encoder3d(nn.Module):
    def __init__(self, dim=128, z_dim=4, dim_mult=[1, 2, 4, 4], num_res_blocks=2, attn_scales=[],
                 temperal_downsample=[True, True, False], dropout=0.0):
        super().__init__()
        dims = [dim * u for u in [1] + dim_mult]
        self.conv1 = CausalConv3d(3, dims[0], 3, padding=1)
        layers = []
        for i, (in_dim, out_dim) in enumerate(zip(dims[:-1], dims[1:])):
            for _ in range(num_res_blocks):
                layers.append(ResidualBlock(in_dim, out_dim, dropout))
                in_dim = out_dim
            if i != len(dim_mult) - 1:
                layers.append(Resample(out_dim, mode="downsample3d" if temperal_downsample[i] else "downsample2d"))
        self.downsamples = nn.Sequential(*layers)
        self.middle = nn.Sequential(ResidualBlock(out_dim, out_dim, dropout), AttentionBlock(out_dim),
                                    ResidualBlock(out_dim, out_dim, dropout))
        self.head = nn.Sequential(RMS_norm(out_dim, images=False), nn.SiLU(), CausalConv3d(out_dim, z_dim, 3, padding=1))


class Decoder3d(nn.Module):
    def __init__(self, dim=128, z_dim=4, dim_mult=[1, 2, 4, 4], num_res_blocks=2, attn_scales=[],
                 temperal_upsample=[False, True, True], dropout=0.0):
        super().__init__()
        dims = [dim * u for u in [dim_mult[-1]] + dim_mult[::-1]]
        self.conv1 = CausalConv3d(z_dim, dims[0], 3, padding=1)
        self.middle = nn.Sequential(ResidualBlock(dims[0], dims[0], dropout), AttentionBlock(dims[0]),
                                    ResidualBlock(dims[0], dims[0], dropout))
        layers = []
        for i, (in_dim, out_dim) in enumerate(zip(dims[:-1], dims[1:])):
            if i in (1, 2, 3):
                in_dim = in_dim // 2
            for _ in range(num_res_blocks + 1):
                layers.append(ResidualBlock(in_dim, out_dim, dropout))
                in_dim = out_dim
            if i != len(dim_mult) - 1:
                layers.append(Resample(out_dim, mode="upsample3d" if temperal_upsample[i] else "upsample2d"))
        self.upsamples = nn.Sequential(*layers)
        self.head = nn.Sequential(RMS_norm(out_dim, images=False), nn.SiLU(), CausalConv3d(out_dim, 3, 3, padding=1))


class VideoVAE_(nn.Module):
    def __init__(self, dim=96, z_dim=16, dim_mult=[1, 2, 4, 4], num_res_blocks=2, attn_scales=[],
                 temperal_downsample=[False, True, True], dropout=0.0):
        super().__init__()
        self.dim, self.z_dim = dim, z_dim
        self.encoder = Encoder3d(dim, z_dim * 2, dim_mult, num_res_blocks, attn_scales, temperal_downsample, dropout)
        self.conv1 = CausalConv3d(z_dim * 2, z_dim * 2, 1)
        self.conv2 = CausalConv3d(z_dim, z_dim, 1)
        self.decoder = Decoder3d(dim, z_dim, dim_mult, num_res_blocks, attn_scales, temperal_downsample[::-1], dropout)


# ---------------------------------------------------------------------------------------------------------
# engine
# ---------------------------------------------------------------------------------------------------------
def _ceil(a, b):
    return (a + b - 1) // b * b


def _pick_tile_w(H, W):
    best, best_cost = 16, None
    for bw in (8, 16, 32, 64, 128):
        bh = 128 // bw
        cost = _ceil(H, bh) * _ceil(W, bw)
        if best_cost is None or cost < best_cost:
            best, best_cost = bw, cost
    return best


class _Conv:
    """Packed conv: bf16 weight [rows, taps*cpad], f32 bias, geometry."""

    def __init__(self, weight, bias, device, s2d=False):
        w = weight.detach().to(device=device, dtype=torch.float32)
        if w.dim() == 4:                       # Conv2d -> kt = 1
            w = w.unsqueeze(2)
        O, I, kt, kh, kw = w.shape
        if s2d:
            # stride-2 3x3 conv == 2x2 conv over the space-to-depth input [H/2,W/2,4I]; tap (bh,bw), phase (dy,dx) takes the
            # original tap (a,b) when it exists, else a zero weight:
            #   s2d=True / "after":  ZeroPad2d((0,1,0,1)) + stride 2 (the VAE's Resample): output o reads pixels 2o..2o+2 =
            #                        blocks o, o+1                    -> a = 2bh+dy,   conv pad 0
            #   s2d="before":        padding 1 + stride 2 (nn.Conv3d(..., stride 2, padding 1)): pixels 2o-1..2o+1 =
            #                        blocks o-1, o                    -> a = 2bh+dy-1, conv pad 1 (block -1 is zero fill)
            off = 1 if s2d == "before" else 0
            w2 = torch.zeros(O, 4 * I, kt, 2, 2, device=device)
            for bh in range(2):
                for bw in range(2):
                    for dy in range(2):
                        for dx in range(2):
                            a, b = 2 * bh + dy - off, 2 * bw + dx - off
                            if 0 <= a <= 2 and 0 <= b <= 2:
                                w2[:, (dy * 2 + dx) * I:(dy * 2 + dx + 1) * I, :, bh, bw] = w[:, :, :, a, b]
            w, (O, I, kt, kh, kw) = w2, w2.shape
        self.c_in_true = I
        self.c_in = max(64, _ceil(I, 8))        # ring channel count (tiny inputs are zero-padded to one full chunk)
        self.cpad = _ceil(self.c_in, 64)
        self.kt, self.kh, self.kw = kt, kh, kw
        self.c_out_true = O
        self.c_out = _ceil(O, 4)
        rows = _ceil(self.c_out, 16)
        packed = torch.zeros(rows, kt, kh, kw, self.cpad, device=device)
        packed[:O, :, :, :, :I] = w.permute(0, 2, 3, 4, 1)
        self.w = packed.reshape(rows, kt * kh * kw * self.cpad).to(torch.bfloat16).contiguous()
        b = torch.zeros(rows, device=device)
        if bias is not None:
            b[:O] = bias.detach().to(device=device, dtype=torch.float32)
        self.b = b


class _Ring:
    """bf16 frame ring [slots + 1, halo + H + halo, W, C]; the last slot is all zeros (empty history).  halo = 1 under
    spatial sharding (rings of convs with a vertical extent): row 0 / row H+1 of a frame hold the neighbour ranks' border
    rows (exchanged when the frame is produced; zero at the image border), rows 1..H are this rank's rows."""

    def __init__(self, slots, H, W, C, device, history, halo=0):
        self.buf = torch.zeros(slots + 1, H + 2 * halo, W, C, device=device, dtype=torch.bfloat16)
        self.slots, self.H, self.W, self.C, self.halo = slots, H, W, C, halo
        self.next, self.history = 0, history
        self.hist = [slots] * history           # slot ids of the most recent frames (oldest first)

    def frame(self, slot):
        """The rank's own rows of a slot: bf16 [H, W, C] (contiguous)."""
        return self.buf[slot, self.halo:self.halo + self.H]

    def rewind(self):
        """Start of a new video: empty history again.  The buffer is NOT cleared — every slot is written in full before it
        is referenced, the padding channels and the outer halo rows are never written (they stay zero from the allocation),
        and the history points at the all-zero slot until real frames exist."""
        self.next = 0
        self.hist = [self.slots] * self.history

    def push(self, n):
        ids = [(self.next + i) % self.slots for i in range(n)]
        self.next = (self.next + n) % self.slots
        return ids


class WanVAEEngine:
    def __init__(self, vae: "WanVideoVAE", device):
        nv.require_cuda(device, "the Wan VAE")
        self.device = torch.device(device)
        self.sig = vae._param_signature()
        m = vae.model
        self.convs, self.gammas, self.attn = {}, {}, {}
        dev = self.device
        for name, mod in m.named_modules():
            if isinstance(mod, Resample):
                if mod.mode.startswith("downsample"):
                    self.convs[name + ".resample.1"] = _Conv(mod.resample[1].weight, mod.resample[1].bias, dev, s2d=True)
                elif mod.mode.startswith("upsample"):
                    self.convs[name + ".resample.1"] = _Conv(mod.resample[1].weight, mod.resample[1].bias, dev)
                if hasattr(mod, "time_conv"):
                    self.convs[name + ".time_conv"] = _Conv(mod.time_conv.weight, mod.time_conv.bias, dev)
            elif isinstance(mod, CausalConv3d) and not name.endswith("time_conv"):
                self.convs[name] = _Conv(mod.weight, mod.bias, dev)
            elif isinstance(mod, RMS_norm):
                self.gammas[name] = mod.gamma.detach().to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
            elif isinstance(mod, AttentionBlock):
                c = mod.dim
                wq = mod.to_qkv.weight.detach().to(dev, torch.float32).reshape(3 * c, c)
                bq = mod.to_qkv.bias.detach().to(dev, torch.float32)
                self.attn[name] = dict(
                    w_qk=wq[:2 * c].to(torch.bfloat16).contiguous(), b_qk=bq[:2 * c].contiguous(),
                    w_v=wq[2 * c:].to(torch.bfloat16).contiguous(), b_v=bq[2 * c:].contiguous(),
                    w_p=mod.proj.weight.detach().to(dev, torch.float32).reshape(c, c).to(torch.bfloat16).contiguous(),
                    b_p=mod.proj.bias.detach().to(dev, torch.float32).contiguous())
        # 1x1x1 convs outside encoder/decoder run on the GEMM kernel
        self.w_conv1 = m.conv1.weight.detach().to(dev, torch.float32).reshape(32, 32)[:16].to(torch.bfloat16).contiguous()
        self.b_conv1 = m.conv1.bias.detach().to(dev, torch.float32)[:16].contiguous()
        self.w_conv2 = m.conv2.weight.detach().to(dev, torch.float32).reshape(16, 16).to(torch.bfloat16).contiguous()
        self.b_conv2 = m.conv2.bias.detach().to(dev, torch.float32).contiguous()
        self.mean = vae.mean.to(dev, torch.float32).contiguous()
        self.std = vae.std.to(dev, torch.float32).contiguous()
        self.inv_std = (1.0 / vae.std).to(dev, torch.float32).contiguous()
        self.neg_mean = (-vae.mean).to(dev, torch.float32).contiguous()
        self.launches = 0
        self.rings = {}
        self.chunk = 0
        self.shard = None        # SpatialShard: this rank computes a band of image rows, halos exchanged per conv
        self.halo_exchanges = 0

    # ------------------------------------------------------------------ low-level helpers
    def reset(self):
        # rings are kept across videos of the same geometry (re-allocating and zero-filling them every video costs a pass
        # over every ring); _ring() replaces one whose geometry changed
        for r in self.rings.values():
            r.rewind()
        self.chunk = 0

    def _ring(self, key, slots, H, W, C, history, halo=0):
        r = self.rings.get(key)
        if r is None or (r.H, r.W, r.C, r.slots, r.halo) != (H, W, C, slots, halo):
            r = _Ring(slots, H, W, C, self.device, history, halo)
            self.rings[key] = r
        return r

    def _halo(self, cv):
        """1 when the conv reads rows above / below its output row and the image is split over ranks."""
        return 1 if (self.shard is not None and cv.kh > 1) else 0

    def _exchange_halo(self, ring, ids):
        """Spatial sharding: the frames just produced in `ids` get their border rows from the neighbour ranks (and send
        theirs): one NCCL send/recv group per conv input.  Replaces nothing in the reference (its VAE is single-GPU; its
        tiled mode blends overlapping tiles, wan_video_vae.py:643-744) — SURVEY.md section 8e."""
        sh = self.shard
        if sh is None or not ring.halo:
            return
        import torch.distributed as dist
        ops = []
        H = ring.H
        for slot in ids:
            fr = ring.buf[slot]
            if sh.up is not None:
                ops += [dist.P2POp(dist.isend, fr[1], sh.up, sh.group), dist.P2POp(dist.irecv, fr[0], sh.up, sh.group)]
            if sh.down is not None:
                ops += [dist.P2POp(dist.isend, fr[H], sh.down, sh.group), dist.P2POp(dist.irecv, fr[H + 1], sh.down, sh.group)]
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()
            self.halo_exchanges += 1

    def _launch_conv(self, cv, ring, slot_table, T, H, W, out, out_frame_stride, out_ld, pad, residual=None, n_split=0,
                     split_offset=0, nxt=None, write_f32=True):
        d = nv.ConvDesc()
        d.x_ring = ring.buf.data_ptr()
        d.ring_slots, d.in_H, d.in_W, d.C_in = ring.slots + 1, ring.H + 2 * ring.halo, ring.W, ring.C
        d.w_packed, d.w_rows, d.w_ld = cv.w.data_ptr(), cv.w.shape[0], cv.w.shape[1]
        # with a halo row on top, ring row = image row + 1: the vertical padding shrinks by the halo (may become -1)
        d.kt, d.kh, d.kw, d.pad_h, d.pad_w = cv.kt, cv.kh, cv.kw, pad - ring.halo, pad
        d.H, d.W, d.T = H, W, T
        for t in range(T):
            for a in range(cv.kt):
                d.slot[t * 3 + a] = slot_table[t][a]
        d.C_out = cv.c_out
        d.tile_w = _pick_tile_w(H, W)
        if out is not None:
            d.out, d.out_frame_stride, d.out_ld = out.data_ptr(), out_frame_stride, out_ld
        else:
            d.out_ld = cv.c_out
        d.n_split, d.split_offset = n_split, split_offset
        d.bias = cv.b.data_ptr()
        if residual is not None:
            d.residual, d.res_frame_stride, d.res_ld = residual.data_ptr(), residual.stride(0), residual.shape[-1]
        d.write_f32 = 1 if write_f32 else 0
        if nxt is not None:       # the epilogue also produces the next conv's input (RMS norm + SiLU + bf16 staging)
            (ncv, nring, nids), gamma, silu = nxt
            d.next_ring = nring.buf.data_ptr() + nring.halo * nring.buf.stride(1) * 2      # first own row of a slot
            d.next_frame_stride = nring.buf.stride(0)
            d.next_ld = nring.C
            for t in range(T):
                d.next_slot[t] = nids[t]
            d.next_gamma = None if gamma is None else gamma.data_ptr()
            d.next_silu = 1 if silu else 0
        nv.conv3d_causal(d)
        self.launches += 1

    def _stage(self, ring, slot, x_frame, gamma=None, silu=False):
        """fp32 channels-last frame [H,W,C] -> (RMS-norm, SiLU,) bf16 into a ring slot (zero-padded channels)."""
        H, W, C = x_frame.shape
        nv.vae_norm_act(x_frame, H * W, C, x_frame.stride(1), gamma, silu, ring.frame(slot), ring.C)
        self.launches += 1

    # ------------------------------------------------------------------ layers (x: f32 [T,H,W,C] contiguous)
    FUSE_MAX_C = 256      # the fused producer needs the whole channel vector of a pixel in one accumulator tile

    def _conv_in(self, name, T, H, W):
        """Reserve T input slots in causal conv `name`'s frame ring: (conv, ring, slot ids).  Whoever fills them — the
        staging kernel or the previous conv's epilogue — the history bookkeeping happens in causal_conv."""
        cv = self.convs[name]
        ring = self._ring(name, 4 + CACHE_T, H, W, cv.c_in, history=CACHE_T, halo=self._halo(cv))
        return cv, ring, ring.push(T)

    def causal_conv(self, name, x, gamma=None, silu=False, residual=None, staged=None, nxt=None, write_f32=True, shape=None):
        """3x3x3 (or 3x1x1) causal conv over the frame stream with two frames of history kept in the ring.
        staged: (conv, ring, ids) from _conv_in whose slots the PREVIOUS conv's epilogue already filled (x is then unused);
        nxt: ((conv, ring, ids), gamma, silu) — this conv's epilogue fills the next conv's slots; write_f32=False drops
        the fp32 output (returns None)."""
        if staged is None:
            T, H, W, C = x.shape
            cv, ring, ids = self._conv_in(name, T, H, W)
            for t in range(T):
                self._stage(ring, ids[t], x[t], gamma, silu)
        else:
            cv, ring, ids = staged
            T, H, W = shape
        self._exchange_halo(ring, ids)
        seq = ring.hist + ids
        table = [[seq[t + a] for a in range(cv.kt)] for t in range(T)] if cv.kt == 3 else [[ids[t]] for t in range(T)]
        ring.hist = seq[-CACHE_T:]
        out = torch.empty(T, H, W, cv.c_out, device=self.device, dtype=torch.float32) if write_f32 else None
        self._launch_conv(cv, ring, table, T, H, W, out, 0 if out is None else out.stride(0), cv.c_out, pad=(cv.kh - 1) // 2,
                          residual=residual, nxt=nxt, write_f32=write_f32)
        return out

    def pointwise_conv(self, name, x):
        """1x1x1 shortcut conv on the raw (un-normalised) activations."""
        cv = self.convs[name]
        T, H, W, C = x.shape
        ring = self._ring(name, 4, H, W, cv.c_in, history=0)
        ids = ring.push(T)
        for t in range(T):
            self._stage(ring, ids[t], x[t])
        out = torch.empty(T, H, W, cv.c_out, device=self.device, dtype=torch.float32)
        self._launch_conv(cv, ring, [[i] for i in ids], T, H, W, out, out.stride(0), cv.c_out, pad=0)
        return out

    def residual_block(self, name, x, staged=None, next_res=None):
        """reference ResidualBlock.forward :213-232.  The activation between the block's two convs exists only as the
        normalised bf16 input of the second conv (written by the first conv's epilogue) when the width allows it; with
        `next_res` (name of a ResidualBlock that consumes this block's output next) the second conv's epilogue also fills
        the next block's first conv input.  Returns (x_out f32, staged input of next_res or None)."""
        T, H, W, _ = x.shape
        h = self.pointwise_conv(name + ".shortcut", x) if (name + ".shortcut") in self.convs else x
        c_mid = self.convs[name + ".residual.2"].c_out_true
        c_out = self.convs[name + ".residual.6"].c_out_true
        s6 = self._conv_in(name + ".residual.6", T, H, W) if c_mid <= self.FUSE_MAX_C else None
        y = self.causal_conv(name + ".residual.2", x, self.gammas[name + ".residual.0"], True, staged=staged, shape=(T, H, W),
                             nxt=None if s6 is None else (s6, self.gammas[name + ".residual.3"], True), write_f32=s6 is None)
        sn = None
        if next_res is not None and c_out <= self.FUSE_MAX_C and self.convs[next_res + ".residual.2"].c_in_true == c_out:
            sn = self._conv_in(next_res + ".residual.2", T, H, W)
        out = self.causal_conv(name + ".residual.6", y, self.gammas[name + ".residual.3"], True, residual=h, staged=s6,
                               shape=(T, H, W), nxt=None if sn is None else (sn, self.gammas[next_res + ".residual.0"], True))
        return out, sn

    def attention_block(self, name, x):
        """reference AttentionBlock.forward :254-273: per-frame single-head attention, 4 GEMMs + row softmax.  Under spatial
        sharding the normalised tokens of all ranks are gathered (K and V need every token; they are 0.4 % of the VAE FLOPs
        and are recomputed on every rank) and the rank attends with the queries of its own rows."""
        a = self.attn[name]
        T, H, W, C = x.shape
        N = H * W
        dev = self.device
        sh = self.shard
        Nk = N if sh is None else sh.total_rows(H) * W            # keys: all tokens of the frame
        Np, Nkp = _ceil(N, 8), _ceil(Nk, 8)
        out = torch.empty_like(x)
        # token count padded to a multiple of 8 (GEMM N / K granularity); pad rows / columns stay zero
        xn = torch.zeros(Np, C, device=dev, dtype=torch.bfloat16)
        xk = xn if sh is None else torch.zeros(Nkp, C, device=dev, dtype=torch.bfloat16)
        q = torch.zeros(Np, C, device=dev, dtype=torch.bfloat16)
        kk = torch.zeros(Nkp, C, device=dev, dtype=torch.bfloat16)
        vT = torch.empty(C, Nkp, device=dev, dtype=torch.bfloat16)
        S = torch.empty(N, Nkp, device=dev, dtype=torch.float32)
        P = torch.empty(N, Nkp, device=dev, dtype=torch.bfloat16)
        O = torch.empty(N, C, device=dev, dtype=torch.bfloat16)
        for t in range(T):
            xt = x[t].reshape(N, C)
            nv.vae_norm_act(xt, N, C, C, self.gammas[name + ".norm"], False, xn, C)
            if sh is not None:
                sh.gather_rows(xn[:N], xk, H, W)
            nv.gemm(xn[:N], a["w_qk"][:C], q[:N], bias=a["b_qk"][:C])
            nv.gemm(xk[:Nk], a["w_qk"][C:], kk[:Nk], bias=a["b_qk"][C:])
            nv.gemm(a["w_v"], xk, vT)                              # V^T without bias (rows of P sum to 1: folded below)
            nv.gemm(q[:N], kk, S)                                  # columns >= Nk are ignored by the softmax
            nv.softmax_rows(S, Nk, C ** -0.5, P)
            nv.gemm(P, vT, O, bias=a["b_v"])
            nv.gemm(O, a["w_p"], out[t].reshape(N, C), bias=a["b_p"], residual=xt)
            self.launches += 8
        return out

    def upsample(self, name, x, temporal):
        """reference Resample.forward upsample2d/3d :119-160."""
        T, H, W, C = x.shape
        if temporal and self.chunk > 0:
            cv = self.convs[name + ".time_conv"]
            ring = self._ring(name + ".time_conv", 4 + CACHE_T, H, W, cv.c_in, history=CACHE_T)
            ids = ring.push(T)
            for t in range(T):
                self._stage(ring, ids[t], x[t])
            seq = ring.hist + ids
            ring.hist = seq[-CACHE_T:]
            y = torch.empty(2 * T, H, W, C, device=self.device, dtype=torch.float32)
            # output frame t -> frames (2t, 2t+1): channels [0,C) | [C,2C)
            self._launch_conv(cv, ring, [[seq[t + a] for a in range(3)] for t in range(T)], T, H, W, y, 2 * y.stride(0), C,
                              pad=0, n_split=C, split_offset=y.stride(0))
            x, T = y, 2 * T
        cv = self.convs[name + ".resample.1"]
        ring = self._ring(name + ".resample.1", 4, 2 * H, 2 * W, C, history=0, halo=self._halo(cv))
        ids = ring.push(T)
        for t in range(T):
            nv.vae_upsample2x(x[t], H, W, C, ring.frame(ids[t]))
            self.launches += 1
        self._exchange_halo(ring, ids)
        out = torch.empty(T, 2 * H, 2 * W, cv.c_out, device=self.device, dtype=torch.float32)
        self._launch_conv(cv, ring, [[i] for i in ids], T, 2 * H, 2 * W, out, out.stride(0), cv.c_out, pad=1)
        return out

    def downsample(self, name, x, temporal):
        """reference Resample.forward downsample2d/3d :157-173."""
        T, H, W, C = x.shape
        cv = self.convs[name + ".resample.1"]
        ring = self._ring(name + ".resample.1", 4, H // 2, W // 2, 4 * C, history=0, halo=self._halo(cv))
        ids = ring.push(T)
        for t in range(T):
            nv.vae_space_to_depth(x[t], H, W, C, ring.frame(ids[t]))
            self.launches += 1
        self._exchange_halo(ring, ids)        # the 2x2 conv over the blocks reads block row o + 1: the lower neighbour's first
        y = torch.empty(T, H // 2, W // 2, cv.c_out, device=self.device, dtype=torch.float32)
        self._launch_conv(cv, ring, [[i] for i in ids], T, H // 2, W // 2, y, y.stride(0), cv.c_out, pad=0)
        if not temporal:
            return y
        cv = self.convs[name + ".time_conv"]
        H2, W2 = H // 2, W // 2
        ring = self._ring(name + ".time_conv", 4 + 1, H2, W2, cv.c_in, history=1)
        ids = ring.push(T)
        for t in range(T):
            self._stage(ring, ids[t], y[t])
        first = self.chunk == 0
        seq = ring.hist + ids
        ring.hist = ids[-1:]
        if first:                                   # time_conv skipped on the first chunk (:166-168)
            return y
        To = (len(seq) - 3) // 2 + 1
        out = torch.empty(To, H2, W2, cv.c_out, device=self.device, dtype=torch.float32)
        self._launch_conv(cv, ring, [[seq[2 * t + a] for a in range(3)] for t in range(To)], To, H2, W2, out, out.stride(0),
                          cv.c_out, pad=0)
        return out

    # ------------------------------------------------------------------ encoder / decoder chunks
    ENC_PLAN = [("res", 0), ("res", 1), ("down", 2, False), ("res", 3), ("res", 4), ("down", 5, True),
                ("res", 6), ("res", 7), ("down", 8, True), ("res", 9), ("res", 10)]
    DEC_PLAN = [("res", 0), ("res", 1), ("res", 2), ("up", 3, True), ("res", 4), ("res", 5), ("res", 6), ("up", 7, True),
                ("res", 8), ("res", 9), ("res", 10), ("up", 11, False), ("res", 12), ("res", 13), ("res", 14)]

    def _run_plan(self, prefix, plan, x):
        """Walk a level plan; consecutive ResidualBlocks hand their activations over through the conv epilogues."""
        staged = None
        for k, item in enumerate(plan):
            n = f"{prefix}.{item[1]}"
            if item[0] == "res":
                nxt = plan[k + 1] if k + 1 < len(plan) else None
                x, staged = self.residual_block(n, x, staged, f"{prefix}.{nxt[1]}" if nxt is not None and nxt[0] == "res" else None)
            elif item[0] == "down":
                x, staged = self.downsample(n, x, item[2]), None
            else:
                x, staged = self.upsample(n, x, item[2]), None
        return x

    def encoder_chunk(self, x):
        """x f32 [T,H,W,8] (3 image channels + zero padding) -> f32 [T',H/8,W/8,32]."""
        p = "encoder"
        x = self.causal_conv(p + ".conv1", x)
        x = self._run_plan(p + ".downsamples", self.ENC_PLAN, x)
        x, _ = self.residual_block(p + ".middle.0", x)
        x = self.attention_block(p + ".middle.1", x)
        x, _ = self.residual_block(p + ".middle.2", x)
        x = self.causal_conv(p + ".head.2", x, self.gammas[p + ".head.0"], True)
        self.chunk += 1
        return x

    def decoder_chunk(self, x):
        """x f32 [1,h,w,16] -> f32 [1 or 4, 8h, 8w, 4] (3 image channels + 1 padding)."""
        p = "decoder"
        x = self.causal_conv(p + ".conv1", x)
        x, _ = self.residual_block(p + ".middle.0", x)
        x = self.attention_block(p + ".middle.1", x)
        x, _ = self.residual_block(p + ".middle.2", x)
        x = self._run_plan(p + ".upsamples", self.DEC_PLAN, x)
        x = self.causal_conv(p + ".head.2", x, self.gammas[p + ".head.0"], True)
        self.chunk += 1
        return x

    # ------------------------------------------------------------------ public entry points
    def encode(self, video):
        """video f32 [3,T,H,W] in [-1,1] (T = 4k+1, H,W % 8 == 0) -> latents f32 [16,k+1,H/8,W/8] (reference :525-550).
        With a SpatialShard every rank encodes its band of rows and the latent bands are gathered on every rank."""
        self.reset()
        C, T, H, W = video.shape
        sh = self.shard
        if sh is not None:
            r0, r1 = sh.band(H // 8)
            video = video[:, :, 8 * r0:8 * r1]
            H = 8 * (r1 - r0)
        video = video.to(device=self.device, dtype=torch.float32).contiguous()
        n_lat = 1 + (T - 1) // 4
        feats = torch.empty(n_lat, H // 8, W // 8, 32, device=self.device, dtype=torch.float32)
        bounds = [(0, 1)] + [(1 + 4 * (i - 1), 1 + 4 * i) for i in range(1, n_lat)]
        for i, (a, b) in enumerate(bounds):
            xin = torch.empty(b - a, H, W, 8, device=self.device, dtype=torch.float32)
            for t in range(a, b):
                nv.vae_from_planar(video[:, t], 3, H * W, None, None, xin[t - a], 8, False, ldc=T * H * W)
                self.launches += 1
            feats[i] = self.encoder_chunk(xin)[0]
        n_pix = n_lat * (H // 8) * (W // 8)
        fb = torch.empty(n_pix, 32, device=self.device, dtype=torch.bfloat16)
        nv.vae_norm_act(feats.reshape(n_pix, 32), n_pix, 32, 32, None, False, fb, 32)
        mu = torch.empty(n_pix, 16, device=self.device, dtype=torch.float32)
        nv.gemm(fb, self.w_conv1, mu, bias=self.b_conv1)
        out = torch.empty(16, n_lat, H // 8, W // 8, device=self.device, dtype=torch.float32)
        nv.vae_to_planar(mu, 16, 16, n_pix, self.neg_mean, self.inv_std, False, out)
        self.launches += 3
        return out if sh is None else sh.gather_bands(out, dim=2, scale=1)

    def decode(self, z):
        """z f32 [16,T,h,w] -> video f32 [3,4T-3,8h,8w] clamped to [-1,1] (reference :552-575, :753-756).
        With a SpatialShard every rank decodes its band of latent rows and the pixel bands are gathered on every rank."""
        self.reset()
        C, T, h, w = z.shape
        sh = self.shard
        if sh is not None:
            r0, r1 = sh.band(h)
            z = z[:, :, r0:r1]
            h = r1 - r0
        z = z.to(device=self.device, dtype=torch.float32).contiguous()
        n_pix = T * h * w
        zb = torch.empty(n_pix, 16, device=self.device, dtype=torch.bfloat16)
        nv.vae_from_planar(z, 16, n_pix, self.std, self.mean, zb, 16, True)        # z / (1/std) + mean
        x = torch.empty(n_pix, 16, device=self.device, dtype=torch.float32)
        nv.gemm(zb, self.w_conv2, x, bias=self.b_conv2)
        self.launches += 2
        x = x.reshape(T, h, w, 16)
        Tout = 4 * T - 3
        out = torch.empty(3, Tout, 8 * h, 8 * w, device=self.device, dtype=torch.float32)
        pos = 0
        for i in range(T):
            fr = self.decoder_chunk(x[i:i + 1])
            for t in range(fr.shape[0]):
                nv.vae_to_planar(fr[t].reshape(-1, fr.shape[-1]), fr.shape[-1], 3, 64 * h * w, None, None, True, out[:, pos],
                                 ldc=Tout * 64 * h * w)
                pos += 1
                self.launches += 1
        return out if sh is None else sh.gather_bands(out, dim=2, scale=8)


class SpatialShard:
    """Split of the image rows over the ranks of a process group for the VAE (SURVEY.md section 8e: the VAE is causal in time,
    so it shards in SPACE).  Latent row r belongs to rank `owner(r)`; every level of the encoder / decoder keeps that split
    (x2 / x4 / x8 rows).  Neighbouring bands exchange one border row per conv input (WanVAEEngine._exchange_halo)."""

    def __init__(self, group=None):
        import torch.distributed as dist
        self.group = group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self._latent_rows = None

    # global ranks of the neighbours inside the group (P2POp takes the global rank)
    def _global(self, r):
        import torch.distributed as dist
        return r if self.group is None else dist.get_global_rank(self.group, r)

    def band(self, latent_rows):
        """[r0, r1) latent rows of this rank; fixes the split for the whole encode / decode."""
        P = self.world
        if latent_rows < P:
            raise RuntimeError(f"svi_b200: cannot split {latent_rows} latent rows over {P} ranks")
        self._latent_rows = latent_rows
        self.bounds = [latent_rows * r // P for r in range(P + 1)]
        self.up = self._global(self.rank - 1) if self.rank > 0 else None
        self.down = self._global(self.rank + 1) if self.rank + 1 < P else None
        return self.bounds[self.rank], self.bounds[self.rank + 1]

    def total_rows(self, my_rows):
        """Rows of the whole image at the level where this rank holds `my_rows` rows."""
        mine = self.bounds[self.rank + 1] - self.bounds[self.rank]
        return self._latent_rows * (my_rows // mine)

    def gather_rows(self, local, full, H, W):
        """local bf16 [H*W, C] (this rank's tokens) -> full bf16 [>= total, C] holding every rank's tokens in row order."""
        import torch.distributed as dist
        mine = self.bounds[self.rank + 1] - self.bounds[self.rank]
        scale = H // mine
        C = local.shape[1]
        counts = [(self.bounds[r + 1] - self.bounds[r]) * scale * W for r in range(self.world)]
        mx = max(counts)
        pad = torch.zeros(mx, C, device=local.device, dtype=local.dtype)
        pad[:local.shape[0]] = local
        parts = torch.empty(self.world, mx, C, device=local.device, dtype=local.dtype)
        dist.all_gather_into_tensor(parts.view(self.world * mx, C), pad, group=self.group)     # concatenated form: NCCL and gloo
        off = 0
        for r in range(self.world):
            full[off:off + counts[r]] = parts[r, :counts[r]]
            off += counts[r]
        return full

    def gather_bands(self, t, dim, scale):
        """Concatenate every rank's band of `t` along `dim` (band heights = latent rows x scale) on every rank."""
        import torch.distributed as dist
        rows = [(self.bounds[r + 1] - self.bounds[r]) * scale for r in range(self.world)]
        mx = max(rows)
        shape = list(t.shape)
        shape[dim] = mx
        pad = torch.zeros(shape, device=t.device, dtype=t.dtype)
        pad.narrow(dim, 0, t.shape[dim]).copy_(t)
        parts = torch.empty([self.world] + shape, device=t.device, dtype=t.dtype)
        dist.all_gather_into_tensor(parts.view([self.world * shape[0]] + shape[1:]), pad.contiguous(), group=self.group)
        return torch.cat([parts[r].narrow(dim, 0, rows[r]) for r in range(self.world)], dim=dim)


class WanVideoVAE(nn.Module):
    """Reference WanVideoVAE (:599-789): encode(list of [3,T,H,W]) -> [B,16,(T+3)//4,H/8,W/8];
    decode([B,16,T,h,w]) -> [B,3,4T-3,8h,8w] in [-1,1]."""

    def __init__(self, z_dim=16):
        super().__init__()
        mean = [-0.7571, -0.7089, -0.9113, 0.1075, -0.1745, 0.9653, -0.1517, 1.5508,
                0.4134, -0.0715, 0.5517, -0.3632, -0.1922, -0.9497, 0.2503, -0.2921]
        std = [2.8184, 1.4541, 2.3275, 2.6558, 1.2196, 1.7708, 2.6052, 2.0743,
               3.2687, 2.1526, 2.8652, 1.5579, 1.6382, 1.1253, 2.8251, 1.9160]
        with torch.device("cpu"):      # constants, not parameters: must be real even when the loader constructs on "meta"
            self.mean = torch.tensor(mean)
            self.std = torch.tensor(std)
        self.scale = [self.mean, 1.0 / self.std]
        self.model = VideoVAE_(z_dim=z_dim).eval().requires_grad_(False)
        self.upsampling_factor = 8
        self._engine = None

    def _param_signature(self):
        s = 0
        for p in self.parameters():
            s = (s * 1000003 + p.data_ptr() + 7919 * p._version) % (1 << 61)
        return s

    def engine(self, device) -> WanVAEEngine:
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        e = self._engine
        if e is None or e.device != device or e.sig != self._param_signature():
            e = WanVAEEngine(self, device)
            self._engine = e
        return e

    _tiled_warned = False

    @classmethod
    def _note_untiled(cls, what):
        """`tiled=True` (the pipelines' default argument) is a DOCUMENTED deviation (INTEGRATION.md): the reference's tiling
        (wan_video_vae.py:643-744) is a memory workaround whose blend ramps change the result against its own untiled path;
        with 80 GB of HBM the untiled computation fits and is what runs.  Said once per process."""
        if not cls._tiled_warned:
            cls._tiled_warned = True
            import warnings
            warnings.warn(f"svi_b200: WanVideoVAE.{what}(tiled=True) runs UNTILED (tile_size / tile_stride ignored): results "
                          f"equal the reference's tiled=False path, not its blended tiles", stacklevel=3)

    def enable_spatial_sharding(self, group=None):
        """Split every encode / decode over the ranks of `group` (default: all ranks): each rank computes a band of image
        rows, neighbouring bands exchange one border row per convolution, results are gathered on every rank."""
        self.shard_group = (group,)

    def _sharded(self, eng):
        eng.shard = SpatialShard(self.shard_group[0]) if getattr(self, "shard_group", None) is not None else None
        return eng

    def encode(self, videos, device, tiled=False, tile_size=(34, 34), tile_stride=(18, 16)):
        if tiled:
            self._note_untiled("encode")
        eng = self._sharded(self.engine(device))
        return torch.stack([eng.encode(v) for v in videos])

    def decode(self, hidden_states, device, tiled=False, tile_size=(34, 34), tile_stride=(18, 16)):
        if tiled:
            self._note_untiled("decode")
        eng = self._sharded(self.engine(device))
        return torch.stack([eng.decode(h) for h in hidden_states])

    @staticmethod
    def state_dict_converter():
        return WanVideoVAEStateDictConverter()


class WanVideoVAEStateDictConverter:
    def from_civitai(self, state_dict):
        """reference :798-808: raw Wan VAE checkpoints hold un-prefixed keys (optionally under 'model_state')."""
        if "model_state" in state_dict:
            state_dict = state_dict["model_state"]
        return {"model." + k: v for k, v in state_dict.items()}
