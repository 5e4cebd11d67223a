"""RIFE frame interpolation (reference ``diffsynth/extensions/RIFE/__init__.py``) on the kernel library.

``IFNet`` is a parameter container with the reference's module names, so ``flownet.pkl`` checkpoints load as they are.
``RIFEEngine`` runs it on the sm_90a kernels of ``include/svi_b200_rife.h``: per block, one launch builds both directions'
space-to-depth input for every pair of the batch, the 12 convolutions run as batched implicit GEMMs with the PReLU (and
residual) in their epilogue, the two heads' ConvTranspose2d layers run as 3x3 sub-pixel convolutions (their first layers
as one GEMM, their second as one block-diagonal GEMM), and one launch upsamples, updates and warps.  The last block also
blends and writes uint8 RGB frames.  Frames cross the bus once, as bytes, in each direction.

``RIFEInterpolater`` and ``RIFESmoother`` keep the reference's call semantics.  Sizes: sides that are multiples of 32 give
the reference's computation; other sides run at full size when every block scale divides them as the network needs
(``check_size``); the reference instead shrinks such frames to ``(side + 31) // 32`` pixels and fails inside IFNet.
"""
import numpy as np
import torch
import torch.nn as nn
from PIL import Image

from ... import _native as nv

BLOCK_LD = 48         # channel pitch of the block input: 4 space-to-depth phases x 11 channels + 4 zeros
C0A = 46              # conv0's first layer: 45 channels + one zero channel, so that a phase holds an even count
FEAT_LD = 96          # bf16 pitch of the 90-channel activations
HEAD2_COLS = 6        # second head layer per phase: flow 4, mask 1, zero 1
HEADS_LD = 8          # f32 pitch of the heads' output


def _conv(cin, cout, stride=1):
    return nn.Sequential(nn.Conv2d(cin, cout, 3, stride, 1, bias=True), nn.PReLU(cout))


class IFBlock(nn.Module):
    """Parameters of one block (reference :32-41): conv0 (two stride-2 convs), four residual pairs, two heads."""

    def __init__(self, in_planes, c=90):
        super().__init__()
        self.conv0 = nn.Sequential(_conv(in_planes, c // 2, 2), _conv(c // 2, c, 2))
        for i in range(4):
            setattr(self, f"convblock{i}", nn.Sequential(_conv(c, c), _conv(c, c)))
        self.conv1 = nn.Sequential(nn.ConvTranspose2d(c, c // 2, 4, 2, 1), nn.PReLU(c // 2), nn.ConvTranspose2d(c // 2, 4, 4, 2, 1))
        self.conv2 = nn.Sequential(nn.ConvTranspose2d(c, c // 2, 4, 2, 1), nn.PReLU(c // 2), nn.ConvTranspose2d(c // 2, 1, 4, 2, 1))


class IFNet(nn.Module):
    """RIFE's IFNet (reference :60-100): block0..2 run, block_tea is loaded and never run."""

    def __init__(self, **kwargs):
        super().__init__()
        self.block0 = IFBlock(7 + 4, c=90)
        self.block1 = IFBlock(7 + 4, c=90)
        self.block2 = IFBlock(7 + 4, c=90)
        self.block_tea = IFBlock(10 + 4, c=90)
        self._engines = {}

    def engine(self, device=None):
        """The RIFEEngine of these weights on `device` (packed once; call drop_engines() after changing the weights)."""
        device = torch.device(device if device is not None else next(self.parameters()).device)
        if device not in self._engines:
            self._engines[device] = RIFEEngine(self, device)
        return self._engines[device]

    def drop_engines(self):
        self._engines = {}

    def load_state_dict(self, *args, **kwargs):
        self.drop_engines()
        return super().load_state_dict(*args, **kwargs)

    @torch.no_grad()
    def forward(self, x, scale_list=[4, 2, 1], training=False):
        """x f32 [N, 6, H, W] (img0 | img1, BGR in [0, 1]) on a CUDA device -> (flow_list, mask, merged) as the reference:
        the flow after each block [N, 4, H, W], sigmoid(mask) of the last block [N, 1, H, W], the blend of each block."""
        eng = self.engine(x.device)
        N, C, H, W = x.shape
        if C != 6:
            raise ValueError(f"IFNet: x must be [N, 6, H, W] (two BGR images), got {tuple(x.shape)}")
        check_size(H, W, scale_list)
        frames = torch.zeros(2 * N, H, W, 4, device=eng.device)
        frames[:N, ..., :3] = x[:, :3].permute(0, 2, 3, 1)
        frames[N:, ..., :3] = x[:, 3:].permute(0, 2, 3, 1)
        flows, merged = [], []
        eng.run(frames[:N], frames[N:], scale_list, record=(flows, merged))
        flow_list = [f.permute(0, 3, 1, 2).contiguous() for f in flows]
        mask = merged[-1][..., 3:4].permute(0, 3, 1, 2).contiguous()
        return flow_list, mask, [m[..., :3].permute(0, 3, 1, 2).contiguous() for m in merged]

    @staticmethod
    def state_dict_converter():
        return IFNetStateDictConverter()


class IFNetStateDictConverter:
    def from_diffusers(self, state_dict):
        return {k.replace("module.", ""): v for k, v in state_dict.items()}

    def from_civitai(self, state_dict):
        return self.from_diffusers(state_dict), {"upcast_to_float32": True}


# ------------------------------------------------------------------------------------------------ sizes
def block_sizes(H, W, scale_list):
    """[(h, w, s)] of the three blocks: the frame resized by 1 / s as F.interpolate(scale_factor=1 / s) does."""
    return [(int(np.floor(H * (1.0 / s))), int(np.floor(W * (1.0 / s))), s) for s in scale_list]


def check_size(H, W, scale_list):
    """Every block scale s must map H and W to whole sizes that are multiples of 4 (conv0 halves them twice, the heads
    double them twice) and back: at scale 1 (s = 4, 2, 1) that is sides that are multiples of 16."""
    for h, w, s in block_sizes(H, W, scale_list):
        if h <= 0 or w <= 0 or h % 4 or w % 4 or h * s != H or w * s != W:
            raise ValueError(f"RIFE: a {W}x{H} frame does not fit block scale {s}: every side divided by each of "
                             f"{list(scale_list)} must be a whole multiple of 4 (at scale 1.0: multiples of 16)")


# ------------------------------------------------------------------------------------------------ weight packing
def _ceil(a, b):
    return (a + b - 1) // b * b


def pack_s2d(weight, group, cpad):
    """A stride-2, padding-1 3x3 conv as a 2x2 conv with padding 1 over the space-to-depth input, whose channel
    (dy * 2 + dx) * group + c holds input channel c of pixel (2 y + dy, 2 x + dx): tap (bh, bw), phase (dy, dx) takes the
    original tap (2 bh + dy - 1, 2 bw + dx - 1) when it exists.  -> f32 [O, 4 cpad] in (tap, channel) order."""
    O, I = weight.shape[:2]
    w = torch.zeros(O, 2, 2, cpad, dtype=weight.dtype)
    for bh in range(2):
        for bw in range(2):
            for dy in range(2):
                for dx in range(2):
                    a, b = 2 * bh + dy - 1, 2 * bw + dx - 1
                    if 0 <= a <= 2 and 0 <= b <= 2:
                        w[:, bh, bw, (dy * 2 + dx) * group:(dy * 2 + dx) * group + I] = weight[:, :, a, b]
    return w.reshape(O, 4 * cpad)


def pack_3x3(weight, cpad):
    O, I = weight.shape[:2]
    w = torch.zeros(O, 3, 3, cpad, dtype=weight.dtype)
    w[..., :I] = weight.permute(0, 2, 3, 1)
    return w.reshape(O, 9 * cpad)


def pack_subpixel(weight, cols, cpad):
    """ConvTranspose2d(k=4, stride 2, padding 1) weight [I, O, 4, 4] as a 3x3 convolution (padding 1) whose column
    q * cols + o is output channel o of phase q = 2 py + px: destination pixel (2 y + py, 2 x + px) takes input pixel
    (y + a - 1, x + b - 1) through kernel tap (py + 1 - 2 (a - 1), px + 1 - 2 (b - 1)) when that lies in [0, 4).
    -> f32 [4 cols, 9 cpad]."""
    I, O = weight.shape[:2]
    w = torch.zeros(4, cols, 3, 3, cpad, dtype=weight.dtype)
    for py in range(2):
        for px in range(2):
            for a in range(3):
                for b in range(3):
                    ky, kx = py + 1 - 2 * (a - 1), px + 1 - 2 * (b - 1)
                    if 0 <= ky < 4 and 0 <= kx < 4:
                        w[py * 2 + px, :O, a, b, :I] = weight[:, :, ky, kx].t()
    return w.reshape(4 * cols, 9 * cpad)


def _phases(v, cols):
    """a per-channel vector of one phase (padded to cols) repeated for the four phases"""
    out = torch.zeros(cols, dtype=v.dtype)
    out[:v.numel()] = v
    return out.repeat(4)


def pack_block(block):
    """f32 kernel operands of one IFBlock: [(name, dict)] in launch order (device-agnostic; tested in fp64)."""
    g = {n: p.detach().double().cpu() for n, p in block.named_parameters()}
    layers = []
    w0 = torch.zeros(C0A, 11, 3, 3, dtype=torch.float64)
    w0[:45] = g["conv0.0.0.weight"]
    layers.append(("conv0a", dict(w=pack_s2d(w0, 11, 64), bias=torch.cat([g["conv0.0.0.bias"], torch.zeros(1, dtype=torch.float64)]),
                                  prelu=torch.cat([g["conv0.0.1.weight"], torch.ones(1, dtype=torch.float64)]))))
    w1 = torch.zeros(90, C0A, 3, 3, dtype=torch.float64)
    w1[:, :45] = g["conv0.1.0.weight"]
    layers.append(("conv0b", dict(w=pack_s2d(w1, C0A, _ceil(4 * C0A, 64)), bias=g["conv0.1.0.bias"], prelu=g["conv0.1.1.weight"])))
    for i in range(4):
        for j in range(2):
            layers.append((f"convblock{i}.{j}", dict(w=pack_3x3(g[f"convblock{i}.{j}.0.weight"], 128),
                                                    bias=g[f"convblock{i}.{j}.0.bias"], prelu=g[f"convblock{i}.{j}.1.weight"])))
    wt = torch.cat([g["conv1.0.weight"], g["conv2.0.weight"]], dim=1)                         # [90, 90, 4, 4]
    layers.append(("head1", dict(w=pack_subpixel(wt, 90, 128),
                                 bias=_phases(torch.cat([g["conv1.0.bias"], g["conv2.0.bias"]]), 90),
                                 prelu=_phases(torch.cat([g["conv1.1.weight"], g["conv2.1.weight"]]), 90))))
    wd = torch.zeros(90, HEAD2_COLS, 4, 4, dtype=torch.float64)                                 # block-diagonal
    wd[:45, :4] = g["conv1.2.weight"]
    wd[45:, 4:5] = g["conv2.2.weight"]
    layers.append(("head2", dict(w=pack_subpixel(wd, HEAD2_COLS, 128),
                                 bias=_phases(torch.cat([g["conv1.2.bias"], g["conv2.2.bias"]]), HEAD2_COLS), prelu=None)))
    return layers


def _pick_tile_w(H, W):
    best, cost = 16, None
    for bw in (8, 16, 32, 64, 128):
        c = -(-H // (128 // bw)) * -(-W // bw)
        if cost is None or c < cost:
            best, cost = bw, c
    return best


# ------------------------------------------------------------------------------------------------ engine
class RIFEEngine:
    """Packed weights of IFNet's three blocks on one device and the per-shape buffers of a batch of pairs."""

    def __init__(self, model: IFNet, device):
        nv.require_cuda(device, "RIFE")
        self.device = torch.device(device)
        self.blocks = []
        for blk in (model.block0, model.block1, model.block2):
            packed = {}
            for name, d in pack_block(blk):
                packed[name] = dict(w=d["w"].to(self.device, torch.bfloat16).contiguous(),
                                    bias=d["bias"].to(self.device, torch.float32).contiguous(),
                                    prelu=None if d["prelu"] is None else d["prelu"].to(self.device, torch.float32).contiguous())
            self.blocks.append(packed)
        self._bufs = {}

    def _buffers(self, P, H, W, h, w):
        key = (P, H, W, h, w)
        if key not in self._bufs:
            z = dict(device=self.device)
            n, h4, w4 = 2 * P, h // 4, w // 4
            self._bufs[key] = dict(
                x0=torch.zeros(n, h // 2, w // 2, BLOCK_LD, dtype=torch.bfloat16, **z),
                x1=torch.zeros(n, h4, w4, 4 * C0A, dtype=torch.bfloat16, **z),
                feat=torch.zeros(n, h4, w4, 90, **z),
                a=torch.zeros(n, h4, w4, FEAT_LD, dtype=torch.bfloat16, **z),
                b=torch.zeros(n, h4, w4, FEAT_LD, dtype=torch.bfloat16, **z),
                hd=torch.zeros(n, h // 2, w // 2, FEAT_LD, dtype=torch.bfloat16, **z),
                heads=torch.zeros(n, h, w, HEADS_LD, **z))
        return self._bufs[key]

    def _conv(self, L, x, kh, pad, C_out, cols, tile_w, **kw):
        nv.rife_conv2d(x, L["w"], kh, kh, pad, C_out, cols, L["bias"], tile_w, prelu=L["prelu"], **kw)

    def block(self, i, img0, img1, state, h, w, s, **update):
        """One IFBlock, both directions, on every pair of img0 / img1 (f32 [pairs, H, W, 4] views), then the update."""
        P, H, W, _ = img0.shape
        Wt = self.blocks[i]
        B = self._buffers(P, H, W, h, w)
        h4, w4 = h // 4, w // 4
        t4, t2 = _pick_tile_w(h4, w4), _pick_tile_w(h // 2, w // 2)
        src = np.float32(1.0 / (1.0 / s))
        nv.rife_block_input(img0, img1, None if i == 0 else state, h, w, src, np.float32(1.0 / s), B["x0"])
        self._conv(Wt["conv0a"], B["x0"], 2, 1, C0A, C0A, t2, out_bf16=B["x1"], bf_s2d=True)
        self._conv(Wt["conv0b"], B["x1"], 2, 1, 90, 90, t4, out=B["feat"], out_bf16=B["a"])
        for r in range(4):
            self._conv(Wt[f"convblock{r}.0"], B["a"], 3, 1, 90, 90, t4, out_bf16=B["b"])
            self._conv(Wt[f"convblock{r}.1"], B["b"], 3, 1, 90, 90, t4, residual=B["feat"],
                       out=None if r == 3 else B["feat"], out_bf16=B["a"])
        self._conv(Wt["head1"], B["a"], 3, 1, 4 * 90, 90, t4, out_bf16=B["hd"])
        self._conv(Wt["head2"], B["hd"], 3, 1, 4 * HEAD2_COLS, HEAD2_COLS, t2, out=B["heads"])
        nv.rife_update_warp(B["heads"], np.float32(1.0 / s), s, img0, img1, state, i == 0, **update)

    def run(self, img0, img1, scale_list, merged=None, clip=False, rgb=None, record=None):
        """All three blocks on the pairs (img0[p], img1[p]); the last block writes merged / rgb (see rife_update_warp).
        record = (flows, merged_list): also collect each block's flow [P, H, W, 4] and blend [P, H, W, 4]."""
        P, H, W, _ = img0.shape
        check_size(H, W, scale_list)
        state = torch.empty(P, H, W, 12, device=self.device)
        for i, (h, w, s) in enumerate(block_sizes(H, W, scale_list)):
            last = i == len(scale_list) - 1
            if record is not None:
                m = torch.empty(P, H, W, 4, device=self.device)
                self.block(i, img0, img1, state, h, w, s, merged=m)
                record[0].append(state[..., 8:12].clone())
                record[1].append(m)
            else:
                self.block(i, img0, img1, state, h, w, s,
                           **(dict(merged=merged, clip=clip, rgb=rgb) if last else {}))
        return state


# ------------------------------------------------------------------------------------------------ public interface
def _scale_list(scale):
    return [4 / scale, 2 / scale, 1 / scale]


class RIFEInterpolater:
    def __init__(self, model, device="cuda"):
        self.model = model
        self.device = device
        self.torch_dtype = torch.float32

    @staticmethod
    def from_model_manager(model_manager):
        return RIFEInterpolater(model_manager.fetch_model("rife"), device=model_manager.device)

    def process_image(self, image):
        """PIL RGB image -> f32 [3, H, W] BGR in [0, 1] (reference :130-137, without its resize of odd sizes)."""
        return torch.from_numpy(np.array(image, dtype=np.float32)[:, :, [2, 1, 0]] / 255).permute(2, 0, 1)

    def process_images(self, images):
        return torch.stack([self.process_image(image) for image in images])

    def decode_images(self, images):
        images = (images[:, [2, 1, 0]].permute(0, 2, 3, 1) * 255).clip(0, 255).numpy().astype(np.uint8)
        return [Image.fromarray(image) for image in images]

    def _engine(self):
        return self.model.engine(self.device)

    def _stage(self, images):
        """uint8 bytes of the frames -> device, f32 BGR frames [F, H, W, 4] and the uint8 frames [F, H, W, 3]."""
        arrs = [np.asarray(im.convert("RGB") if im.mode != "RGB" else im, dtype=np.uint8) for im in images]
        H, W = arrs[0].shape[:2]
        if any(a.shape != (H, W, 3) for a in arrs):
            raise ValueError("RIFE: every frame must have the size of the first")
        u8 = torch.from_numpy(np.stack(arrs)).to(self._engine().device)
        frames = torch.empty(len(arrs), H, W, 4, device=u8.device)
        nv.rife_stage_frames(u8, frames)
        return frames, u8

    @staticmethod
    def _to_pil(u8):
        return [Image.fromarray(a) for a in u8.cpu().numpy()]

    def _pairs(self, img0, img1, scale, batch_size, progress_bar=lambda x: x, **out):
        """Interpolate pairs (img0[p], img1[p]) in batches; out: merged / rgb views with one frame per pair."""
        eng = self._engine()
        n = img0.shape[0]
        for b0 in progress_bar(range(0, n, batch_size)):
            b1 = min(b0 + batch_size, n)
            eng.run(img0[b0:b1], img1[b0:b1], _scale_list(scale),
                    **{k: (v[b0:b1] if k in ("merged", "rgb") else v) for k, v in out.items()})

    @torch.no_grad()
    def interpolate_(self, images, scale=1.0):
        """The frame between each pair of neighbours (reference :155-164): len(images) - 1 frames, one batch."""
        frames, _ = self._stage(images)
        F, H, W, _ = frames.shape
        check_size(H, W, _scale_list(scale))
        rgb = torch.empty(F - 1, H, W, 3, dtype=torch.uint8, device=frames.device)
        self._pairs(frames[:-1], frames[1:], scale, max(F - 1, 1), rgb=rgb)
        return self._to_pil(rgb)

    @torch.no_grad()
    def interpolate(self, images, scale=1.0, batch_size=4, num_iter=1, progress_bar=lambda x: x):
        """Insert an interpolated frame between every pair of neighbours, num_iter times (reference :167-194):
        2^num_iter (len(images) - 1) + 1 frames."""
        frames, u8 = self._stage(images)
        check_size(frames.shape[1], frames.shape[2], _scale_list(scale))
        for _ in range(num_iter):
            F, H, W, _ = frames.shape
            nf = torch.empty(2 * F - 1, H, W, 4, device=frames.device)
            nu = torch.empty(2 * F - 1, H, W, 3, dtype=torch.uint8, device=frames.device)
            nf[0::2] = frames
            nu[0::2] = u8
            self._pairs(frames[:-1], frames[1:], scale, batch_size, progress_bar, merged=nf[1::2], clip=True, rgb=nu[1::2])
            frames, u8 = nf, nu
        return self._to_pil(u8)


class RIFESmoother(RIFEInterpolater):
    def __init__(self, model, device="cuda"):
        super().__init__(model, device=device)

    @staticmethod
    def from_model_manager(model_manager):
        # as the reference (:203-205): this returns a RIFEInterpolater
        return RIFEInterpolater(model_manager.fetch_model("rife"), device=model_manager.device)

    @torch.no_grad()
    def __call__(self, rendered_frames, scale=1.0, batch_size=4, num_iter=1, **kwargs):
        """Replace every inner frame by the blend of itself with the interpolation of its two neighbours (reference
        :218-239); the first and last frames stay."""
        frames, u8 = self._stage(rendered_frames)
        F, H, W, _ = frames.shape
        if F < 3:
            raise ValueError("RIFESmoother: needs at least 3 frames")
        check_size(H, W, _scale_list(scale))
        mid = torch.empty(F - 2, H, W, 4, device=frames.device)
        out = torch.empty(F - 2, H, W, 4, device=frames.device)
        for it in range(num_iter):
            self._pairs(frames[:-2], frames[2:], scale, batch_size, merged=mid)
            last = it == num_iter - 1
            self._pairs(frames[1:-1], mid, scale, batch_size, merged=out, **(dict(rgb=u8[1:-1]) if last else {}))
            frames[1:-1] = out
        return self._to_pil(u8)
