"""ESRGAN 4x upscaling (reference ``diffsynth/extensions/ESRGAN/__init__.py``) on the kernel library.

``RRDBNet`` is a parameter container with the reference's module names, so ``RealESRGAN_x4.pth`` loads as it is.
``ESRGANEngine`` runs it on the sm_90a kernels of ``include/svi_b200_esrgan.h``: every layer is one batched 3x3
implicit-GEMM launch whose epilogue applies the bias, the LeakyReLU and the scaled residuals of the dense blocks and RRDBs.
A dense block keeps ``x | x1 | x2 | x3 | x4`` in one 192-channel bf16 buffer: conv k reads the first 64 + 32 (k - 1)
channels and writes its 32 just past them, so no concatenation is ever copied.  The two nearest-x2 upsamplings are
written by the epilogue of the conv before them, and conv_last writes uint8 RGB.  Frames cross the bus once, as bytes, in
each direction.

``ESRGAN`` keeps the reference's call semantics.  Every conv has stride 1 and padding 1, so any frame size runs.
"""
import numpy as np
import torch
import torch.nn as nn
from PIL import Image

from ... import _native as nv
from ..RIFE import _pick_tile_w, pack_3x3

FEAT, GROW = 64, 32
DENSE_LD = FEAT + 4 * GROW      # x | x1 | x2 | x3 | x4
IN_LD = 8                       # channels of the staged input pixel: R, G, B and 5 zeros
LAST_COLS = 4                   # conv_last's GEMM columns: R, G, B and a zero column (the epilogue moves channel pairs)
SLOPE = 0.2                     # LeakyReLU negative slope
RES_SCALE = 0.2                 # x5 * 0.2 + x and out * 0.2 + x


class ResidualDenseBlock(nn.Module):
    """Parameters of one dense block (reference :7-24)."""

    def __init__(self, num_feat=64, num_grow_ch=32):
        super().__init__()
        for k in range(1, 6):
            setattr(self, f"conv{k}", nn.Conv2d(num_feat + (k - 1) * num_grow_ch, num_grow_ch if k < 5 else num_feat, 3, 1, 1))


class RRDB(nn.Module):
    """Three dense blocks (reference :27-39)."""

    def __init__(self, num_feat, num_grow_ch=32):
        super().__init__()
        self.rdb1 = ResidualDenseBlock(num_feat, num_grow_ch)
        self.rdb2 = ResidualDenseBlock(num_feat, num_grow_ch)
        self.rdb3 = ResidualDenseBlock(num_feat, num_grow_ch)


def check_config(num_in_ch, num_out_ch, num_feat, num_block, num_grow_ch):
    for field, value, want in (("num_in_ch", num_in_ch, 3), ("num_out_ch", num_out_ch, 3), ("num_feat", num_feat, FEAT),
                               ("num_grow_ch", num_grow_ch, GROW)):
        if value != want:
            raise ValueError(f"ESRGAN: unsupported config {field}={value!r} (only {want!r} is implemented: the RGB x4 "
                             f"RRDBNet of RealESRGAN_x4)")
    if not isinstance(num_block, int) or num_block < 1:
        raise ValueError(f"ESRGAN: unsupported config num_block={num_block!r} (must be an integer >= 1)")


class RRDBNet(nn.Module):
    """ESRGAN's RRDBNet (reference :42-71): x f32 [N, 3, H, W] -> f32 [N, 3, 4H, 4W]."""

    def __init__(self, num_in_ch=3, num_out_ch=3, num_feat=64, num_block=23, num_grow_ch=32, **kwargs):
        super().__init__()
        check_config(num_in_ch, num_out_ch, num_feat, num_block, num_grow_ch)
        self.conv_first = nn.Conv2d(num_in_ch, num_feat, 3, 1, 1)
        self.body = nn.Sequential(*[RRDB(num_feat=num_feat, num_grow_ch=num_grow_ch) for _ in range(num_block)])
        self.conv_body = nn.Conv2d(num_feat, num_feat, 3, 1, 1)
        self.conv_up1 = nn.Conv2d(num_feat, num_feat, 3, 1, 1)
        self.conv_up2 = nn.Conv2d(num_feat, num_feat, 3, 1, 1)
        self.conv_hr = nn.Conv2d(num_feat, num_feat, 3, 1, 1)
        self.conv_last = nn.Conv2d(num_feat, num_out_ch, 3, 1, 1)
        self._engines = {}

    def engine(self, device=None):
        """The ESRGANEngine of these weights on `device` (packed once; call drop_engines() after changing the weights)."""
        device = torch.device(device if device is not None else self.conv_first.weight.device)
        if device not in self._engines:
            self._engines[device] = ESRGANEngine(self, device)
        return self._engines[device]

    def drop_engines(self):
        self._engines = {}

    def load_state_dict(self, *args, **kwargs):
        self.drop_engines()
        return super().load_state_dict(*args, **kwargs)

    @torch.no_grad()
    def forward(self, x):
        eng = self.engine(x.device)
        N, C, H, W = x.shape
        if C != 3:
            raise ValueError(f"ESRGAN: x must be [N, 3, H, W], got {tuple(x.shape)}")
        B = eng.buffers(N, H, W)
        B["x"].zero_()
        B["x"][..., :3] = x.permute(0, 2, 3, 1)
        out = torch.empty(N, 4 * H, 4 * W, LAST_COLS, device=eng.device)
        eng.run(N, H, W, out=out)
        return out[..., :3].permute(0, 3, 1, 2).contiguous()

    @staticmethod
    def state_dict_converter():
        return RRDBNetStateDictConverter()


class RRDBNetStateDictConverter:
    def from_diffusers(self, state_dict):
        return state_dict, {"upcast_to_float32": True}

    def from_civitai(self, state_dict):
        return state_dict, {"upcast_to_float32": True}


# ------------------------------------------------------------------------------------------------ weight packing
def pack_model(model):
    """f32 kernel operands {conv name: (w [rows, 9 cpad], bias [rows])} of every conv (device-agnostic; tested in fp64).
    cpad = the conv's input channels rounded up to 64; conv_last gets LAST_COLS rows, the last one zero."""
    out = {}
    for name, m in model.named_modules():
        if not isinstance(m, nn.Conv2d):
            continue
        w, b = m.weight.detach().double().cpu(), m.bias.detach().double().cpu()
        if name == "conv_last":
            w = torch.cat([w, w.new_zeros(LAST_COLS - w.shape[0], *w.shape[1:])])
            b = torch.cat([b, b.new_zeros(LAST_COLS - b.shape[0])])
        out[name] = (pack_3x3(w, (w.shape[1] + 63) // 64 * 64), b)
    return out


# ------------------------------------------------------------------------------------------------ engine
class ESRGANEngine:
    """Packed weights of RRDBNet on one device and the per-shape buffers of a batch."""

    def __init__(self, model: RRDBNet, device):
        nv.require_cuda(device, "ESRGAN")
        self.device = torch.device(device)
        self.num_block = len(model.body)
        self.w = {n: (w.to(self.device, torch.bfloat16).contiguous(), b.to(self.device, torch.float32).contiguous())
                  for n, (w, b) in pack_model(model).items()}
        self._bufs = {}

    def buffers(self, N, H, W):
        key = (N, H, W)
        if key not in self._bufs:
            self._bufs = {}             # one shape at a time: the 4x buffers are large
            z = dict(device=self.device)
            bf = dict(dtype=torch.bfloat16, **z)
            self._bufs[key] = dict(
                x=torch.zeros(N, H, W, IN_LD, **bf),
                F0=torch.empty(N, H, W, FEAT, **z), R=torch.empty(N, H, W, FEAT, **z), S=torch.empty(N, H, W, FEAT, **z),
                Da=torch.zeros(N, H, W, DENSE_LD, **bf), Db=torch.zeros(N, H, W, DENSE_LD, **bf),
                U1=torch.empty(N, 2 * H, 2 * W, FEAT, **bf),
                U2=torch.empty(N, 4 * H, 4 * W, FEAT, **bf), U3=torch.empty(N, 4 * H, 4 * W, FEAT, **bf))
        return self._bufs[key]

    def _conv(self, name, x, C_out, tile_w, **kw):
        w, b = self.w[name]
        nv.esrgan_conv2d(x, w, C_out, b, tile_w, **kw)

    def plan(self, N, H, W, rgb=None, out=None):
        """The launches of one batch in order: (conv name, input view, C_out, tile_w, epilogue kwargs).  The input is
        buffers(N, H, W)["x"]; rgb uint8 [N, 4H, 4W, 3] and / or out f32 [N, 4H, 4W, 4] receive conv_last."""
        B = self.buffers(N, H, W)
        t1, t2, t4 = _pick_tile_w(H, W), _pick_tile_w(2 * H, 2 * W), _pick_tile_w(4 * H, 4 * W)
        steps = [("conv_first", B["x"], FEAT, t1, dict(out=B["F0"], out_bf16=B["Da"][..., :FEAT]))]
        cur, nxt = B["Da"], B["Db"]
        for i in range(self.num_block):
            r_in = B["F0"] if i == 0 else B["R"]           # the RRDB's input stream; F0 is never written
            for r in (1, 2, 3):
                pre = f"body.{i}.rdb{r}."
                for k in range(1, 5):
                    c0 = FEAT + GROW * (k - 1)
                    steps.append((pre + f"conv{k}", cur[..., :c0], GROW, t1,
                                  dict(slope=SLOPE, out_bf16=cur[..., c0:c0 + GROW])))
                ep = dict(residual=r_in if r == 1 else B["S"], res_scale=RES_SCALE, out=B["S"], out_bf16=nxt[..., :FEAT])
                if r == 3:
                    ep.update(residual2=r_in, res2_scale=RES_SCALE, out=B["R"])
                steps.append((pre + "conv5", cur, FEAT, t1, ep))
                cur, nxt = nxt, cur                          # conv5 cannot write the buffer it reads
        steps += [
            ("conv_body", cur[..., :FEAT], FEAT, t1, dict(residual=B["F0"], res_scale=1.0, out_bf16=B["U1"], bf_up2=True)),
            ("conv_up1", B["U1"], FEAT, t2, dict(slope=SLOPE, out_bf16=B["U2"], bf_up2=True)),
            ("conv_up2", B["U2"], FEAT, t4, dict(slope=SLOPE, out_bf16=B["U3"])),
            ("conv_hr", B["U3"], FEAT, t4, dict(slope=SLOPE, out_bf16=B["U2"])),
            ("conv_last", B["U2"], LAST_COLS, t4, dict(out_u8=rgb, out=out)),
        ]
        return steps

    def run(self, N, H, W, rgb=None, out=None):
        for name, x, C_out, tile_w, ep in self.plan(N, H, W, rgb=rgb, out=out):
            self._conv(name, x, C_out, tile_w, **ep)

    def upscale_u8(self, u8, rgb):
        """uint8 RGB frames [N, H, W, 3] on the device -> rgb uint8 [N, 4H, 4W, 3]."""
        N, H, W, _ = u8.shape
        nv.esrgan_stage_frames(u8, self.buffers(N, H, W)["x"])
        self.run(N, H, W, rgb=rgb)


# ------------------------------------------------------------------------------------------------ public interface
class ESRGAN(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.model = model

    @staticmethod
    def from_model_manager(model_manager):
        return ESRGAN(model_manager.fetch_model("esrgan"))

    def process_image(self, image):
        return torch.Tensor(np.array(image, dtype=np.float32) / 255).permute(2, 0, 1)

    def process_images(self, images):
        return torch.stack([self.process_image(image) for image in images])

    def decode_images(self, images):
        images = (images.permute(0, 2, 3, 1) * 255).clip(0, 255).numpy().astype(np.uint8)
        return [Image.fromarray(image) for image in images]

    @torch.no_grad()
    def upscale(self, images, batch_size=4, progress_bar=lambda x: x):
        """4x upscale of a PIL image or a list of them (reference :109-137): the bytes of
        decode_images(RRDBNet(process_images(images)))."""
        is_single_image = not isinstance(images, list)
        if is_single_image:
            images = [images]
        eng = self.model.engine(self.model.conv_first.weight.device)
        arrs = [np.asarray(im.convert("RGB") if im.mode != "RGB" else im, dtype=np.uint8) for im in images]
        H, W = arrs[0].shape[:2]
        if any(a.shape != (H, W, 3) for a in arrs):
            raise ValueError("ESRGAN: every frame must have the size of the first")
        u8 = torch.from_numpy(np.stack(arrs)).to(eng.device)
        rgb = torch.empty(len(arrs), 4 * H, 4 * W, 3, dtype=torch.uint8, device=eng.device)
        for b0 in progress_bar(range(0, len(arrs), batch_size)):
            b1 = min(b0 + batch_size, len(arrs))
            eng.upscale_u8(u8[b0:b1], rgb[b0:b1])
        out = [Image.fromarray(a) for a in rgb.cpu().numpy()]
        return out[0] if is_single_image else out
