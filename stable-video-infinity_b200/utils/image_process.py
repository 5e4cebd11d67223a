"""Host-side image helpers the harness scripts star-import (reference utils/image_process.py).
Pure CPU / PIL / torch code at the clip boundary; nothing here is on the GPU hot path."""
import os

import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image


def tensor_to_pil(x):
    """[H,W,C] tensor in [0,1] (or uint8) -> PIL (reference :20-36)."""
    arr = x.cpu().numpy()
    if arr.dtype != np.uint8:
        arr = (np.clip(arr, 0, 1) * 255).astype(np.uint8)
    return Image.fromarray(arr)


def to_normalized(x):
    """0..255 -> -1..1"""
    return x / 255.0 * 2.0 - 1.0


def from_normalized(x):
    """-1..1 -> 0..255"""
    return (x + 1.0) / 2.0 * 255.0


def tensor2pil(x):
    """PIL image or tensor -> RGB PIL image (``test_svi_talk.py``, ``test_svi_dance.py``).  A 3-D tensor with 1 or 3
    leading channels is taken as CHW; non-uint8 data is clipped to [0, 1], scaled by 255 and truncated to uint8."""
    if isinstance(x, Image.Image):
        return x.convert("RGB")
    if not torch.is_tensor(x):
        raise TypeError(f"Expect tensor or PIL, got {type(x)}")
    if x.dim() == 3 and x.shape[0] in (1, 3):
        x = x.permute(1, 2, 0)
    arr = x.detach().cpu().numpy()
    if arr.dtype != np.uint8:
        arr = (np.clip(arr, 0, 1) * 255).astype(np.uint8)
    return Image.fromarray(arr)


def calculate_dimensions(image_input, max_width=640):
    """(height, width): width-limited, aspect preserved, floored to multiples of 16 (reference :39-70)."""
    img = image_input if isinstance(image_input, Image.Image) else Image.open(image_input)
    w0, h0 = img.size
    if w0 <= max_width:
        w, h = w0, h0
    else:
        w, h = max_width, int(max_width * (h0 / w0))
    return (h // 16) * 16, (w // 16) * 16


def find_reference_image(ref_image_root):
    """frame.jpg > frame.png > first jpg/jpeg > first png (reference :173-204)."""
    for name in ("frame.jpg", "frame.png"):
        p = os.path.join(ref_image_root, name)
        if os.path.exists(p):
            return p
    files = os.listdir(ref_image_root)
    for exts in ((".jpg", ".jpeg", ".JPG", ".JPEG"), (".png", ".PNG")):
        for ext in exts:
            for f in files:
                if f.endswith(ext):
                    return os.path.join(ref_image_root, f)
    raise FileNotFoundError(f"No reference image (jpg/png) found in {ref_image_root}")


def save_tensor_as_image(tensor, save_path, auto_detect_channels=True):
    """Save a 3-D tensor (2-D without ``auto_detect_channels``) as an image, min / max scaled to 0..255 (a constant tensor is scaled by 255 alone).
    With ``auto_detect_channels`` the channel axis is the only axis of size 1, 3 or 4, the smallest such axis when there
    are several, or else the smallest axis; it is moved last.  A channel axis past the third is not handled: nothing is
    saved."""
    arr = tensor.detach().cpu().numpy()
    if auto_detect_channels:
        shape = arr.shape
        candidates = [i for i, n in enumerate(shape) if n in (1, 3, 4)]
        if candidates:
            channel_dim = min(candidates, key=lambda i: shape[i])
        else:
            channel_dim = shape.index(min(shape))
        if channel_dim == 0:
            arr = np.transpose(arr, (1, 2, 0))
        elif channel_dim == 1:
            arr = np.transpose(arr, (0, 2, 1))
        elif channel_dim != 2:
            print(f"Warning: cannot place channel axis {channel_dim} of a {len(shape)}-D array; nothing saved")
            return
    if arr.max() != arr.min():
        arr = ((arr - arr.min()) / (arr.max() - arr.min()) * 255).astype(np.uint8)
    else:
        arr = (arr * 255).astype(np.uint8)
    if arr.ndim == 3 and arr.shape[-1] == 1:
        arr = arr.squeeze(-1)
    Image.fromarray(arr).save(save_path)


def resize_and_pad_to_target(tensor, target_size, pad_value=0):
    """[B, C, h, w] -> [B, C, th, tw] of the same dtype: scaled by min(th / h, tw / w) with nearest-neighbour sampling to
    (int(h * s), int(w * s)), then centred with ``pad_value`` (the odd pixel of padding goes bottom / right).  The
    SVI-Dance script fits its uint8 pose video to the clip size with it."""
    th, tw = target_size
    h, w = tensor.shape[-2:]
    s = min(th / h, tw / w)
    nh, nw = int(h * s), int(w * s)
    out = F.interpolate(tensor, size=(nh, nw), mode="nearest")
    top, left = (th - nh) // 2, (tw - nw) // 2
    return F.pad(out, (left, tw - nw - left, top, th - nh - top), mode="constant", value=pad_value)
