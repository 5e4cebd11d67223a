"""Host-side video helpers the SVI-Talk and SVI-Dance harness scripts import (reference utils/video_process.py).

``test_svi_talk.py`` imports ``image_compose_width``; ``test_svi_dance.py`` star-imports this module and takes the name
``imageio`` from it to read its pose video.  imageio is therefore bound at module level, but it is optional: without it
this module still imports, and any use of ``imageio`` (or ``save_dwpose_as_mp4``) raises an ImportError that says what
to install.  Pure CPU / PIL code at the clip boundary; nothing here is on the GPU hot path.
"""
import numpy as np
import torch
from PIL import Image

try:
    import imageio
except ImportError as e:
    _imageio_error = e                        # the `as` name is unbound when the except block ends

    class _MissingImageio:
        """Stands in for the imageio module when it is not installed; every attribute access raises."""

        def __getattr__(self, name):
            raise ImportError("imageio is not installed; reading and writing videos needs it "
                              "(pip install imageio imageio-ffmpeg)") from _imageio_error

    imageio = _MissingImageio()


def save_dwpose_as_mp4(dwpose_data, output_path, fps=30, quality=9, normalize=True, ffmpeg_params=None):
    """Write a pose tensor ([T, C, H, W], or [C, T, H, W] when dim 0 is 3; numpy or torch) as an MP4 through imageio.

    One channel is repeated to three, more than three are cut to the first three, fewer are zero-padded.  With
    ``normalize`` the data is scaled by its global min / max (+1e-8) to [0, 1]; frames are ``(x * 255).astype(uint8)``."""
    get_writer = imageio.get_writer                # the ImportError naming imageio, before any work, when it is missing
    if isinstance(dwpose_data, np.ndarray):
        dwpose_data = torch.from_numpy(dwpose_data)
    if dwpose_data.shape[0] == 3:
        dwpose_data = dwpose_data.permute(1, 0, 2, 3)
    T, C, H, W = dwpose_data.shape
    data = dwpose_data.detach().cpu().numpy()
    if C == 1:
        data = np.repeat(data, 3, axis=1)
    elif C > 3:
        data = data[:, :3]
    elif C < 3:
        data = np.concatenate([data, np.zeros((T, 3 - C, H, W))], axis=1)
    if normalize:
        data = (data - data.min()) / (data.max() - data.min() + 1e-8)
    frames = (data * 255).astype(np.uint8).transpose(0, 2, 3, 1)
    writer = get_writer(output_path, fps=fps, quality=quality, ffmpeg_params=ffmpeg_params)
    for frame in frames:
        writer.append_data(frame)
    writer.close()
    print(f"Video saved to: {output_path}")


def image_compose_width(imag, imag_1):
    """A new RGB image, as tall as ``imag``, holding ``imag`` at (0, 0) and ``imag_1`` to its right (PIL paste: a
    taller second image is cropped, a shorter one leaves black below it)."""
    width, height = imag.size
    out = Image.new("RGB", (width + imag_1.size[0], height))
    out.paste(imag, (0, 0))
    out.paste(imag_1, (width, 0))
    return out
