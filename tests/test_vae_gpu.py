"""GPU parity of the native VAE (wgmma implicit-GEMM convs through the C ABI) against the streaming oracle.

The reference runs the VAE in fp32; the native path uses bf16 conv operands with fp32 accumulation and fp32
activations, so decode parity is asserted in uint8 pixel levels (what the clip loop actually recycles,
svi_video.py:366-370) and encode parity relative to the latent scale."""
import os

import numpy as np
import pytest
import torch

from tools import synth_vae

pytestmark = pytest.mark.gpu


def _vae():
    from diffsynth.models.wan_video_vae import WanVideoVAE
    sd = {k: v.to(torch.bfloat16).float() if v.dim() > 1 and "gamma" not in k else v
          for k, v in synth_vae.make_vae_state_dict(seed=0).items()}
    m = WanVideoVAE().eval()
    m.load_state_dict(sd)
    return m.to("cuda"), sd


def _levels(a, b):
    d = (a - b).abs() * 127.5
    return d.max().item(), d.mean().item()


@pytest.mark.parametrize("T,H,W", [(9, 32, 48), (5, 64, 96)])
def test_vae_decode_matches_oracle(T, H, W):
    from oracle import wan_vae_oracle as V
    m, sd = _vae()
    g = torch.Generator().manual_seed(5)
    tl = (T - 1) // 4 + 1
    z = torch.randn(1, 16, tl, H // 8, W // 8, generator=g)
    with torch.no_grad():
        ref = V.vae_decode(sd, z)
    out = m.decode(z.cuda(), device="cuda").cpu()
    assert out.shape == ref.shape
    mx, mean = _levels(out, ref)
    print(f"decode {T}x{H}x{W}: max {mx:.2f} levels, mean {mean:.3f} levels")
    assert mx < 6.0 and mean < 0.6


@pytest.mark.parametrize("T,H,W", [(9, 32, 48), (5, 64, 96)])
def test_vae_encode_matches_oracle(T, H, W):
    from oracle import wan_vae_oracle as V
    m, sd = _vae()
    g = torch.Generator().manual_seed(6)
    video = torch.rand(3, T, H, W, generator=g) * 2 - 1
    with torch.no_grad():
        ref = V.vae_encode(sd, video.unsqueeze(0))
    out = m.encode([video.cuda()], device="cuda").cpu()
    assert out.shape == ref.shape
    err = (out - ref).abs()
    print(f"encode {T}x{H}x{W}: max {err.max().item():.4e} mean/std {err.mean().item() / ref.std().item():.4e}")
    assert err.max().item() < 0.05 * ref.std().item() + 0.02 and err.mean().item() < 6e-3 * ref.std().item()


def test_vae_golden_fixture():
    """against the committed output of the real reference VAE (fp32 weights)"""
    from diffsynth.models.wan_video_vae import WanVideoVAE
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "vae_tiny.npz"))
    m = WanVideoVAE().eval()
    m.load_state_dict(synth_vae.make_vae_state_dict(seed=0))
    m.to("cuda")
    dec = m.decode(torch.from_numpy(g["z"]).cuda(), device="cuda").cpu()
    lat = m.encode([torch.from_numpy(g["video"]).cuda()], device="cuda").cpu()
    mx, mean = _levels(dec, torch.from_numpy(g["dec"]))
    assert mx < 6.0 and mean < 0.6
    ref = torch.from_numpy(g["lat"])
    assert (lat - ref).abs().max().item() < 0.05 * ref.std().item() + 0.02
