"""GPU: the video processors on the sm_90a kernels of include/svi_b200_processors.h — the editors byte for byte against
Pillow's ImageEnhance at SVI frame sizes and at edge sizes, the RIFE average against its torch formula, the RIFE
smoother against the fp32 oracle, and a four-processor chain on the device against the same processors run one by one
through PIL."""
import numpy as np
import pytest
import torch
from PIL import Image, ImageEnhance

from oracle import processors_oracle as P
from oracle import rife_oracle as O
from test_processors_cpu import RATES, SWEEP
from tools import synth_rife as S

pytestmark = pytest.mark.gpu

COVERED = {
    "svi_luma_sum_u8": ["test_luma_sum_exact", "test_editors_match_pillow_at_svi_sizes"],
    "svi_enhance_blend_u8": ["test_editors_match_pillow_at_svi_sizes", "test_editors_match_pillow_at_edge_sizes"],
    "svi_sharpen_u8": ["test_editors_match_pillow_at_svi_sizes", "test_editors_match_pillow_at_edge_sizes",
                       "test_abi_validation_returns_status"],
    "svi_rife_average_u8": ["test_rife_average_matches_torch_formula", "test_abi_validation_returns_status"],
}

DEV = "cuda"


def _u8(images):
    return np.stack([np.asarray(im) for im in images])


def _pil(frames):
    return [Image.fromarray(f) for f in frames]


def _editors():
    from diffsynth.processors.PILEditor import ContrastEditor, SharpnessEditor
    return ContrastEditor, SharpnessEditor


@pytest.fixture(scope="module")
def sd():
    return S.make_state_dict(seed=0)


@pytest.fixture(scope="module")
def model(sd):
    from diffsynth.extensions.RIFE import IFNet
    m = IFNet().eval()
    m.load_state_dict(sd)
    return m.to(DEV)


def test_luma_sum_exact():
    from diffsynth import _native as nv
    rng = np.random.default_rng(0)
    frames = rng.integers(0, 256, (5, 720, 1280, 3), dtype=np.uint8)
    frames[3] = 255
    frames[4] = 0
    sums = nv.luma_sum_u8(torch.from_numpy(frames).to(DEV), torch.empty(5, dtype=torch.int64, device=DEV))
    assert sums.tolist() == [P.luma_sum(f) for f in frames]
    assert sums[3].item() == 255 * 720 * 1280


@pytest.mark.parametrize("H,W", [(480, 832), (720, 1280)])
def test_editors_match_pillow_at_svi_sizes(H, W):
    Contrast, Sharpness = _editors()
    rng = np.random.default_rng(H)
    frames = rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8)
    frames[1] = np.asarray(S.make_frames(1, H, W, seed=1)[0])
    frames[2] = np.clip(100 + rng.integers(-3, 4, (H, W, 3)), 0, 255).astype(np.uint8)
    pil = _pil(frames)
    for rate in RATES:
        for editor, enhance in ((Contrast, ImageEnhance.Contrast), (Sharpness, ImageEnhance.Sharpness)):
            got = _u8(editor(rate=rate)(pil))
            ref = np.stack([np.asarray(enhance(im).enhance(rate)) for im in pil])
            assert np.array_equal(got, ref), f"{editor.__name__} rate {rate}: {int((got != ref).sum())} bytes differ"


def test_editors_match_pillow_at_edge_sizes():
    Contrast, Sharpness = _editors()
    for name, frame in SWEEP:
        im = Image.fromarray(frame)
        for rate in RATES:
            assert np.array_equal(np.asarray(Contrast(rate=rate)([im])[0]),
                                  np.asarray(ImageEnhance.Contrast(im).enhance(rate))), (name, rate)
            assert np.array_equal(np.asarray(Sharpness(rate=rate)([im])[0]),
                                  np.asarray(ImageEnhance.Sharpness(im).enhance(rate))), (name, rate)


def test_rife_average_matches_torch_formula():
    from diffsynth import _native as nv
    g = torch.Generator(device="cpu").manual_seed(0)
    F, H, W = 6, 480, 832
    rgb = torch.randint(0, 256, (F, H, W, 3), dtype=torch.uint8, generator=g).to(DEV)
    frames = nv.rife_stage_frames(rgb, torch.empty(F, H, W, 4, device=DEV))
    merged = (torch.rand(F - 2, H, W, 4, generator=g) * 1.4 - 0.2).to(DEV)        # the blend is not clipped
    out = nv.rife_average_u8(frames, merged, rgb.clone())
    ref = rgb.clone()
    avg = (frames[1:-1, ..., :3] + merged[..., :3]) / 2
    ref[1:-1] = (avg[..., [2, 1, 0]] * 255).clip(0, 255).to(torch.uint8)
    assert torch.equal(out, ref)
    assert torch.equal(out[[0, -1]], rgb[[0, -1]])


def test_abi_validation_returns_status():
    from diffsynth import _native as nv
    lib = nv.load()
    stream = nv._stream()
    buf = torch.zeros(3, 8, 8, 4, device=DEV)
    u8 = torch.zeros(3, 8, 8, 3, dtype=torch.uint8, device=DEV)
    assert lib.svi_rife_average_u8(nv._ptr(buf), nv._ptr(buf), 2, 64, nv._ptr(u8), stream) < 0          # < 3 frames
    assert lib.svi_sharpen_u8(nv._ptr(u8), 3, 8, 8, 1.5, nv._ptr(u8), stream) < 0                        # in place
    assert lib.svi_sharpen_u8(nv._ptr(u8), 3, 8, 8, float("inf"), nv._ptr(torch.empty_like(u8)), stream) < 0
    assert lib.svi_luma_sum_u8(None, 3, 64, None, stream) < 0
    assert lib.svi_enhance_blend_u8(nv._ptr(u8), 0, 64, nv._ptr(buf), 1.0, nv._ptr(u8), stream) < 0
    torch.cuda.synchronize()


def _oracle_smooth(sd, frames, interpolate, batch=4):
    """processors_oracle.rife_smooth with IFNet on the device"""
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    x = O.to_tensor(frames).to(DEV)

    def run(inp):
        return torch.cat([O.ifnet(sdd, inp[b:b + batch])[2][2] for b in range(0, inp.shape[0], batch)])

    torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        mid = run(torch.cat((x[:-2], x[2:]), 1))
        if not interpolate:
            return P.average_u8(x.cpu(), mid.cpu())
        x[1:-1] = run(torch.cat((x[1:-1], mid), 1))
    return O.to_uint8(x.cpu())


@pytest.mark.parametrize("interpolate", [True, False])
def test_rife_smoother_matches_oracle_and_is_reproducible(model, sd, interpolate):
    from diffsynth.processors.RIFE import RIFESmoother
    frames = _u8(S.make_frames(7, 480, 832, seed=2))
    r = RIFESmoother(model, device=DEV, batch_size=4, interpolate=interpolate)
    got = _u8(r(_pil(frames)))
    ref = _oracle_smooth(sd, frames, interpolate)
    d = np.abs(got.astype(int) - ref.astype(int))
    print(f"RIFE processor interpolate={interpolate} 7 frames 832x480: mean|d| {d.mean():.3f}, within 2: {(d <= 2).mean():.4%}")
    assert np.array_equal(got[[0, -1]], frames[[0, -1]])
    assert d.mean() <= 0.5 and (d <= 2).mean() >= 0.99
    r.batch_size = 1
    assert np.array_equal(_u8(r(_pil(frames))), got)
    r.batch_size = 4
    t = torch.from_numpy(frames).to(DEV)
    out = r(t)
    assert torch.is_tensor(out) and np.array_equal(out.cpu().numpy(), got) and np.array_equal(t.cpu().numpy(), frames)


class _Manager:
    device = DEV

    def __init__(self, model):
        self.model = model

    def fetch_model(self, name, *args, **kwargs):
        assert name == "rife"
        return self.model


def test_four_processor_chain_on_device_matches_pil(model):
    from diffsynth.processors.sequencial_processor import SequencialProcessor
    frames = S.make_frames(6, 480, 832, seed=5)
    guide = S.make_frames(6, 480, 832, seed=6)
    chain = SequencialProcessor.from_model_manager(_Manager(model), [
        {"processor_type": "FastBlend", "config": {"inference_mode": "fast", "batch_size": 4, "window_size": 3}},
        {"processor_type": "RIFE", "config": {"batch_size": 2, "interpolate": True}},
        {"processor_type": "Contrast", "config": {"rate": 1.3}},
        {"processor_type": "Sharpness", "config": {"rate": 1.8}}])
    one_by_one = frames
    for p in chain.processors:
        one_by_one = p(one_by_one, original_frames=guide)
    ref = _u8(one_by_one)
    got = chain(frames, original_frames=guide)
    assert all(isinstance(f, Image.Image) for f in got) and np.array_equal(_u8(got), ref)
    t = torch.from_numpy(_u8(frames)).to(DEV)
    out = chain(t, original_frames=guide)
    assert torch.is_tensor(out) and out.is_cuda and np.array_equal(out.cpu().numpy(), ref)


def test_bad_input_raises(model):
    from diffsynth.processors.RIFE import RIFESmoother
    Contrast, Sharpness = _editors()
    frames = S.make_frames(3, 480, 832, seed=0)
    torch.cuda.synchronize()
    for p in (Contrast(), Sharpness(), RIFESmoother(model, device=DEV)):
        with pytest.raises(ValueError, match="size of the first"):
            p(frames[:2] + S.make_frames(1, 480, 816))
        with pytest.raises(ValueError, match="mode RGB"):
            p(frames[:2] + [frames[2].convert("RGBA")])
        with pytest.raises(ValueError, match="uint8"):
            p(torch.zeros(3, 480, 832, 3, device=DEV))
    with pytest.raises(ValueError, match="at least 3 frames"):
        RIFESmoother(model, device=DEV)(frames[:2])
    with pytest.raises(ValueError, match="multiple of 4"):
        RIFESmoother(model, device=DEV)(S.make_frames(3, 488, 832))
    torch.cuda.synchronize()
