"""GPU: FastBlend's balanced and accurate modes and keyframe interpolation on the sm_90a kernels
(include/svi_b200_fastblend_modes.h).

Each entry point against the oracles' restatement (through the stand-ins of tests/nv_emulation_fastblend_modes.py, run on
the same device) bit for bit; the pairwise patch error against the reference's own kernel (compiled by build() into
oracle/_ref/libfastblend_ref.so); and each runner at 832x480 against oracle/fastblend_modes_oracle.py, byte for byte and
identical across two runs."""
import ctypes
import os

import numpy as np
import pytest
import torch

import nv_emulation_fastblend_modes as emu
from oracle import fastblend_modes_oracle as M
from test_fastblend_gpu import DEV, REF_LIB, frames4, random_nnf, same

pytestmark = pytest.mark.gpu

COVERED = {
    "svi_fastblend_candidate": ["test_candidate_matches_oracle"],
    "svi_fastblend_select": ["test_select_matches_oracle", "test_pairwise_error_within_reference_contraction"],
    "svi_fastblend_batch_mean": ["test_blends_match_oracle"],
    "svi_fastblend_running_mean": ["test_blends_match_oracle"],
    "svi_fastblend_to_u8": ["test_blends_match_oracle"],
}


@pytest.fixture(scope="module")
def nv():
    from diffsynth import _native
    _native.load()
    return _native


@pytest.fixture(scope="module")
def ref():
    if not os.path.exists(REF_LIB):
        pytest.skip("oracle/_ref/libfastblend_ref.so was not built (build() makes it where the reference tree exists)")
    lib = ctypes.CDLL(REF_LIB)
    i, p = ctypes.c_int, ctypes.c_void_p
    lib.ref_pairwise_patch_error.argtypes = [i] * 6 + [p] * 6
    return lib


@pytest.mark.parametrize("mode,kw", [(1, dict(dir=0)), (1, dict(dir=3)), (2, dict(draw=77, radius=4)),
                                     (3, dict(shift=1)), (3, dict(shift=-2)), (3, dict(shift=5)),
                                     (3, dict(shift=1, pairwise=True)), (3, dict(shift=-3, pairwise=True))])
def test_candidate_matches_oracle(nv, mode, kw):
    B, H, W = 6, 45, 80
    nnf = random_nnf(B, H, W, seed=mode)
    got = nv.fastblend_candidate(nnf, torch.full_like(nnf, -1), mode, **kw)
    assert same(got, emu.fastblend_candidate(nnf, torch.empty_like(nnf), mode, **kw))


def _select_inputs(B, H, W, seed):
    sg, ss, tg = frames4(B, H, W, seed), frames4(B, H, W, seed + 1), frames4(B, H, W, seed + 2)
    nnf, cand = random_nnf(B, H, W, seed), random_nnf(B, H, W, seed + 3)
    err = torch.rand(B, H, W, generator=torch.Generator().manual_seed(seed)).to(DEV) * 4e7
    return sg, ss, tg, nnf, cand, err


@pytest.mark.parametrize("patch", [13, 5])
@pytest.mark.parametrize("style", ["per_entry", "shared", "pairwise"])
@pytest.mark.parametrize("select", [0, 1])
def test_select_matches_oracle(nv, patch, style, select):
    B, H, W = 4, 45, 80
    sg, ss, tg, nnf, cand, err = _select_inputs(B, H, W, seed=patch)
    ts = {"per_entry": frames4(B, H, W, 9), "shared": frames4(1, H, W, 9)[0], "pairwise": None}[style]
    nin, ein = (nnf, err) if select else (None, None)
    want_n, want_e = torch.empty_like(nnf), torch.empty_like(err)
    emu.fastblend_select(sg, ss, tg, ts, cand, nin, ein, want_n, want_e, patch, 10.0, pairwise=style == "pairwise")
    got_n, got_e = torch.full_like(nnf, -1), torch.full_like(err, -1.0)
    nv.fastblend_select(sg, ss, tg, ts, cand, nin, ein, got_n, got_e, patch, 10.0, pairwise=style == "pairwise")
    assert same(got_n, want_n) and same(got_e, want_e)
    if select:
        assert 0 < (got_n != nnf).any(-1).float().mean() < 1
    if style == "pairwise":
        assert not torch.equal(got_e[0::2], got_e[1::2])     # the pair shares the style term, not the guide terms


@pytest.mark.parametrize("patch", [13, 5])
def test_pairwise_error_within_reference_contraction(nv, ref, patch):
    """guide_weight 0 leaves the pairwise style error alone; the reference's compiler contracts e += d * d into FMAs,
    so the two agree within taps * 3 * 2^-24 relative"""
    B, H, W = 4, 45, 80
    sg, ss, tg, _, cand, _ = _select_inputs(B, H, W, seed=patch)
    got_n, got_e = torch.empty_like(cand), torch.empty(B, H, W, device=DEV)
    nv.fastblend_select(sg, ss, tg, None, cand, None, None, got_n, got_e, patch, 0.0, pairwise=True)
    pad = 6
    padf = lambda t: torch.nn.functional.pad(t[..., :3], (0, 0, pad, pad, pad, pad)).contiguous()   # noqa: E731
    sa, sb = padf(ss[0::2]), padf(ss[1::2])
    na, nb = cand[0::2].contiguous(), cand[1::2].contiguous()
    err = torch.zeros(B // 2, H, W, device=DEV)
    assert ref.ref_pairwise_patch_error(B // 2, H, W, 3, patch, pad, sa.data_ptr(), na.data_ptr(), sb.data_ptr(),
                                        nb.data_ptr(), err.data_ptr(), None) == 0
    torch.cuda.synchronize()
    want = err.repeat_interleave(2, 0)
    rel = ((got_e.double() - want.double()).abs() / want.double().clamp_min(1e-30)).max().item()
    bound = patch * patch * 3 * 2.0 ** -24
    print(f"patch {patch}: max relative difference to the reference pairwise kernel {rel:.3e} (bound {bound:.3e})")
    assert rel <= bound


def test_blends_match_oracle(nv):
    H, W = 48, 80
    g = torch.Generator().manual_seed(0)
    u8 = torch.randint(0, 256, (H, W, 4), generator=g).float()
    u8[..., 3] = 0
    u8 = u8.to(DEV)
    stack = frames4(7, H, W, 1, scale=300.0) - 20.0                  # reaches past both ends of [0, 255]
    stack[..., 3] = 0
    got = nv.fastblend_batch_mean(stack, torch.full((H, W, 4), 7.0, device=DEV))
    assert same(got, emu.fastblend_batch_mean(stack, torch.empty(H, W, 4, device=DEV)))
    f64 = frames4(1, H, W, 3)[0].double() * 1.000000001
    for frame, frame_u8, w in [(u8, True, 1), (f64, False, 2), (f64, False, 6)]:
        got = nv.fastblend_running_mean(frame, w / (w + 1), stack[w], w + 1, torch.full((H, W, 4), 7.0, dtype=torch.float64,
                                                                                        device=DEV), frame_u8=frame_u8)
        want = emu.fastblend_running_mean(frame, w / (w + 1), stack[w], w + 1, torch.empty(H, W, 4, dtype=torch.float64,
                                                                                           device=DEV), frame_u8=frame_u8)
        assert same(got, want), w
    for a, a_u8 in [(u8, True), (stack[0], False), (stack[1].double() * 1.5, False)]:
        got = nv.fastblend_to_u8(a, torch.full((H, W, 3), 7, dtype=torch.uint8, device=DEV), a_u8=a_u8)
        assert same(got, emu.fastblend_to_u8(a, torch.empty(H, W, 3, dtype=torch.uint8, device=DEV)))


# ------------------------------------------------------------------------------------------- full size
def _video(n, seed):
    from tools.synth_fastblend import make_frames
    guide = make_frames(n, 480, 832, seed)
    style = np.ascontiguousarray(make_frames(n, 480, 832, seed + 1)[..., ::-1] // 2 + guide // 2)
    return list(guide), list(style)


def _config(**kw):
    return dict(dict(minimum_patch_size=5, threads_per_block=8, num_iter=5, gpu_id=0, guide_weight=10.0,
                     initialize="identity", tracking_window_size=0), **kw)


def _twice_and_oracle(run, oracle):
    a = np.stack([np.asarray(f) for f in run()])
    b = np.stack([np.asarray(f) for f in run()])
    assert np.array_equal(a, b)
    want, _ = oracle()
    assert a.shape == want.shape and np.array_equal(a, want), f"{int((a != want).sum())} bytes differ"


@pytest.mark.slow
def test_balanced_832x480_matches_oracle_bytes(nv):
    from diffsynth.extensions.FastBlend.runners import BalancedModeRunner
    guide, style = _video(6, seed=3)
    _twice_and_oracle(lambda: BalancedModeRunner().run(guide, style, 8, 2, _config()),
                      lambda: M.balanced(guide, style, 8, 2, device=DEV))


@pytest.mark.slow
def test_accurate_832x480_tracking_matches_oracle_bytes(nv):
    from diffsynth.extensions.FastBlend.runners import AccurateModeRunner
    guide, style = _video(4, seed=4)
    _twice_and_oracle(lambda: AccurateModeRunner().run(guide, style, 8, 1, _config(tracking_window_size=1)),
                      lambda: M.accurate(guide, style, 8, 1, device=DEV, tracking_window_size=1))


@pytest.mark.slow
def test_interpolation_832x480_matches_oracle_bytes(nv):
    from diffsynth.extensions.FastBlend.runners import InterpolationModeRunner
    guide, style = _video(9, seed=5)
    keys = [2, 6]
    _twice_and_oracle(lambda: InterpolationModeRunner().run(guide, [style[k] for k in keys], keys, 8,
                                                            _config(minimum_patch_size=15)),
                      lambda: M.interpolation(guide, [style[k] for k in keys], keys, 8, device=DEV, minimum_patch_size=15))


@pytest.mark.slow
def test_single_frame_832x480_tracking_matches_oracle_bytes(nv):
    from diffsynth.extensions.FastBlend.runners import InterpolationModeSingleFrameRunner
    guide, style = _video(12, seed=6)
    _twice_and_oracle(lambda: InterpolationModeSingleFrameRunner().run(guide, [style[5]], [5], 8,
                                                                       _config(tracking_window_size=2)),
                      lambda: M.single_frame(guide, [style[5]], [5], 8, device=DEV, tracking_window_size=2))
