"""svi_gemm_bf16's tile schedule (ping-pong consumer warpgroups on 128 x 128 tiles, batched epilogue loads) against an fp64
reference: tile counts of 1, odd, below and above the SM count; ragged M, N and K; in-place residuals with a row pitch
wider than N; strided outputs inside a NaN canary; bit-identical repeats and e4m3 == bf16(e4m3) weights."""
import math

import pytest
import torch

from diffsynth import _native as nv

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (M, N, K): M around the 64-row halves and 128-row tiles, N not a multiple of 128, K not a multiple of 64; tile counts
# 1 (1 x 128), odd (127 x 1288 -> 11), below the SM count (65 x 392 -> 4) and many waves (32760 x 1536 -> 3072)
SHAPES = [(1, 128, 64), (63, 136, 72), (64, 256, 128), (65, 392, 1536), (127, 1288, 200), (129, 1536, 1536),
          (32760, 1536, 1536)]


def _inputs(M, N, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(M, K, generator=g, device=DEV).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g, device=DEV) * K ** -0.5).to(torch.bfloat16)
    bias = torch.randn(N, generator=g, device=DEV) * 0.1
    gate = torch.randn(N, generator=g, device=DEV) * 0.5
    return g, a, w, bias, gate


def _acc_bound(a, w):
    """fp32 accumulation over K of exact bf16 products: |err| <= K u sum|a w| (u = 2^-23 leaves a factor of two)."""
    K = a.shape[1]
    return K * 2.0 ** -23 * (a.double().abs() @ w.double().abs().t())


def _check(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    assert not bad.any(), f"{what}: {int(bad.sum())} elements out of bound, worst excess {float((err - bound).max()):.3e}"


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_bias_gelu_bf16(M, N, K):
    _, a, w, bias, _ = _inputs(M, N, K, 1)
    out = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    nv.gemm(a, w, out, bias=bias, act=nv.ACT_GELU_TANH)
    acc = a.double() @ w.double().t() + bias.double()
    ref = torch.nn.functional.gelu(acc, approximate="tanh")
    bound = 1.2 * _acc_bound(a, w) + 2.0 ** -8 * ref.abs() + 1e-5 * (acc.abs() + 1e-3)
    _check(out, ref, bound, "bias + gelu_tanh -> bf16")


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_residual_in_place_wide_pitch(M, N, K):
    g, a, w, bias, gate = _inputs(M, N, K, 2)
    buf = torch.randn(M, N + 24, generator=g, device=DEV)
    buf[:, N:] = float("nan")
    x = buf[:, :N]
    x0 = x.double().clone()
    nv.gemm(a, w, x, bias=bias, gate=gate, residual=x)
    v = (a.double() @ w.double().t() + bias.double()) * gate.double()
    ref = v + x0
    bound = _acc_bound(a, w) * gate.double().abs() + 2.0 ** -22 * (v.abs() + ref.abs() + 1e-30)
    _check(x, ref, bound, "bias + gate + in-place residual (ldr = N + 24)")
    assert torch.isnan(buf[:, N:]).all(), "wrote outside the residual / out columns"


@pytest.mark.parametrize("M,N,K", [s for s in SHAPES if s[1] % 128 == 0])
def test_strided_out_canary_sumsq(M, N, K):
    _, a, w, bias, _ = _inputs(M, N, K, 3)
    big = torch.full((M + 5, 3 * N), float("nan"), device=DEV, dtype=torch.bfloat16)
    out = big[:M, :N]                       # ldo = 3N, like cross q writing qkv[:, :d]
    P = N // 128
    ss = torch.full((M, 1, P), float("nan"), device=DEV)
    nv.gemm(a, w, out, bias=bias, sumsq=ss, sumsq_group_cols=N)
    ref = a.double() @ w.double().t() + bias.double()
    bound = _acc_bound(a, w)
    _check(out, ref, bound + 2.0 ** -8 * ref.abs(), "bias -> strided bf16")
    assert torch.isnan(big[:M, N:]).all() and torch.isnan(big[M:]).all(), "wrote outside the strided output"
    seg = ref.view(M, P, 128)
    ss_ref = (seg * seg).sum(-1)
    ss_bound = (2 * seg.abs() * bound.view(M, P, 128) + bound.view(M, P, 128) ** 2).sum(-1) + 1e-5 * ss_ref
    _check(ss.view(M, P), ss_ref, ss_bound, "partial row sums of squares")


@pytest.mark.parametrize("M,N,K", [(129, 1288, 200), (32760, 1536, 1536)])
def test_repeat_bit_identical(M, N, K):
    _, a, w, bias, gate = _inputs(M, N, K, 4)
    outs = []
    for _ in range(2):
        out = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
        nv.gemm(a, w, out, bias=bias, gate=gate, act=nv.ACT_GELU_TANH)
        outs.append(out)
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("M,N,K", [(32760, 4608, 1536), (32760, 1536, 1536), (32760, 8960, 1536), (32760, 1536, 8960),
                                   (65, 392, 1536)])
def test_e4m3_equals_bf16(M, N, K):
    g, a, _, bias, gate = _inputs(M, N, K, 5)
    w8 = (torch.randn(N, K, generator=g, device=DEV) * K ** -0.5).to(torch.float8_e4m3fn)
    x = torch.randn(M, N, generator=g, device=DEV)
    got = []
    for w in (w8, w8.to(torch.bfloat16)):
        out = x.clone()
        nv.gemm(a, w, out, bias=bias, gate=gate, residual=out)
        got.append(out)
    assert torch.equal(got[0], got[1]), "e4m3 weights differ from their bf16 values"
    assert math.isfinite(float(got[0].abs().max()))
