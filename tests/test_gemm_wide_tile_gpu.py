"""svi_gemm_bf16 on 128 x 256 tiles shared by both consumer warpgroups, at the edges that tile width creates, against an fp64
reference: N inside one tile and N % 256 not in {0, 128}; M below one warpgroup's 64 rows with ragged K; tile counts below
and just above the SM count (a partial last wave of the persistent grid); row sums of squares whose group starts in the
middle of a tile; the LayerNorm fold's a_next / row_stats; nothing written outside [M, N] of a strided output; and LoRA
column groups of an odd multiple of 128 columns (launched one group at a time) equal to one call per group."""
import pytest
import torch

from diffsynth import _native as nv

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _tiles_for(n_tiles_target, N):
    """M that makes ceil(M / 128) * ceil(N / 256) = n_tiles_target (n_tiles_target a multiple of the column tiles)."""
    cols = (N + 255) // 256
    return 128 * (n_tiles_target // cols) - 5


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(M, N, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(M, K, generator=g, device=DEV).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g, device=DEV) * K ** -0.5).to(torch.bfloat16)
    bias = torch.randn(N, generator=g, device=DEV) * 0.1
    gate = torch.randn(N, generator=g, device=DEV) * 0.5
    return g, a, w, bias, gate


def _acc_bound(a, w):
    """fp32 accumulation over K of exact bf16 products: |err| <= K u sum|a w| (u = 2^-23 leaves a factor of two)."""
    return a.shape[1] * 2.0 ** -23 * (a.double().abs() @ w.double().abs().t())


def _check(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    assert not bad.any(), f"{what}: {int(bad.sum())} elements out of bound, worst excess {float((err - bound).max()):.3e}"


# N in (128, 256), N % 256 in {8, 136, 200}; M below 64 with ragged K; M = 1
EDGE_SHAPES = [(1, 200, 64), (37, 136, 40), (63, 392, 200), (200, 648, 136), (300, 264, 1544)]


@pytest.mark.parametrize("M,N,K", EDGE_SHAPES)
def test_edge_shapes_residual_wide_pitch_canary(M, N, K):
    g, a, w, bias, gate = _inputs(M, N, K, 21)
    buf = torch.randn(M + 3, N + 40, generator=g, device=DEV)
    buf[M:] = float("nan")
    buf[:, N:] = float("nan")
    x = buf[:M, :N]
    x0 = x.double().clone()
    nv.gemm(a, w, x, bias=bias, gate=gate, residual=x)
    ref = (a.double() @ w.double().t() + bias.double()) * gate.double() + x0
    bound = 1.2 * _acc_bound(a, w) * gate.double().abs() + 2.0 ** -23 * (ref.abs() + x0.abs()) * 4 + 1e-30
    _check(x, ref, bound, "bias + gate + in-place residual")
    assert torch.isnan(buf[M:]).all() and torch.isnan(buf[:, N:]).all(), "written outside [M, N] of the residual"


@pytest.mark.parametrize("which", ["below", "above"])
def test_partial_last_wave(which):
    """ceil(M/128) * ceil(N/256) just below / just above the SM count: the last wave of the persistent grid is partial."""
    sms, N, K = _sms(), 1536, 512
    tiles = (sms // 6 - 1) * 6 if which == "below" else (sms // 6 + 1) * 6
    M = _tiles_for(tiles, N)
    assert ((M + 127) // 128) * 6 == tiles and (tiles < sms if which == "below" else tiles > sms)
    _, a, w, bias, _ = _inputs(M, N, K, 22)
    out = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    nv.gemm(a, w, out, bias=bias, act=nv.ACT_GELU_TANH)
    acc = a.double() @ w.double().t() + bias.double()
    ref = torch.nn.functional.gelu(acc, approximate="tanh")
    _check(out, ref, 1.2 * _acc_bound(a, w) + 2.0 ** -8 * ref.abs() + 1e-5 * (acc.abs() + 1e-3), "bias + gelu -> bf16")


@pytest.mark.parametrize("parts", [True, False])
def test_sumsq_group_starts_mid_tile(parts):
    """Groups of 384 columns: group 1 starts at column 384, the middle of the second 256-column tile.  Stored partials
    [M, groups * 3] (one per 128 columns) or atomic sums [M, groups]; strided bf16 output inside a NaN canary."""
    M, N, K, gc = 333, 1152, 200, 384
    g, a, w, bias, _ = _inputs(M, N, K, 23)
    canvas = torch.full((M + 2, N + 64), float("nan"), device=DEV, dtype=torch.bfloat16)
    out = canvas[1:M + 1, 16:16 + N]
    groups = N // gc
    ss = torch.full((M, groups, gc // 128), float("nan"), device=DEV) if parts else torch.zeros(M, groups, device=DEV)
    nv.gemm(a, w, out, bias=bias, sumsq=ss, sumsq_group_cols=gc)
    ref = a.double() @ w.double().t() + bias.double()
    bound = _acc_bound(a, w)
    _check(out, ref, 1.2 * bound + 2.0 ** -8 * ref.abs(), "bias -> strided bf16")
    keep = torch.ones_like(canvas, dtype=torch.bool)
    keep[1:M + 1, 16:16 + N] = False
    assert torch.isnan(canvas[keep].float()).all(), "written outside [M, N] of the strided output"
    got = ss.sum(-1) if parts else ss
    sref = (ref ** 2).view(M, groups, gc).sum(-1)
    sbound = (2 * ref.abs() * bound + bound ** 2).view(M, groups, gc).sum(-1) * 1.2 + gc * 2.0 ** -23 * sref + 1e-6
    _check(got, sref, sbound, "row sums of squares per group")


def test_fold_emit_a_next_row_stats():
    """Producer side of the LayerNorm fold on a ragged N: a_next = bf16(v * g_next), row_stats += (sum v, sum v^2)."""
    M, N, K = 190, 392, 264
    g, a, w, bias, gate = _inputs(M, N, K, 24)
    x = torch.randn(M, N, generator=g, device=DEV)
    x0 = x.double().clone()
    gn = torch.randn(N, generator=g, device=DEV)
    an_canvas = torch.full((M, N + 8), float("nan"), device=DEV, dtype=torch.bfloat16)
    a_next = an_canvas[:, :N]
    stats = torch.zeros(M, 2, device=DEV)
    nv.gemm(a, w, x, bias=bias, gate=gate, residual=x, emit=(a_next, gn, stats))
    v = (a.double() @ w.double().t() + bias.double()) * gate.double() + x0
    bound = 1.2 * _acc_bound(a, w) * gate.double().abs() + 2.0 ** -21 * (v.abs() + x0.abs())
    _check(x, v, bound, "residual out")
    _check(a_next, v * gn.double(), (bound * gn.double().abs()) * 1.2 + 2.0 ** -8 * (v * gn.double()).abs(), "a_next")
    assert torch.isnan(an_canvas[:, N:].float()).all(), "a_next written past N"
    vb = bound.sum(1)
    _check(stats[:, 0], v.sum(1), 1.2 * vb + N * 2.0 ** -23 * v.abs().sum(1) + 1e-6, "row_stats sum")
    q = (v ** 2).sum(1)
    _check(stats[:, 1], q, 1.2 * (2 * v.abs() * bound + bound ** 2).sum(1) + N * 2.0 ** -23 * q + 1e-6, "row_stats sum sq")


@pytest.mark.parametrize("w_dtype", [torch.bfloat16, torch.float8_e4m3fn])
def test_lora_odd_128_groups_equal_one_call_per_group(w_dtype):
    """group_cols = 384 (three 128-column segments): every group is its own launch, bit-identical to calling each group
    on its own columns with its block of U, row sums of squares included."""
    M, d, K, R = 700, 384, 256, 64
    g = torch.Generator(device=DEV).manual_seed(25)
    a = torch.randn(M, K, generator=g, device=DEV).to(torch.bfloat16)
    w = (torch.randn(3 * d, K, generator=g, device=DEV) * K ** -0.5).to(w_dtype)
    u = (torch.randn(M, 3 * R, generator=g, device=DEV) * 0.1).to(torch.bfloat16)
    b = (torch.randn(3 * d, R, generator=g, device=DEV) * R ** -0.5).to(torch.bfloat16)
    bias = torch.randn(3 * d, generator=g, device=DEV)
    out = torch.empty(M, 3 * d, device=DEV, dtype=torch.bfloat16)
    ss = torch.empty(M, 3, d // 128, device=DEV)
    nv.gemm_lora(a, w, out, u, b, R, d, bias=bias, sumsq=ss, sumsq_group_cols=d)
    for gi in range(3):
        cols = slice(gi * d, (gi + 1) * d)
        o = torch.empty(M, d, device=DEV, dtype=torch.bfloat16)
        s = torch.empty(M, 1, d // 128, device=DEV)
        nv.gemm_lora(a, w[cols], o, u[:, gi * R:(gi + 1) * R], b[cols], R, 0, bias=bias[cols], sumsq=s, sumsq_group_cols=d)
        assert torch.equal(out[:, cols].view(torch.int16), o.view(torch.int16))
        assert torch.equal(ss[:, gi:gi + 1].view(torch.int32), s.view(torch.int32))
    A = a.double()
    W = w.float().double()
    ref = torch.cat([A @ W[gi * d:(gi + 1) * d].t() + u[:, gi * R:(gi + 1) * R].double() @ b[gi * d:(gi + 1) * d].double().t()
                     for gi in range(3)], 1) + bias.double()
    bound = (K + R) * 2.0 ** -23 * (A.abs() @ W.abs().t() + torch.cat(
        [u[:, gi * R:(gi + 1) * R].double().abs() @ b[gi * d:(gi + 1) * d].double().abs().t() for gi in range(3)], 1))
    _check(out, ref, 1.2 * bound + 2.0 ** -8 * ref.abs(), "LoRA with 384-column groups")
