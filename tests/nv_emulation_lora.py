"""Torch stand-in for svi_gemm_lora_bf16 (include/svi_b200_lora.h) — TEST INFRASTRUCTURE ONLY.

Extends tests/nv_emulation.py: the LoRA segment is restated as what the kernel's k-blocks compute, one GEMM over [a | U]
and a weight whose extra columns hold B block-diagonally per column group, fed through nv_emulation.gemm (fp64
accumulation, the same epilogue).  `install(monkeypatch)` swaps it into diffsynth._native with the base stand-ins.
"""
import torch

import nv_emulation as base


def gemm_lora(a, w, out, u, b, R, group_cols=0, bias=None, act=0, gate=None, residual=None, sumsq=None, sumsq_group_cols=0,
              ln=None, emit=None):
    assert ln is None and emit is None, "svi_gemm_lora_bf16 takes no LayerNorm fold"
    assert act in (0, 1) and R % 64 == 0
    N, K = w.shape
    gc = group_cols or N
    groups = N // gc
    a_cat = torch.cat([a] + [u[:, g * R:(g + 1) * R] for g in range(groups)], dim=1)
    w_cat = torch.zeros(N, K + groups * R, dtype=torch.float64, device=w.device)
    w_cat[:, :K] = w.double()
    for g in range(groups):
        w_cat[g * gc:(g + 1) * gc, K + g * R:K + (g + 1) * R] = b[g * gc:(g + 1) * gc, :R].double()
    return base.gemm(a_cat, w_cat, out, bias=bias, act=act, gate=gate, residual=residual, sumsq=sumsq,
                     sumsq_group_cols=sumsq_group_cols)


def install(monkeypatch=None):
    from diffsynth import _native as nv
    base.install(monkeypatch)
    if monkeypatch is not None:
        monkeypatch.setattr(nv, "gemm_lora", gemm_lora)
    else:
        nv.gemm_lora = gemm_lora
