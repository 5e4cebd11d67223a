"""GPU: strict per-kernel parity of every C-ABI entry point against plain torch fp32 references of the same op
(GEMM + every epilogue, attention incl. ragged / strided / accumulate, row kernels, causal conv variants).
The cases live in tools/gpu_check.py (which also prints diagnostics when run by hand)."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("section", ["gemm", "gemm_epi", "attn", "attn_cross", "attn_bench", "abi3", "ln_fold", "ew", "conv",
                                     "conv_tiles", "gemm_edges", "attn_online", "attn_sp_one_gpu",
                                     pytest.param("attn_sp_one_gpu_long", marks=pytest.mark.slow), "attn_small_long"])
def test_kernel_section(section):
    from tools import gpu_check as G
    G.RESULTS.clear()
    getattr(G, "sec_" + section)()
    bad = [n for n, ok in G.RESULTS if not ok]
    assert G.RESULTS and not bad, f"failed cases: {bad}"
