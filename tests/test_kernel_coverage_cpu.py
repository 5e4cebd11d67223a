"""CPU: every entry point of include/svi_b200.h is exercised on the GPU by a named case, or exempt with a reason.

The table lives next to the cases, in tests/test_kernel_conformance_gpu.py (COVERED / EXEMPT).  A new entry point without a
case fails here, on the CPU, before anyone runs the GPU suite."""
import os
import re

import test_attention_fp64_gpu as attn64
import test_kernel_conformance_gpu as conf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _read(*parts):
    with open(os.path.join(ROOT, *parts)) as f:
        return f.read()


def header_entry_points():
    """names of the functions the C header declares (int / size_t / void / const char* svi_*(...))"""
    text = _read("include", "svi_b200.h")
    return set(re.findall(r"^(?:int|size_t|void|const char\*)\s+(svi_\w+)\s*\(", text, re.M))


def test_header_parser_finds_the_entry_points():
    names = header_entry_points()
    assert {"svi_gemm_bf16", "svi_attn_fwd_sp", "svi_col_stats_workspace_bytes", "svi_conv3d_causal", "svi_attn_plan",
            "svi_last_error"} <= names
    assert len(names) >= 50
    from diffsynth import _native
    assert names == set(_native.SIGNATURES), "the header and the ctypes signature table disagree"


def missing_entries(names, covered, exempt):
    return sorted(n for n in names if n not in covered and n not in exempt)


def test_every_entry_point_has_a_case_or_an_exemption():
    names = header_entry_points()
    missing = missing_entries(names, conf.COVERED, conf.EXEMPT)
    assert not missing, f"entry points with no GPU case and no exemption: {missing}"
    stale = sorted((set(conf.COVERED) | set(conf.EXEMPT)) - names)
    assert not stale, f"coverage table names entry points the header does not declare: {stale}"
    assert not set(conf.COVERED) & set(conf.EXEMPT)
    assert all(reason.strip() for reason in conf.EXEMPT.values())


def test_named_cases_exist():
    """A:<name> is a test function of the conformance module; B:<name> is a tools/gpu_check.py section that
    tests/test_kernels_gpu.py runs; F:<name> is a test function of tests/test_attention_fp64_gpu.py."""
    gpu_check = _read("tools", "gpu_check.py")
    sections = _read("tests", "test_kernels_gpu.py")
    for entry, cases in conf.COVERED.items():
        assert cases, f"{entry}: empty case list"
        for case in cases:
            kind, name = case.split(":", 1)
            if kind in ("A", "F"):
                mod = conf if kind == "A" else attn64
                assert callable(getattr(mod, name, None)) and name.startswith("test_"), f"{entry}: no test {name}"
            else:
                assert kind == "B", f"{entry}: case {case} is neither A:, B: nor F:"
                assert re.search(rf"^def sec_{name}\(", gpu_check, re.M), f"{entry}: gpu_check has no section {name}"
                assert f'"{name}"' in sections, f"{entry}: test_kernels_gpu.py does not run section {name}"


def test_guard_fails_when_an_entry_point_leaves_the_table():
    names = header_entry_points()
    for entry in ("svi_gemm_bf16", "svi_attn_fwd_sp", "svi_sp_push"):
        covered = {k: v for k, v in conf.COVERED.items() if k != entry}
        exempt = {k: v for k, v in conf.EXEMPT.items() if k != entry}
        assert missing_entries(names, covered, exempt) == [entry]
