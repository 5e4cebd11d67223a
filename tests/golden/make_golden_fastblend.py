"""Generate tests/golden/fastblend_tiny.npz by running the REAL reference FastBlend host code on the CPU.

CuPy is not needed: a numpy stand-in is put into sys.modules["cupy"] before the reference package
(diffsynth/extensions/FastBlend) is loaded by file path.  The stand-in gives the reference's calls their numpy meaning,
plus: `.get()`; a no-op `cuda.Device`; the memory-pool calls; `random` drawing from the counter-based stream of
include/svi_b200_fastblend.h (the counter reset before each top-level call); and `RawKernel`, which dispatches the
reference's three kernel names to literal numpy restatements of their CUDA source, each square and each addition
rounded on its own as the native kernels do.  Nothing from the reference is copied into this repository; the committed
output pins oracle/fastblend_oracle.py to the reference's host logic (tests/test_fastblend_cpu.py).

usage:  python tests/golden/make_golden_fastblend.py [--ref /root/reference]
"""
import argparse
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle.fastblend_oracle import stream_u  # noqa: E402  (the stream's definition, shared with the kernels)
from tools.synth_fastblend import digest, make_frames, nnf_inputs  # noqa: E402


# ---------------------------------------------------------------------------------------------------- numpy "cupy"
class ndarray(np.ndarray):
    def get(self):
        return np.asarray(self)


def _w(x):
    return np.asarray(x).view(ndarray)


class _Random:
    k = 0

    def _next(self):
        self.k += 1
        return self.k - 1

    def randint(self, low, high=None, size=None, dtype=int):
        n = int(np.prod(size))
        u = stream_u(self._next(), np.arange(n, dtype=np.uint32)) % np.uint32(high - low)
        return _w((low + u.astype(np.int64)).astype(dtype).reshape(size))

    def permutation(self, n):
        assert n == 4
        j = int(stream_u(self._next(), 0)) % 24
        rest = [0, 1, 2, 3]
        return _w(np.array([rest.pop(d) for d in (j // 6, (j // 2) % 3, j % 2, 0)]))


def _remap(height, width, channel, patch_size, pad_size, source_style, nnf, target_style):
    """remapping_kernel: target[pixel] += source[nnf(pixel + (px, py)) - (px, py)] over the valid taps, then /= num"""
    r = (patch_size - 1) // 2
    B = source_style.shape[0]
    y = np.arange(height).reshape(1, height, 1)
    x = np.arange(width).reshape(1, 1, width)
    b = np.arange(B).reshape(B, 1, 1)
    acc = np.zeros((B, height, width, channel), np.float32)
    num = np.zeros((B, height, width), np.int64)
    for px in range(-r, r + 1):
        for py in range(-r, r + 1):
            ny, nx = y + px, x + py
            inside = (ny >= 0) & (ny < height) & (nx >= 0) & (nx < width)
            m = np.asarray(nnf)[b, ny.clip(0, height - 1), nx.clip(0, width - 1)]
            sy, sx = m[..., 0] - px, m[..., 1] - py
            ok = inside & (sy >= 0) & (sx >= 0) & (sy < height) & (sx < width)
            v = np.asarray(source_style)[b, sy.clip(0, height - 1) + pad_size, sx.clip(0, width - 1) + pad_size]
            acc = np.where(ok[..., None], acc + v, acc)
            num += ok
    target_style[:, pad_size:pad_size + height, pad_size:pad_size + width] = acc / num[..., None].astype(np.float32)


def _patch_error(height, width, channel, patch_size, pad_size, source, nnf, target, error):
    """patch_error_kernel: e += (target[pixel + (px, py)] - source[nnf + (px, py)])^2, px, py, c order"""
    r = (patch_size - 1) // 2
    B = source.shape[0]
    b = np.arange(B).reshape(B, 1, 1)
    nnf = np.asarray(nnf)
    src, tgt = np.asarray(source), np.asarray(target)
    e = np.zeros((B, height, width), np.float32)
    for px in range(-r, r + 1):
        for py in range(-r, r + 1):
            s = src[b, nnf[..., 0] + pad_size + px, nnf[..., 1] + pad_size + py]
            t = tgt[:, pad_size + px:pad_size + px + height, pad_size + py:pad_size + py + width]
            for c in range(channel):
                d = t[..., c] - s[..., c]
                e = e + d * d
    error[...] = e


class _RawKernel:
    def __init__(self, code, name):
        self.name = name

    def __call__(self, grid, block, args):
        if self.name == "remap":
            return _remap(*args)
        if self.name == "patch_error":
            return _patch_error(*args)
        raise NotImplementedError(self.name)      # pairwise_patch_error: not on the fast mode's path


class _Device:
    def __init__(self, *a):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


class _Pool:
    def free_all_blocks(self):
        pass


def make_cupy():
    cp = types.ModuleType("cupy")
    cp.ndarray = ndarray
    cp.float32, cp.int32 = np.float32, np.int32
    for name in ("pad", "zeros", "concatenate", "clip", "stack", "repeat", "tile", "arange"):
        setattr(cp, name, (lambda f: lambda *a, **k: _w(f(*a, **k)))(getattr(np, name)))
    cp.array = lambda x, dtype=None: _w(np.array(x, dtype=dtype))
    cp.random = _Random()
    cp.RawKernel = _RawKernel
    cp.cuda = types.SimpleNamespace(Device=_Device)
    cp.get_default_memory_pool = cp.get_default_pinned_memory_pool = lambda: _Pool()
    return cp


def load_reference(ref_root):
    sys.modules["cupy"] = make_cupy()
    path = os.path.join(ref_root, "diffsynth", "extensions", "FastBlend")
    spec = importlib.util.spec_from_file_location("_ref_fastblend", os.path.join(path, "__init__.py"),
                                                  submodule_search_locations=[path])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["_ref_fastblend"] = mod
    spec.loader.exec_module(mod)
    return mod, sys.modules["cupy"]


# ---------------------------------------------------------------------------------------------------- inputs
NNF_CASES = {"a": (64, 96), "b": (57, 83)}      # levels that divide exactly / a level that does not; input seed = B
RUN = dict(n=9, H=56, W=72, window_size=4, seed=11)   # inputs are regenerated from these by the tests


def golden(ref_root):
    ref, cp = load_reference(ref_root)
    out = {}
    for tag, (H, W) in NNF_CASES.items():
        for B in (8, 3):
            sg, tg, ss = nnf_inputs(H, W, B, seed=B)
            cp.random.k = 0
            m = ref.PyramidPatchMatcher(H, W, 3, 5)
            nnf, ts = m.estimate_nnf(sg, tg, ss)
            # the fields and frames are pinned by digest (the arrays would make the file too large to keep in
            # the repository); the batch-3 fields are kept whole, and a few statistics, to show where a mismatch lies
            nnf, ts = np.asarray(nnf).astype(np.int32), np.asarray(ts, np.float32)
            out[f"{tag}{B}_nnf_sha256"], out[f"{tag}{B}_ts_sha256"] = digest(nnf, np.int32), digest(ts, np.float32)
            out[f"{tag}{B}_ts_sum"], out[f"{tag}{B}_ts_max"] = ts.astype(np.float64).sum(), ts.max()
            if B == 3:
                out[f"{tag}{B}_nnf"] = nnf.astype(np.int16)
            out[f"{tag}{B}_draws"] = np.int64(cp.random.k)
    tm = ref.TableManager()
    for n in (1, 2, 5, 9, 16, 17):
        out[f"tasks{n}"] = np.array([[t["source"], t["target"], t["level"]] for t in tm.task_list(n)], np.int64).reshape(-1, 3)
    queries = [(l, r) for r in range(0, 20) for l in (max(r - 4, 0), max(r - 7, 0), 0)]
    out["tree_lr"] = np.array(queries, np.int64)
    out["tree_nodes"] = np.array([len(tm.tree_query(l, r)) for l, r in queries], np.int64)
    out["tree_flat"] = np.array([v for l, r in queries for node in tm.tree_query(l, r) for v in node], np.int64)
    frames = make_frames(RUN["n"], RUN["H"], RUN["W"], seed=RUN["seed"])
    smoother = ref.FastBlendSmoother()
    for B in (8, 3):
        cp.random.k = 0
        res = smoother.run(list(frames), list(frames), B, RUN["window_size"], smoother.ebsynth_config)
        out[f"run{B}"] = np.stack([np.asarray(f) for f in res])
    out["run8_sha256"], out["run3_sha256"] = digest(out["run8"], np.uint8), digest(out["run3"], np.uint8)
    out["run_differ"] = np.int64((out["run8"] != out["run3"]).sum())
    del out["run8"]                                 # run3 stays whole; run8 is pinned by its digest
    np.savez_compressed(os.path.join(HERE, "fastblend_tiny.npz"), **out)
    print("fastblend: run8 vs run3 differ in", int(out["run_differ"]), "bytes;",
          "draws", {k: int(v) for k, v in out.items() if k.endswith("_draws")})


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    golden(ap.parse_args().ref)
