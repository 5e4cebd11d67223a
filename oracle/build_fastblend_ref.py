"""Compile the reference's own FastBlend kernels into oracle/_ref/libfastblend_ref.so (sm_90a), for the GPU tests.

The reference keeps its three kernels as CUDA source strings in diffsynth/extensions/FastBlend/cupy_kernels.py (run
through CuPy's RawKernel).  This recipe reads those strings at build time, adds thin `extern "C"` launchers with the
RawKernel launch shape (8 x 8 threads, grid (ceil(H / 8), ceil(W / 8), batch)) and compiles them with nvcc's defaults
(FMA contraction on, as NVRTC compiles them).  Nothing of the reference enters the repository: the generated source and
the library stay under oracle/_ref/, which git ignores.  Without the reference tree the recipe leaves an existing library
as it is (and builds nothing).

usage:  python oracle/build_fastblend_ref.py [--ref DIR]   (default: $SVI_REFERENCE_ROOT, else /root/reference)
"""
import argparse
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT_DIR, "libfastblend_ref.so")
SOURCE = os.path.join("diffsynth", "extensions", "FastBlend", "cupy_kernels.py")
DEFAULT_REF = os.environ.get("SVI_REFERENCE_ROOT", "/root/reference")   # where the golden recipes look for it too

LAUNCHERS = r'''
static dim3 grid_of(int h, int w, int b) { return dim3((h + 7) / 8, (w + 7) / 8, b); }
extern "C" int ref_remap(int b, int h, int w, int c, int patch, int pad, const float* src, const int* nnf, float* tgt,
                         void* stream) {
  remap<<<grid_of(h, w, b), dim3(8, 8), 0, (cudaStream_t)stream>>>(h, w, c, patch, pad, src, nnf, tgt);
  return (int)cudaGetLastError();
}
extern "C" int ref_patch_error(int b, int h, int w, int c, int patch, int pad, const float* src, const int* nnf,
                               const float* tgt, float* err, void* stream) {
  patch_error<<<grid_of(h, w, b), dim3(8, 8), 0, (cudaStream_t)stream>>>(h, w, c, patch, pad, src, nnf, tgt, err);
  return (int)cudaGetLastError();
}
extern "C" int ref_pairwise_patch_error(int b, int h, int w, int c, int patch, int pad, const float* sa, const int* na,
                                        const float* sb, const int* nb, float* err, void* stream) {
  pairwise_patch_error<<<grid_of(h, w, b), dim3(8, 8), 0, (cudaStream_t)stream>>>(h, w, c, patch, pad, sa, na, sb, nb, err);
  return (int)cudaGetLastError();
}
'''


def build(ref_root=DEFAULT_REF, nvcc="nvcc"):
    try:
        with open(os.path.join(ref_root, SOURCE)) as f:
            text = f.read()
    except OSError:                     # no reference tree here (or not readable): keep what was built before
        return LIB if os.path.exists(LIB) else None
    kernels = re.findall(r"RawKernel\(r'''(.*?)'''", text, re.S)
    if len(kernels) != 3:
        raise RuntimeError(f"{SOURCE}: expected 3 kernel sources, found {len(kernels)}")
    os.makedirs(OUT_DIR, exist_ok=True)
    cu = os.path.join(OUT_DIR, "fastblend_ref.cu")
    text = "#include <cuda_runtime.h>\n" + "\n".join(kernels) + LAUNCHERS
    if os.path.exists(LIB) and os.path.exists(cu) and open(cu).read() == text:
        return LIB
    with open(cu, "w") as f:
        f.write(text)
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-Xcompiler", "-fPIC", "-shared",
                        "-cudart", "shared", cu, "-o", LIB], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("building the reference FastBlend kernels failed:\n" + r.stderr[-4000:])
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default=DEFAULT_REF)
    print(build(ap.parse_args().ref))
