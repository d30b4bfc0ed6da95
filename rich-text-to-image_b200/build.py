"""In-tree build of the sm_90a C-ABI library (librtti_b200.so) with nvcc.

nvcc cross-compiles without a GPU; the resulting .so sits next to this file (git-ignored), so the package is
importable from the repository tree.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
BUILD_DIR = os.path.join(PKG_DIR, "build")
LIB_PATH = os.path.join(PKG_DIR, "librtti_b200.so")
SOURCES = ["common.cu", "elementwise.cu", "attn_fwd.cu", "gemm_geglu.cu", "attn_probs_mean.cu", "gather_blend.cu", "vae_kernels.cu", "stripe_exchange.cu", "peer_push.cu", "kmeans.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _newer(src_paths, out):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(s) > t for s in src_paths)


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ for sm_90a and link librtti_b200.so. Returns the library path."""
    os.makedirs(BUILD_DIR, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(PKG_DIR, "..", "include", "rtti_b200.h"))
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    nvcc = _nvcc()

    def compile_one(src):
        obj = os.path.join(BUILD_DIR, src.replace(".cu", ".o"))
        spath = os.path.join(CSRC, src)
        if force or _newer([spath] + headers, obj):
            cmd = [nvcc] + NVCC_FLAGS + ["-c", spath, "-o", obj]
            if verbose:
                print(" ".join(cmd), flush=True)
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    if force or _newer(objs, LIB_PATH):
        cmd = [nvcc, "-shared", "-o", LIB_PATH] + objs + ["-cudart", "static"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
