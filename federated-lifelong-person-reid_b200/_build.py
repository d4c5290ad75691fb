"""In-tree build of the sm_90a native library (``lib/libflpr_b200.so``).

Plain ``nvcc`` (no torch C++ headers: the kernels expose a C ABI and are driven through ``ctypes``), so a full
rebuild takes well under a minute and the resulting ``.so`` travels with the repo snapshot to the GPU box.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_DIR = os.path.join(PKG_DIR, "lib")
OBJ_DIR = os.path.join(PKG_DIR, "build")
LIB_PATH = os.path.join(LIB_DIR, "libflpr_b200.so")
STAMP = os.path.join(LIB_DIR, "build.stamp")

CUDA_SOURCES = ["gemm_wgmma.cu", "fedcomm.cu", "fused_ops.cu", "loss_ops.cu", "layer_ops.cu", "rerank.cu"]
CXX_SOURCES = ["runtime.cpp"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found; cannot build the flpr_b200 native library")
    return cand


def _source_hash() -> str:
    h = hashlib.sha256()
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".cpp", ".h")):
            with open(os.path.join(CSRC, name), "rb") as f:
                h.update(name.encode())
                h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_current() -> bool:
    if not (os.path.exists(LIB_PATH) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as f:
        return f.read().strip() == _source_hash()


def build(force: bool = False, verbose: bool = True) -> str:
    """Compile every native source for sm_90a and link ``libflpr_b200.so``. Returns the library path."""
    if not force and is_current():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    os.makedirs(OBJ_DIR, exist_ok=True)
    nvcc = _nvcc()
    sources = [s for s in CUDA_SOURCES + CXX_SOURCES if os.path.exists(os.path.join(CSRC, s))]

    def compile_one(src: str) -> str:
        obj = os.path.join(OBJ_DIR, os.path.splitext(src)[0] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if src.endswith(".cpp"):
            cmd = [nvcc, "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-x", "cu", "-gencode",
                   "arch=compute_90a,code=sm_90a", "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print("[flpr_b200 build]", " ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return obj

    with ThreadPoolExecutor(max_workers=min(4, len(sources))) as pool:
        objs = list(pool.map(compile_one, sources))
    link = [nvcc, "-shared", "-o", LIB_PATH, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-lpthread"]
    if verbose:
        print("[flpr_b200 build]", " ".join(link), flush=True)
    r = subprocess.run(link, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(STAMP, "w") as f:
        f.write(_source_hash())
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
