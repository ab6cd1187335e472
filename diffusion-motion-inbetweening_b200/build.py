"""Build libcondmdi_b200.so (sm_90a, H100) in-tree with nvcc.

The library is the product: every kernel of the sampling path plus the C ABI of include/condmdi_b200.h.
It is compiled here (nvcc cross-compiles without a GPU) and travels to the GPU box with the tree.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libcondmdi_b200.so")
SOURCES = ["gemm2.cu", "gemm_chain.cu", "attention.cu", "elementwise.cu", "unet_kernels.cu", "backward.cu", "attention_bwd_tc.cu", "attention_bwd_simt_test.cu", "tma_host.cu", "capi_test.cu", "engine.cu"]
HEADERS = ["common.cuh", "kernels.h", "gemm_epilogue.cuh", "engine_unet.inc", os.path.join("..", "..", "include", "condmdi_b200.h")]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA extension cannot be built (there is no CPU fallback)")


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(ARCH + FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = [os.path.join(CSRC, h) for h in HEADERS] + [os.path.join(CSRC, s) for s in srcs]
    stamp = os.path.join(BUILD, "stamp.txt")
    digest = _digest(deps)
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == digest:
        return LIB
    nvcc = _nvcc()

    def compile_one(src: str) -> str:
        obj = os.path.join(BUILD, src.replace(".cu", ".o"))
        cmd = [nvcc, *ARCH, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [nvcc, *ARCH, "-shared", "-o", LIB, *objs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
