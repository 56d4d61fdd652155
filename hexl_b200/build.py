"""In-tree build of libhexl_b200.so (nvcc, sm_90a only).

    python -m hexl_b200.build            # incremental
    python -m hexl_b200.build --force

The shared library has no Python or torch dependency: it is the C-ABI product
(include/hexl_b200.h).  cudart is linked statically, so the only run-time
requirement is the NVIDIA driver.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(PKG, "_obj")
LIB_DIR = os.path.join(PKG, "lib")
LIB = os.path.join(LIB_DIR, "libhexl_b200.so")

SOURCES = ["capi.cu", "capi_ntt.cu", "capi_eltwise.cu", "capi_keyswitch.cu", "capi_galois.cu", "capi_hybrid.cu",
           "ntt.cu", "ntt_multi.cu", "eltwise.cu", "seal.cu", "galois.cu", "rns.cu", "bfv.cu", "capi_bfv.cu",
           "plain.cu", "capi_plain.cu", "numtheory.cpp"]
HEADERS = ["capi.h", "internal.h", "modarith.cuh", "ntt_kernels.cuh", "galois.cuh", "hybrid_rotation.h", "numtheory.h",
           os.path.join(ROOT, "include", "hexl_b200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-std=c++17", "-O3", "-lineinfo", "-diag-suppress=177",
    "-Xcompiler", "-fPIC,-Wall",
    "-Xptxas", "-v",
]


def nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _newer(target: str, deps) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps)


def _compile(src: str, force: bool) -> str:
    path = os.path.join(CSRC, src)
    obj = os.path.join(OBJ, os.path.splitext(src)[0] + ".o")
    deps = [path] + [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    if not force and _newer(obj, deps):
        return obj
    cmd = [nvcc()] + NVCC_FLAGS + ["-c", path, "-o", obj]
    res = subprocess.run(cmd, capture_output=True, text=True)
    with open(obj + ".log", "w") as f:  # ptxas -v output: registers / spills per kernel
        f.write(res.stdout + res.stderr)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError(f"nvcc failed on {src}")
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(LIB_DIR, exist_ok=True)
    with ThreadPoolExecutor(max_workers=4) as ex:
        objs = list(ex.map(lambda s: _compile(s, force), SOURCES))
    if force or not _newer(LIB, objs):
        cmd = [nvcc(), "-shared", "-o", LIB] + objs + ["-Xlinker", "--exclude-libs,ALL"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
            raise RuntimeError("link failed")
    if verbose:
        print(LIB)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
