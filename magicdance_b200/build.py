"""Builds the sm_90a kernel library (C ABI, include/magicdance_b200.h) in-tree with nvcc.

nvcc cross-compiles without a GPU, so this runs in the CPU-only build container; the resulting
magicdance_b200/lib/libmagicdance_b200.so travels to the GPU box with the repo snapshot.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB_DIR = os.path.join(PKG, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libmagicdance_b200.so")
STAMP = os.path.join(LIB_DIR, "build.stamp")
SOURCES = ["gemm.cu", "gemm_bwd.cu", "attention.cu", "attention_bwd.cu", "norm.cu", "norm_bwd.cu", "conv_bwd.cu", "misc.cu"]
HEADERS = ["common.cuh", "wgmma.cuh", "norm.cuh", os.path.join("..", "..", "include", "magicdance_b200.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC or put /usr/local/cuda/bin on PATH)")


def _digest() -> str:
    h = hashlib.sha256()
    for rel in SOURCES + HEADERS:
        with open(os.path.join(CSRC, rel), "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_fresh() -> bool:
    if not (os.path.isfile(LIB_PATH) and os.path.isfile(STAMP)):
        return False
    with open(STAMP) as f:
        return f.read().strip() == _digest()


def _file_digest(src: str) -> str:
    h = hashlib.sha256()
    for rel in [src] + HEADERS:
        with open(os.path.join(CSRC, rel), "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu into lib/libmagicdance_b200.so; returns the library path.  Translation units are
    compiled in parallel and cached per source digest (lib/obj/*.o), then linked."""
    if not force and is_fresh():
        return LIB_PATH
    from concurrent.futures import ThreadPoolExecutor
    obj_dir = os.path.join(LIB_DIR, "obj")
    os.makedirs(obj_dir, exist_ok=True)
    cflags = [f for f in NVCC_FLAGS if f != "-shared"]

    def compile_one(src):
        obj = os.path.join(obj_dir, src.replace(".cu", ".o"))
        stamp = obj + ".stamp"
        dig = _file_digest(src)
        if not force and os.path.isfile(obj) and os.path.isfile(stamp) and open(stamp).read().strip() == dig:
            return obj, ""
        cmd = [_nvcc()] + cflags + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj, src]
        proc = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
        if proc.returncode != 0:
            raise RuntimeError(f"nvcc failed ({' '.join(cmd)}):\n{proc.stdout}\n{proc.stderr}")
        with open(stamp, "w") as f:
            f.write(dig)
        return obj, proc.stderr

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        results = list(ex.map(compile_one, SOURCES))
    if verbose:
        for _, err in results:
            print(err)
    cmd = [_nvcc(), "-shared", "-o", LIB_PATH] + [o for o, _ in results]
    proc = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"link failed ({' '.join(cmd)}):\n{proc.stdout}\n{proc.stderr}")
    with open(STAMP, "w") as f:
        f.write(_digest())
    return LIB_PATH


if __name__ == "__main__":
    print(build(force=True, verbose=True))
