"""Builds libb200_collective.so (sm_90a, H100) in-tree with nvcc.

    python -m ray_b200.build [--force] [--verbose]

The shared object is written next to this file so it travels with the source tree
(it is git-ignored).  Objects are cached under ray_b200/csrc/build/ keyed by a hash
of the sources and flags, so repeated calls are cheap.
"""
from __future__ import annotations

import concurrent.futures
import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
INCLUDE = PKG_DIR.parent / "include"
BUILD_DIR = CSRC / "build"
LIB_PATH = PKG_DIR / "libb200_collective.so"

SOURCES = ["bootstrap.cu", "allreduce.cu", "allreduce_pipe.cu", "reduce_ops.cu", "copy_ops.cu", "p2p.cu", "grad.cu"]
HEADERS = ["common.cuh", "comm.h", "kernel_utils.cuh", "allreduce_core.cuh", "bulk_copy.cuh", "pipe.h", "policy.h",
           "staged.cuh", "tensor_table.cuh"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "--cudart", "static",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found; libb200_collective.so cannot be built")


def _digest() -> str:
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    for name in HEADERS + SOURCES:
        h.update((CSRC / name).read_bytes())
    h.update((INCLUDE / "b200_collective.h").read_bytes())
    return h.hexdigest()


def _compile_one(nvcc: str, src: str, verbose: bool) -> str:
    obj = BUILD_DIR / (Path(src).stem + ".o")
    cmd = [nvcc, *NVCC_FLAGS, "-I", str(INCLUDE), "-c", str(CSRC / src), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{res.stdout}\n{res.stderr}")
    (BUILD_DIR / (Path(src).stem + ".ptxas.log")).write_text(res.stderr)
    if verbose:
        print(f"[b200 build] compiled {src}")
    return str(obj)


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile (if needed) and return the path of libb200_collective.so."""
    BUILD_DIR.mkdir(parents=True, exist_ok=True)
    stamp = PKG_DIR / "libb200_collective.so.digest"  # next to the .so so it travels with it
    digest = _digest()
    if not force and LIB_PATH.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB_PATH
    nvcc = _nvcc()
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 4)) as ex:
        objs = list(ex.map(lambda s: _compile_one(nvcc, s, verbose), SOURCES))
    cmd = [nvcc, "-shared", "--cudart", "static", "-gencode", "arch=compute_90a,code=sm_90a",
           "-o", str(LIB_PATH), *objs, "-lpthread", "-ldl", "-lrt"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    stamp.write_text(digest)
    if verbose:
        print(f"[b200 build] linked {LIB_PATH}")
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose=True)
    print(p)
