"""Builds the CUDA library in-tree for H100 (sm_90a); nvcc cross-compiles without a GPU.

Output: opensfm_b200/lib/libopensfm_b200.so (git-ignored build product).
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libopensfm_b200.so")
SOURCES = ["core.cu", "match.cu", "match_tc.cu", "words.cu", "vlad.cu", "bow.cu", "tracks.cu", "triangulate.cu", "rotransac.cu", "resect.cu", "relpose.cu", "ba.cu", "dense.cu", "undistort.cu"]
# per-source flags: dense.cu and undistort.cu are checked bit for bit against host restatements, so no product may
# become an FMA
SOURCE_FLAGS = {"dense.cu": ["-fmad=false"], "undistort.cu": ["-fmad=false"]}
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [ "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "opensfm_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src: str) -> str:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + SOURCE_FLAGS.get(src, []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        subprocess.check_call(cmd)
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ARCH + ["-ccbin", "/usr/bin/g++", "-cudart", "static", "-ldl"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
