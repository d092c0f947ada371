"""Compiles the CUDA engine into ``bvh_b200/libbvh_c.so`` (in-tree, so that it travels with the
repository tree).  sm_90a (H100) only; nvcc cross-compiles without a GPU.

    python -m bvh_b200.build_ext [--force] [--verbose]
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
# A/B builds (experiments): BVH_B200_BUILD_TAG=x BVH_B200_EXTRA_NVCC="-DFOO=1" -> bvh_b200/libbvh_c_x.so, selected at
# run time with BVH_B200_LIB=<path> (bvh_b200/api.py)
TAG = os.environ.get("BVH_B200_BUILD_TAG", "")
OBJ = os.path.join(HERE, "build" + ("_" + TAG if TAG else ""))
LIB = os.path.join(HERE, "libbvh_c" + ("_" + TAG if TAG else "") + ".so")

SOURCES = ["lbvh_build.cu", "traverse.cu", "c_api.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--fmad=false",                      # parity arithmetic is written with explicit *_rn intrinsics; never contract the rest either
    "-Xcompiler", "-fPIC,-ffp-contract=off,-fvisibility=hidden,-Wall,-Wno-unused-function",
    "-I", os.path.join(ROOT, "include"), "-I", CSRC,
]


def _deps():
    out = []
    for d in (CSRC, os.path.join(ROOT, "include"), os.path.join(ROOT, "include", "bvh", "v2", "c_api")):
        out += [os.path.join(d, f) for f in os.listdir(d) if f.endswith((".cu", ".cuh", ".h"))]
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    newest = max(os.path.getmtime(f) for f in _deps() + [os.path.abspath(__file__)])
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= newest:
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(OBJ, exist_ok=True)

    def compile_one(src):
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, *os.environ.get("BVH_B200_EXTRA_NVCC", "").split(), "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), flush=True)
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0 or verbose:
            sys.stderr.write(res.stdout + res.stderr)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}")
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as pool:
        objs = list(pool.map(compile_one, SOURCES))
    cmd = [nvcc, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
