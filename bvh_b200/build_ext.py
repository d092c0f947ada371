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


TEST_KERNELS_SRC = os.path.join(ROOT, "tests", "device_api_kernels.cu")
TEST_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_api_kernels.so")
QUERY_KERNELS_SRC = os.path.join(ROOT, "tests", "device_query_kernels.cu")
QUERY_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_query_kernels.so")
BOTTOM_UP_KERNELS_SRC = os.path.join(ROOT, "tests", "device_bottom_up_kernels.cu")
BOTTOM_UP_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_bottom_up_kernels.so")


def _build_test_kernels(src: str, out: str, force: bool, verbose: bool) -> str:
    """Compiles test kernels that use the device traversal API (src) into tests/_build/ (out), linked against the
    library, with the library's flags (C++20: the files also include the C++ surface header; x86-64-v3 host code).
    Rebuilt when stale and nvcc is present; an existing build is used as it is otherwise."""
    deps = [src, LIB, os.path.abspath(__file__), os.path.join(ROOT, "include", "bvh", "v2", "cuda", "intersect.cuh"),
            os.path.join(ROOT, "include", "bvh", "v2", "b200_surface.h")] + _deps()
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    fresh = os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(f) for f in deps if os.path.exists(f))
    if not force and os.path.exists(out) and (fresh or not os.path.exists(nvcc)):
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    flags = ["-std=c++20" if f == "-std=c++17" else f for f in NVCC_FLAGS]
    # the host half runs the C++ surface's Bvh::intersect, whose fast slab test is one FMA only where the target has one
    # (fast_mul_add, FP_FAST_FMAF), as the device's is
    flags += ["-Xcompiler", "-march=x86-64-v3"]
    cmd = [nvcc, *flags, "-shared", src, "-o", out, "-L", HERE, "-lbvh_c", "-Xlinker", "-rpath,$ORIGIN/../../bvh_b200"]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0 or verbose:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed on {os.path.relpath(src, ROOT)}")
    return out


def build_device_api_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_api_kernels.cu: the device traversal API's ray test kernels."""
    return _build_test_kernels(TEST_KERNELS_SRC, TEST_KERNELS_LIB, force, verbose)


def build_device_query_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_query_kernels.cu: the test kernels of DeviceView::traverse_top_down (box overlap, nearest point)."""
    return _build_test_kernels(QUERY_KERNELS_SRC, QUERY_KERNELS_LIB, force, verbose)


def build_device_bottom_up_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_bottom_up_kernels.cu: the test kernels of DeviceView::traverse_bottom_up (counts and boxes, mass and
    centre, Barnes-Hut through the three-argument node test)."""
    return _build_test_kernels(BOTTOM_UP_KERNELS_SRC, BOTTOM_UP_KERNELS_LIB, force, verbose)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
