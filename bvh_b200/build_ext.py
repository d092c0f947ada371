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
TRACE_KERNELS_SRC = os.path.join(ROOT, "tests", "device_trace_kernels.cu")
TRACE_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_trace_kernels.so")
QUERY_BATCH_KERNELS_SRC = os.path.join(ROOT, "tests", "device_query_batch_kernels.cu")
QUERY_BATCH_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_query_batch_kernels.so")
TRIANGLE_TRACE_KERNELS_SRC = os.path.join(ROOT, "tests", "device_triangle_trace_kernels.cu")
TRIANGLE_TRACE_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_triangle_trace_kernels.so")
PATH_TRACE_KERNELS_SRC = os.path.join(ROOT, "tests", "device_path_trace_kernels.cu")
PATH_TRACE_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_path_trace_kernels.so")
INSTANCE_TRACE_KERNELS_SRC = os.path.join(ROOT, "tests", "device_instance_trace_kernels.cu")
INSTANCE_TRACE_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_instance_trace_kernels.so")
INSTANCE_PATH_TRACE_KERNELS_SRC = os.path.join(ROOT, "tests", "device_instance_path_trace_kernels.cu")
INSTANCE_PATH_TRACE_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_instance_path_trace_kernels.so")
MOTION_INSTANCE_KERNELS_SRC = os.path.join(ROOT, "tests", "device_motion_instance_kernels.cu")
MOTION_INSTANCE_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_motion_instance_kernels.so")
MOTION_TRIANGLE_KERNELS_SRC = os.path.join(ROOT, "tests", "device_motion_triangle_kernels.cu")
MOTION_TRIANGLE_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_motion_triangle_kernels.so")
MOTION_NODES_KERNELS_SRC = os.path.join(ROOT, "tests", "device_motion_nodes_kernels.cu")
MOTION_NODES_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_motion_nodes_kernels.so")
DEFORMING_INSTANCE_KERNELS_SRC = os.path.join(ROOT, "tests", "device_deforming_instance_kernels.cu")
DEFORMING_INSTANCE_KERNELS_LIB = os.path.join(ROOT, "tests", "_build", "libdevice_deforming_instance_kernels.so")


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


def build_device_trace_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_trace_kernels.cu: the test tracers of DeviceView::trace (triangles, spheres, leaf-call recorders)
    and the same tracers one thread per ray."""
    return _build_test_kernels(TRACE_KERNELS_SRC, TRACE_KERNELS_LIB, force, verbose)


def build_device_query_batch_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_query_batch_kernels.cu: the test queriers of DeviceView::query (overlap, nearest, containment,
    Barnes-Hut) and the same queriers one thread per query."""
    return _build_test_kernels(QUERY_BATCH_KERNELS_SRC, QUERY_BATCH_KERNELS_LIB, force, verbose)


def build_device_triangle_trace_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_triangle_trace_kernels.cu: the test shaders of DeviceView::trace_triangles (recording filters, the
    plain array shader, an in-kernel camera) and the same filters one thread per ray."""
    return _build_test_kernels(TRIANGLE_TRACE_KERNELS_SRC, TRIANGLE_TRACE_KERNELS_LIB, force, verbose)


def build_device_path_trace_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_path_trace_kernels.cu: the test shaders of DeviceView::trace_paths (a path tracer with next-event
    shadow segments, as one call and as a wavefront loop of trace_triangles; a recording shader of scripted segments)
    and the same segments one thread each."""
    return _build_test_kernels(PATH_TRACE_KERNELS_SRC, PATH_TRACE_KERNELS_LIB, force, verbose)


def build_device_instance_trace_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_instance_trace_kernels.cu: the test shaders of DeviceView::trace_instances and prepare_instances (a
    recording shader, the same rays nested by hand one thread each, the benchmark's plain shaders and a hand-nested
    DeviceView::trace tracer)."""
    return _build_test_kernels(INSTANCE_TRACE_KERNELS_SRC, INSTANCE_TRACE_KERNELS_LIB, force, verbose)


def build_device_instance_path_trace_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_instance_path_trace_kernels.cu: the test shaders of DeviceView::trace_instance_paths (a path tracer
    with next-event shadow segments over placed meshes, as one call, as a wavefront loop of trace_instances and as
    trace_paths on one mesh; a recording shader of scripted segments) and the same segments nested by hand one thread
    each."""
    return _build_test_kernels(INSTANCE_PATH_TRACE_KERNELS_SRC, INSTANCE_PATH_TRACE_KERNELS_LIB, force, verbose)


def build_device_motion_instance_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_motion_instance_kernels.cu: the test shaders of the motion forms of DeviceView::trace_instances and
    trace_instance_paths, prepare_motion_instances and instance_at (a recording shader with a time per ray, the same
    rays nested by hand one thread each, a path tracer with a time per path as one call and as a wavefront loop, the
    benchmark's plain shader)."""
    return _build_test_kernels(MOTION_INSTANCE_KERNELS_SRC, MOTION_INSTANCE_KERNELS_LIB, force, verbose)


def build_device_motion_triangle_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_motion_triangle_kernels.cu: the test shaders of the motion forms of DeviceView::trace_triangles and
    trace_paths, prepare_motion_triangles and triangle_at (a recording shader with a time per ray, the same rays nested
    by hand one thread each, a path tracer with a time per path as one call, as a wavefront loop and as the static call,
    the benchmark's plain shader and traversal counts)."""
    return _build_test_kernels(MOTION_TRIANGLE_KERNELS_SRC, MOTION_TRIANGLE_KERNELS_LIB, force, verbose)


def build_device_motion_nodes_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_motion_nodes_kernels.cu: the test shaders of prepare_motion_nodes, node_at and the motion-node forms
    of DeviceView::trace_triangles and trace_paths (the deforming-mesh recording shader and path tracer, one thread per
    ray through a node_at node test, subtree extents for containment, the benchmark's plain shader)."""
    return _build_test_kernels(MOTION_NODES_KERNELS_SRC, MOTION_NODES_KERNELS_LIB, force, verbose)


def build_device_deforming_instance_tests(force: bool = False, verbose: bool = False) -> str:
    """tests/device_deforming_instance_kernels.cu: the test shaders of the deforming forms of DeviceView::trace_instances
    and trace_instance_paths, make_deforming_instance and prepare_deforming_instances (a recording shader with a time
    per ray, the same rays nested by hand one thread each, the motion and triangle calls they reduce to, scripted paths,
    the benchmark's plain shader)."""
    return _build_test_kernels(DEFORMING_INSTANCE_KERNELS_SRC, DEFORMING_INSTANCE_KERNELS_LIB, force, verbose)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
