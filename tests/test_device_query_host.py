"""DeviceView::traverse_top_down and bvhNN_build_boxes without a GPU.

The traversal with the caller's node test (include/bvh/v2/cuda/intersect.cuh) compiled by g++ as host code runs on the
golden trees of the unmodified reference with the same node and leaf functions as Bvh<Node>::traverse_top_down of the
C++ surface (tests/device_query_host_test.cpp): per query the same leaf calls in the same order, the same node-function
calls and the same result.  Also: the new exports, the device header as C11, and the Python binding's checks."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tests.conftest import golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDES = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "bvh_b200", "csrc")]
LIB = os.path.join(ROOT, "bvh_b200", "libbvh_c.so")
OVERLAP, CONTAINS, NEAREST, REJECT_ALL, ACCEPT_ALL, ACCEPT_ALL_SWAPPED_ANY = range(6)


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "device_query_host_test")
    src = os.path.join(ROOT, "tests", "device_query_host_test.cpp")
    deps = [src, os.path.join(ROOT, "tests", "device_queries.h"), os.path.join(ROOT, "include", "bvh", "v2", "cuda", "intersect.cuh"),
            os.path.join(ROOT, "include", "bvh", "v2", "b200_surface.h"), os.path.join(ROOT, "include", "bvh_b200_device.h"),
            os.path.join(ROOT, "bvh_b200", "csrc", "traverse_core.cuh"), os.path.join(ROOT, "bvh_b200", "csrc", "core.cuh")]
    if not os.path.exists(out) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(out):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["g++", "-std=gnu++20", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-Wall", "-Werror",
                               *INCLUDES, src, "-o", out])
    return out


def tri_boxes(tris):
    v = tris.reshape(-1, 3, 3)
    return np.concatenate([v.min(axis=1), v.max(axis=1)], axis=1)


def queries(boxes, dtype, seed=3, m=300):
    """Query boxes (min3, max3; the point queries use min3): small and large boxes around primitives, points inside
    primitive boxes, boxes enclosing everything, inverted (empty) boxes and NaN coordinates."""
    rng = np.random.default_rng(seed)
    lo, hi = boxes[:, :3].min(axis=0), boxes[:, 3:].max(axis=0)
    ext = hi - lo
    pick = boxes[rng.integers(boxes.shape[0], size=m)]
    c = (pick[:, :3] + pick[:, 3:]) / 2
    h = ext * (rng.random((m, 1)) ** 3) * 0.3
    q = np.concatenate([c - h, c + h], axis=1)
    kind = np.arange(m) % 8
    q[kind == 1, :3] = q[kind == 1, 3:] = pick[kind == 1, :3] + (pick[kind == 1, 3:] - pick[kind == 1, :3]) * rng.random((int((kind == 1).sum()), 3))
    q[kind == 2] = np.concatenate([lo - 1, hi + 1])
    q[kind == 3] = np.concatenate([c[kind == 3] + h[kind == 3], c[kind == 3] - h[kind == 3]], axis=1)   # inverted
    nan_rows = np.nonzero(kind == 4)[0]
    q[nan_rows, rng.integers(6, size=nan_rows.shape[0])] = np.nan
    q[kind == 5] = np.nan
    q[kind == 6, :3] = lo - ext                                     # points outside the scene
    return q.astype(dtype)


def run_case(exe, tmp_path, bounds, index, prim_ids, boxes, qs):
    dtype = boxes.dtype
    rec = np.dtype([("bounds", dtype, 6), ("index", np.uint32 if dtype == np.float32 else np.uint64)])
    nodes = np.zeros(bounds.shape[0], rec)
    nodes["bounds"], nodes["index"] = bounds, index
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(np.array([nodes.shape[0], prim_ids.shape[0], qs.shape[0]], np.uint64).tobytes())
        f.write(nodes.tobytes())
        f.write(np.asarray(prim_ids, np.uint64).tobytes())
        f.write(np.ascontiguousarray(boxes).tobytes())
        f.write(np.ascontiguousarray(qs).tobytes())
    res = subprocess.run([exe, str(path), "d" if dtype == np.float64 else "f"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = {}
    for line in res.stdout.splitlines():
        m = re.match(r"kind (\d) start (\d) mismatches 0 leaf_calls (\d+) node_calls (\d+) result (\d+)", line)
        if m:
            lines[int(m[1]), int(m[2])] = tuple(int(x) for x in m.groups()[2:])
    assert len(lines) == 18, res.stdout
    return lines


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "box12_f32", "soup1k_f64"])
def test_node_functions_match_reference(exe, tmp_path, name):
    g = golden(name)
    boxes = tri_boxes(g["tris"])
    qs = queries(boxes, boxes.dtype)
    index = g["ref_index"].astype(np.uint64)
    got = run_case(exe, tmp_path, g["ref_bounds"], index, g["ref_prim_ids"], boxes, qs)
    leaves = int(((index & 15) != 0).sum())
    m = qs.shape[0]
    assert got[ACCEPT_ALL, 0][0] == m * leaves                      # every leaf, from the root
    assert got[ACCEPT_ALL, 0][1] == m * (leaves - 1)                # every inner node once
    assert got[REJECT_ALL, 0][0] == 0 and got[REJECT_ALL, 0][1] == m
    assert got[ACCEPT_ALL_SWAPPED_ANY, 0][0] == min(3, leaves) * m
    for kind in (OVERLAP, CONTAINS, NEAREST):
        assert got[kind, 0][0] > 0 and got[kind, 0][2] > 0, kind
    for kind in range(6):                                           # a leaf start: one leaf call, no node test
        assert got[kind, 2][:2] == (m, 0), kind


def test_one_primitive_tree(exe, tmp_path):
    """The root is a leaf: every query kind makes exactly one leaf call and no node-function call."""
    boxes = np.array([[0, 0, 0, 1, 1, 1]], np.float32)
    bounds = np.array([[0, 1, 0, 1, 0, 1]], np.float32)
    qs = queries(np.concatenate([boxes, boxes + 0.5]), np.float32, m=40)
    got = run_case(exe, tmp_path, bounds, np.array([1], np.uint64), np.array([0], np.uint64), boxes, qs)
    for kind in range(6):
        for start in range(3):
            assert got[kind, start][:2] == (40, 0), (kind, start)


def test_library_exports_build_boxes():
    if not os.path.exists(LIB):
        from bvh_b200 import build_ext
        build_ext.build()
    lib = C.CDLL(LIB)
    assert hasattr(lib, "bvh3f_build_boxes") and hasattr(lib, "bvh3d_build_boxes")


def test_device_header_compiles_as_c11():
    src = ("#include <bvh_b200_device.h>\n"
           "struct bvh3f* (*f)(const struct bvh_bbox3f*, const struct bvh_vec3f*, size_t, const struct bvh_build_config*,"
           " unsigned) = bvh3f_build_boxes;\n"
           "struct bvh3d* (*d)(const struct bvh_bbox3d*, const struct bvh_vec3d*, size_t, const struct bvh_build_config*,"
           " unsigned) = bvh3d_build_boxes;\n"
           "int main(void) { return 0; }\n")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), "-x", "c", "-"],
                   input=src, text=True, check=True)


def test_header_compiles_as_host_cxx(tmp_path):
    """traverse_top_down instantiated by plain g++ with a std::tuple node function."""
    src = tmp_path / "only_header.cpp"
    src.write_text("#include <bvh/v2/cuda/intersect.cuh>\n#include <tuple>\n"
                   "int main() {\n"
                   "    bvh::v2::cuda::DeviceView<double> view;\n"
                   "    bvh::v2::cuda::DeviceView<double>::SmallStack<4> stack;\n"
                   "    if (view.nodes) view.traverse_top_down<true>(view.root_index(), stack, [](size_t, size_t) { return true; },\n"
                   "        [](const auto&, const auto&) { return std::make_tuple(true, false, 1); });\n"
                   "    return 0;\n}\n")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", *INCLUDES, str(src)])


def test_binding_checks_shapes():
    """A malformed array or a device address without count and dtype is refused before it reaches the library."""
    from bvh_b200 import api
    b, c = np.zeros((4, 6), np.float32), np.zeros((4, 3), np.float32)
    for bad in ((np.zeros((4, 3), np.float32), c), (b, np.zeros((5, 3), np.float32)), (b, np.zeros((4, 6), np.float32)),
                (np.zeros(24, np.float32), c), (b, 0)):
        with pytest.raises(ValueError):
            api.Bvh.build_boxes(*bad)
    with pytest.raises(ValueError, match="count and dtype"):
        api.Bvh.build_boxes(1 << 20, 2 << 20, flags=api.DEVICE_POINTERS)
    with pytest.raises(ValueError, match="count and dtype"):
        api.Bvh.build_boxes(1 << 20, 2 << 20, count=4, flags=api.DEVICE_POINTERS)
