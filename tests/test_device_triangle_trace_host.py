"""DeviceView::trace_triangles (include/bvh/v2/cuda/intersect.cuh) compiled by g++ as host code, no GPU needed.

On the golden trees of the unmodified reference and on a one-primitive tree, a recording shader gets per ray the accept
calls a host leaf loop makes inside Bvh<Node>::intersect of the C++ surface (PrecomputedTri::intersect, the same tie rule,
the same filter), in the same order and with the same id, t, u and v, and its finish receives the same record, for
closest-hit, any-hit and robust rays under both tie rules, five filters, NaN-interval rays and zero and axis-parallel
directions (tests/device_triangle_trace_host_test.cpp).  With every hit accepted the records also equal the host
emulation's traverse_ray, the library kernels' own traversal."""
import os
import subprocess

import numpy as np
import pytest

from tests.conftest import golden
from tests.test_device_api_host import extra_rays

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDES = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "bvh_b200", "csrc")]
FILTERS = 5
MODES = 8


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "device_triangle_trace_host_test")
    src = os.path.join(ROOT, "tests", "device_triangle_trace_host_test.cpp")
    csrc = os.path.join(ROOT, "bvh_b200", "csrc")
    deps = [src, os.path.join(ROOT, "include", "bvh", "v2", "cuda", "intersect.cuh"),
            os.path.join(ROOT, "include", "bvh", "v2", "b200_surface.h"), os.path.join(ROOT, "include", "bvh_b200_device.h")]
    deps += [os.path.join(csrc, f) for f in ("traverse_core.cuh", "core.cuh", "persistent_core.cuh", "trace_plan.h")]
    if not os.path.exists(out) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(out):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["g++", "-std=gnu++20", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-Wall", *INCLUDES,
                               src, "-o", out])
    return out


def run_case(exe, tmp_path, bounds, index, prim_ids, tris, rays):
    dtype = tris.dtype
    rec = np.dtype([("bounds", dtype, 6), ("index", np.uint32 if dtype == np.float32 else np.uint64)])
    nodes = np.zeros(bounds.shape[0], rec)
    nodes["bounds"], nodes["index"] = bounds, index
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(np.array([nodes.shape[0], prim_ids.shape[0], rays.shape[0]], np.uint64).tobytes())
        f.write(nodes.tobytes())
        f.write(prim_ids.astype(np.uint64).tobytes())
        f.write(np.ascontiguousarray(tris).tobytes())
        f.write(np.ascontiguousarray(rays).tobytes())
    res = subprocess.run([exe, str(path), "d" if dtype == np.float64 else "f"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return res.stdout


def table(log):
    """(filter, mode) -> (hits, accept calls) of the whole batch"""
    out = {}
    for line in log.splitlines():
        w = line.split()
        if w and w[0] == "filter":
            out[(int(w[1]), int(w[3]))] = (int(w[-4]), int(w[-1]))
    return out


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "box12_f32", "soup1k_f64"])
def test_trace_triangles_matches_host_leaf_loop(exe, tmp_path, name):
    g = golden(name)
    tris = g["tris"]
    rays = np.concatenate([g["rays"], extra_rays(tris, tris.dtype)])
    log = run_case(exe, tmp_path, g["ref_bounds"], g["ref_index"], g["ref_prim_ids"], tris, rays)
    assert "empty batch ok, small workspace throws, null workspace throws, no triangles throws" in log, log
    t = table(log)
    assert len(t) == FILTERS * MODES, log
    for mode in range(MODES):
        hits, calls = t[(0, mode)]
        assert hits > 0 and calls >= hits, (mode, log)
        assert t[(1, mode)][0] == 0, log                         # reject-all: every ray misses ...
        assert t[(1, mode)][1] >= hits, log                      # ... after at least as many candidates
        if name != "box12_f32":
            # the filters change something: odd ids, the cut-out and the origin triangle are each dropped somewhere
            for f in (2, 3, 4):
                assert t[(f, mode)] != t[(0, mode)], (f, mode, log)


def test_one_primitive_tree(exe, tmp_path):
    """The root is a leaf: a ray through the triangle gets one accept call; NaN-interval rays get none."""
    tri = np.array([[0, 0, 0, 1, 0, 0, 0, 1, 0]], np.float32)
    bounds = np.array([[0, 1, 0, 1, 0, 0]], np.float32)
    index = np.array([1], np.uint64)
    rays = np.concatenate([np.array([[0.2, 0.2, 1, 0, 0, -1, 0, np.inf], [0.2, 0.2, 1, 0, 0, -1, np.nan, np.inf],
                                     [5, 5, 1, 0, 0, -1, 0, np.inf]], np.float32), extra_rays(tri, np.float32)])
    log = run_case(exe, tmp_path, bounds, index, np.array([0], np.uint64), tri, rays)
    t = table(log)
    for mode in range(MODES):
        assert t[(0, mode)][0] >= 1, log
        assert t[(1, mode)][0] == 0, log
        assert t[(4, mode)][0] == 0, log                         # the only triangle is every hitting ray's origin
