"""DeviceView::trace_paths (include/bvh/v2/cuda/intersect.cuh) compiled by g++ as host code, no GPU needed.

On the golden trees of the unmodified reference and on a one-primitive tree, a recording shader runs 160 scripted paths
of 0 to 64 segments each, mixing Closest and Occlusion segments over the golden rays plus NaN-interval, zero and
axis-parallel rays.  Every segment gets the accept calls a host leaf loop makes inside Bvh<Node>::intersect of the C++
surface (PrecomputedTri::intersect, the same tie rule, the same filter) with IsAnyHit set for occlusion segments, in the
same order and with the same id, t, u and v, and next receives the same record and the scripted ray unchanged; start and
finish are called once per path.  Both robust settings and both tie rules (tests/device_path_trace_host_test.cpp)."""
import os
import subprocess

import numpy as np
import pytest

from tests.conftest import golden
from tests.test_device_api_host import extra_rays
from tests.test_device_triangle_trace_host import INCLUDES, ROOT, run_case

MODES = 4


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "device_path_trace_host_test")
    src = os.path.join(ROOT, "tests", "device_path_trace_host_test.cpp")
    csrc = os.path.join(ROOT, "bvh_b200", "csrc")
    deps = [src, os.path.join(ROOT, "include", "bvh", "v2", "cuda", "intersect.cuh"),
            os.path.join(ROOT, "include", "bvh", "v2", "b200_surface.h"), os.path.join(ROOT, "include", "bvh_b200_device.h")]
    deps += [os.path.join(csrc, f) for f in ("traverse_core.cuh", "core.cuh", "persistent_core.cuh", "trace_plan.h")]
    if not os.path.exists(out) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(out):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["g++", "-std=gnu++20", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-Wall", *INCLUDES,
                               src, "-o", out])
    return out


def table(log):
    """mode -> (segments, occlusion segments, NaN segments, hits, accept calls)"""
    out = {}
    for line in log.splitlines():
        w = line.split()
        if w and w[0] == "mode":
            out[int(w[1])] = (int(w[3]), int(w[5]), int(w[7]), int(w[-4]), int(w[-1]))
    return out


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "box12_f32", "soup1k_f64"])
def test_trace_paths_matches_host_leaf_loop(exe, tmp_path, name):
    g = golden(name)
    tris = g["tris"]
    rays = np.concatenate([g["rays"], extra_rays(tris, tris.dtype)])
    log = run_case(exe, tmp_path, g["ref_bounds"], g["ref_index"], g["ref_prim_ids"], tris, rays)
    assert "empty batch ok, small workspace throws, null workspace throws, deep tree throws, no triangles throws" in log, log
    assert "failures 0" in log, log
    t = table(log)
    assert len(t) == MODES, log
    for mode in range(MODES):
        segments, occlusion, nan, hits, calls = t[mode]
        assert segments > 3000 and 0.3 < occlusion / segments < 0.7, log    # both kinds, mixed within paths
        assert hits > 0 and calls >= hits, log


def test_one_primitive_tree(exe, tmp_path):
    """The root is a leaf: rays through the triangle hit it in both segment kinds; NaN-interval rays get no accept call."""
    tri = np.array([[0, 0, 0, 1, 0, 0, 0, 1, 0]], np.float32)
    bounds = np.array([[0, 1, 0, 1, 0, 0]], np.float32)
    index = np.array([1], np.uint64)
    rays = np.array([[0.2, 0.2, 1, 0, 0, -1, 0, np.inf], [0.2, 0.2, 1, 0, 0, -1, np.nan, np.inf],
                     [0.1, 0.3, -1, 0, 0, 1, 0, np.inf], [0.2, 0.2, 1, 0, 0, -1, 0, np.nan], [5, 5, 1, 0, 0, -1, 0, np.inf]],
                    np.float32)
    log = run_case(exe, tmp_path, bounds, index, np.array([0], np.uint64), tri, rays)
    assert "failures 0" in log, log
    t = table(log)
    for mode in range(MODES):
        segments, occlusion, nan, hits, calls = t[mode]
        assert nan > 0 and hits > 0 and calls == hits, log      # one candidate per hitting segment, none on NaN ones
