"""The motion forms of DeviceView::trace_triangles and trace_paths, prepare_motion_triangles and triangle_at
(include/bvh/v2/cuda/intersect.cuh) compiled by g++ as host code, no GPU needed.

Each golden tree of the unmodified reference (and box12 and a one-triangle tree) keeps its topology, refitted from the
boxes of prepare_motion_triangles, under key pairs that are equal, translate, turn and scale, move each vertex on its
own, collapse triangles at one end, flip them over the shutter, sit at 1e4, move by a few ulps at 1e4, or hold a
non-finite entry
(tests/device_motion_triangle_host_test.cpp).  Rays and paths carry the times 0, 1, 0.5, 0.3, a random time, -1, 2 and
NaN.  Per ray and per segment, the accept calls (original id, bits of t, u, v), the record and the ray next receives equal
the static trace_triangles with the triangles at that time on the same tree, and the C++ surface's Bvh::intersect with a
PrecomputedTri(triangle_at(...))::intersect leaf, for any-hit and closest-hit, both robust settings, both tie rules and
three filters.  triangle_at gives the keys at 0 and 1; every box holds its triangle at 65 uniform, at adversarial and at
1024 random times, at which the ulps pair's triangles leave the plain union of the key boxes (so the box check sees a
missing or short widening); the centres are tri_bounds_center's at 0.5, and with equal keys boxes and centres are
tri_bounds_center's of the key bit for bit."""
import os
import subprocess

import numpy as np
import pytest

from tests.conftest import golden
from tests.test_device_api_host import extra_rays
from tests.test_device_instance_trace_host import INCLUDES, one_triangle, run_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCENES = ["equal", "translate", "rotscale", "jitter", "collapse", "flip", "offset", "ulps", "non_finite"]


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "device_motion_triangle_host_test")
    src = os.path.join(ROOT, "tests", "device_motion_triangle_host_test.cpp")
    csrc = os.path.join(ROOT, "bvh_b200", "csrc")
    deps = [src, os.path.join(ROOT, "include", "bvh", "v2", "cuda", "intersect.cuh"),
            os.path.join(ROOT, "include", "bvh", "v2", "b200_surface.h"), os.path.join(ROOT, "include", "bvh_b200_device.h")]
    deps += [os.path.join(csrc, f) for f in ("traverse_core.cuh", "core.cuh", "persistent_core.cuh", "trace_plan.h")]
    if not os.path.exists(out) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(out):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["g++", "-std=gnu++20", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-Wall", *INCLUDES,
                               src, "-o", out])
    return out


def lines(log, kind):
    """(scene, filter, mode) -> the words of each `kind` line"""
    out = {}
    for line in log.splitlines():
        w = line.split()
        if w and w[0] == kind:
            out[(w[1], int(w[3]), int(w[5]))] = w
    return out


def union_misses(log, scene):
    """vertices at the checked times outside the union of the key boxes (what the widening is for)"""
    return int(log.split(f"scene {scene} ")[1].split("union misses")[1].split()[0])


def check_log(log, hits=True):
    assert "failures 0" in log, log
    assert "empty batch ok, errors thrown 8 of 8" in log, log
    for scene in SCENES:
        assert f"scene {scene} keys mismatches 0 box misses 0 static box mismatches 0 centre mismatches 0" in log, log
    assert union_misses(log, "equal") == 0, log
    rays_t, paths_t = lines(log, "rays"), lines(log, "paths")
    assert len(rays_t) == len(SCENES) * 3 * 8 and len(paths_t) == len(SCENES) * 3 * 4, log
    if hits:
        for scene in SCENES:
            for mode in range(8):
                assert int(rays_t[(scene, 0, mode)][12]) > 0, (scene, mode, log)      # hits
            for mode in range(4):
                assert int(paths_t[(scene, 0, mode)][17]) > 0, (scene, mode, log)


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "soup1k_f64", "box12_f32"])
def test_motion_equals_static_at_ray_time(exe, tmp_path, name):
    g = golden(name)
    tris = g["tris"]
    rays = np.concatenate([g["rays"][:1536], extra_rays(tris, tris.dtype)])
    log = run_case(exe, tmp_path, [(g["ref_bounds"], g["ref_index"], g["ref_prim_ids"], tris)], rays)
    check_log(log)
    empty = int(log.split("scene non_finite")[1].split("empty boxes")[1].split()[0])
    assert empty == (tris.shape[0] + 6) // 7, log
    # the checked times reach what the rounding of the blend does: without the widening, boxes would miss vertices
    assert union_misses(log, "ulps") > 0, log


def test_one_triangle_tree(exe, tmp_path):
    """A tree whose root is a leaf, with NaN-interval rays."""
    bounds, index, ids, tri = one_triangle(np.float32)
    rays = np.concatenate([np.array([[0.2, 0.2, 1, 0, 0, -1, 0, np.inf], [0.2, 0.2, 1, 0, 0, -1, np.nan, np.inf],
                                     [0.3, 0.3, -1, 0, 0, 1, 0, np.inf], [5, 5, 1, 0, 0, -1, 0, np.inf]], np.float32),
                           extra_rays(tri, np.float32)])
    log = run_case(exe, tmp_path, [(bounds, index, ids, tri)], rays)
    check_log(log, hits=False)
    assert int(lines(log, "rays")[("translate", 0, 0)][12]) > 0, log
