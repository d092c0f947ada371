"""The motion forms of DeviceView::trace_instances and trace_instance_paths, prepare_motion_instances and instance_at
(include/bvh/v2/cuda/intersect.cuh) compiled by g++ as host code, no GPU needed.

The golden trees of the unmodified reference (and box12 and a one-primitive tree) are the bottom meshes, placed by key
pairs that are equal, translate, rotate and scale, pass through a singular placement at one end or at both, or hold a
non-finite entry (tests/device_motion_instance_host_test.cpp).  Rays and paths carry the times 0, 1, 0.5, 0.3, a random
time, -1, 2 and NaN.  Per ray and per segment, the accept calls (instance, original id, bits of t, u, v), the record,
its instance and the world ray next receives equal the static trace_instances over instance_at(records[k], time) on the
same top tree, for any-hit and closest-hit, both robust settings, both tie rules and three filters.  instance_at gives
the keys and prepare_instance's inverses at 0 and 1, and every box of prepare_motion_instances holds the bottom mesh
under the rounded placement at 65 times."""
import os
import subprocess

import numpy as np
import pytest

from tests.conftest import golden
from tests.test_device_api_host import extra_rays
from tests.test_device_instance_trace_host import INCLUDES, one_triangle, run_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCENES = ["equal", "translate", "rotscale", "singular_end", "both_singular", "non_finite"]


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "device_motion_instance_host_test")
    src = os.path.join(ROOT, "tests", "device_motion_instance_host_test.cpp")
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


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "soup1k_f64"])
def test_motion_equals_static_at_ray_time(exe, tmp_path, name):
    g = golden(name)
    tris = g["tris"]
    others = [golden("box12_f32")] if tris.dtype == np.float32 else []
    meshes = [(g["ref_bounds"], g["ref_index"], g["ref_prim_ids"], tris)]
    meshes += [(o["ref_bounds"], o["ref_index"], o["ref_prim_ids"], o["tris"]) for o in others]
    meshes.append(one_triangle(tris.dtype))
    rays = np.concatenate([g["rays"], extra_rays(tris, tris.dtype)])
    log = run_case(exe, tmp_path, meshes, rays)
    assert "failures 0" in log, log
    assert "empty batch ok, errors thrown 6 of 6" in log, log
    for scene in SCENES:
        assert f"scene {scene} keys mismatches 0 box misses 0" in log, log
    assert "scene non_finite keys mismatches 0 box misses 0 empty boxes 2" in log, log
    rays_t, paths_t = lines(log, "rays"), lines(log, "paths")
    assert len(rays_t) == len(SCENES) * 3 * 8 and len(paths_t) == len(SCENES) * 3 * 4, log
    for scene in SCENES:
        for mode in range(8):
            assert int(rays_t[(scene, 0, mode)][9]) > 0, (scene, mode, log)          # hits
        for mode in range(4):
            assert int(paths_t[(scene, 0, mode)][14]) > 0, (scene, mode, log)


def test_one_primitive_mesh(exe, tmp_path):
    """A bottom tree whose root is a leaf, as the only mesh, with NaN-interval rays."""
    bounds, index, ids, tri = one_triangle(np.float32)
    rays = np.concatenate([np.array([[0.2, 0.2, 1, 0, 0, -1, 0, np.inf], [0.2, 0.2, 1, 0, 0, -1, np.nan, np.inf],
                                     [5, 5, 1, 0, 0, -1, 0, np.inf]], np.float32), extra_rays(tri, np.float32)])
    log = run_case(exe, tmp_path, [(bounds, index, ids, tri)], rays)
    assert "failures 0" in log, log
