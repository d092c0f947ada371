"""prepare_motion_nodes, node_at and the motion-node forms of DeviceView::trace_triangles and trace_paths
(include/bvh/v2/cuda/intersect.cuh) compiled by g++ as host code, no GPU needed.

Each golden tree of the unmodified reference (and box12 and a one-triangle tree) keeps its topology, refitted from the
boxes of prepare_motion_triangles, and gets its motion nodes from prepare_motion_nodes under the deforming-mesh host
test's nine kinds of key pair and one with part of the mesh static (tests/device_motion_nodes_host_test.cpp).  Rays and paths carry the times 0, 1, 0.5, 0.3,
a random time, -1, 2 and NaN.  Per ray and per segment, the accept calls (original id, bits of t, u, v), the record and
the ray next receives equal the motion call without motion nodes and the C++ surface's Bvh::intersect with a triangle_at
leaf, both on a copy of the tree whose node bounds are node_at at that time, for any-hit and closest-hit, both robust
settings, both tie rules and three filters; a view whose node bounds are NaN gives the same, and robust closest-hit
records with canonical ties equal the motion call on the shutter-box tree.  With equal keys both keys
of every record are the refitted bounds bit for bit and the call is the motion call on the shutter-box tree.  Every
node_at box holds its subtree's triangles at 65 uniform, at adversarial and at 1024 random times, at which the ulps
pair's triangles leave the blend of the unwidened key boxes (so the check sees a missing or short widening).  A small
tree where a static leaf and a moving one meet at one key, under 500 offsets and 1000 times each, checks that the
parent's box holds the static vertex and that a ray down the static edge keeps its hit."""
import os
import subprocess

import pytest

from tests.conftest import golden
from tests.test_device_api_host import extra_rays
from tests.test_device_instance_trace_host import INCLUDES, one_triangle, run_case

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCENES = ["equal", "translate", "rotscale", "jitter", "collapse", "flip", "offset", "ulps", "non_finite", "partial"]


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "device_motion_nodes_host_test")
    src = os.path.join(ROOT, "tests", "device_motion_nodes_host_test.cpp")
    csrc = os.path.join(ROOT, "bvh_b200", "csrc")
    deps = [src, os.path.join(ROOT, "include", "bvh", "v2", "cuda", "intersect.cuh"),
            os.path.join(ROOT, "include", "bvh", "v2", "b200_surface.h"), os.path.join(ROOT, "include", "bvh_b200_device.h")]
    deps += [os.path.join(csrc, f) for f in ("traverse_core.cuh", "core.cuh", "persistent_core.cuh", "trace_plan.h",
                                             "refit_core.cuh")]
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


def scene_count(log, scene, what):
    return int(log.split(f"scene {scene} ")[1].split(what)[1].split()[0])


def check_log(log, hits=True):
    assert "failures 0" in log, log
    assert "empty batch ok, errors thrown 11 of 11" in log, log
    # a static leaf beside a moving one whose bound meets it at one key: their parent's blended bound must not pass the
    # static vertex, and rays down the static edge keep their hit
    assert "meet box misses 0 lost hits 0" in log, log
    for scene in SCENES:
        assert (f"scene {scene} index mismatches 0 equal-key mismatches 0 box misses 0 empty misses 0 nan bounds 0"
                in log), log
    assert scene_count(log, "equal", "plain misses") == 0, log
    rays_t, paths_t = lines(log, "rays"), lines(log, "paths")
    assert len(rays_t) == len(SCENES) * 3 * 8 and len(paths_t) == len(SCENES) * 3 * 4, log
    if hits:
        for scene in SCENES:
            for mode in range(8):
                assert int(rays_t[(scene, 0, mode)][15]) > 0, (scene, mode, log)      # hits
            for mode in range(4):
                assert int(paths_t[(scene, 0, mode)][17]) > 0, (scene, mode, log)


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "soup1k_f64", "grid2k_f64", "box12_f32"])
def test_motion_nodes_equal_tree_at_ray_time(exe, tmp_path, name):
    g = golden(name.replace("grid2k_f64", "grid2k_f32"))
    dtype = np.float64 if name.endswith("f64") else np.float32      # grid2k_f64: the float grid and its tree in double
    tris = g["tris"].astype(dtype)
    rays = np.concatenate([g["rays"][:1536].astype(dtype), extra_rays(tris, dtype)])
    log = run_case(exe, tmp_path, [(g["ref_bounds"].astype(dtype), g["ref_index"], g["ref_prim_ids"], tris)], rays)
    check_log(log)
    # the checked times reach what the rounding of the two blends does: without the widening, node boxes would miss
    # triangles.  That takes a leaf whose extreme coordinate comes from different vertices at the two keys, vertices a
    # few ulps apart: the grid's shared vertices in both precisions, and the float soup's close vertices at 1e4 (the
    # double soup has none so close)
    if name != "soup1k_f64":
        assert scene_count(log, "ulps", "plain misses") > 0, log


def test_one_triangle_tree(exe, tmp_path):
    """A tree whose root is a leaf, with NaN-interval rays."""
    bounds, index, ids, tri = one_triangle(np.float32)
    rays = np.concatenate([np.array([[0.2, 0.2, 1, 0, 0, -1, 0, np.inf], [0.2, 0.2, 1, 0, 0, -1, np.nan, np.inf],
                                     [0.3, 0.3, -1, 0, 0, 1, 0, np.inf], [5, 5, 1, 0, 0, -1, 0, np.inf]], np.float32),
                           extra_rays(tri, np.float32)])
    log = run_case(exe, tmp_path, [(bounds, index, ids, tri)], rays)
    check_log(log, hits=False)
    assert int(lines(log, "rays")[("translate", 0, 0)][15]) > 0, log
