"""DeviceView::trace_instance_paths (include/bvh/v2/cuda/intersect.cuh) compiled by g++ as host code, no GPU needed.

The golden trees of the unmodified reference (and box12 and a one-primitive tree) are the bottom meshes.  Placed by
identity, translation, power-of-two scale, axis permutation, rotation and singular matrices, prepared with
prepare_instances and topped by a tree over the prepared boxes, a recording shader runs scripted paths of 0 to 64 mixed
Closest and Occlusion segments, NaN-interval and axis-parallel rays included
(tests/device_instance_path_trace_host_test.cpp).  Per segment, the accept calls (instance, original id, bits of t, u,
v), the record and its instance equal the nested loop over the C++ surface's Bvh<Node>::intersect that the
trace_instances host test uses, and next receives the scripted world ray bit for bit, for both robust settings, both tie
rules and three filters.  One identity instance equals trace_paths on the bare mesh."""
import os
import subprocess

import numpy as np
import pytest

from tests.conftest import golden
from tests.test_device_api_host import extra_rays
from tests.test_device_instance_trace_host import INCLUDES, one_triangle, run_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILTERS = 3
MODES = 4
SCENES = ["identity", "translate", "scale", "permute", "pair", "many"]


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "device_instance_path_trace_host_test")
    src = os.path.join(ROOT, "tests", "device_instance_path_trace_host_test.cpp")
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
    """(scene, filter, mode) -> dict of the line's counters"""
    out = {}
    for line in log.splitlines():
        w = line.split()
        if w and w[0] == "scene":
            out[(w[1], int(w[3]), int(w[5]))] = {"segments": int(w[7]), "occlusion": int(w[9]), "nan": int(w[11]),
                                                 "hits": int(w[-4]), "calls": int(w[-1])}
    return out


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "soup1k_f64"])
def test_trace_instance_paths_matches_nested_loop(exe, tmp_path, name):
    g = golden(name)
    tris = g["tris"]
    others = [golden("box12_f32")] if tris.dtype == np.float32 else []
    meshes = [(g["ref_bounds"], g["ref_index"], g["ref_prim_ids"], tris)]
    meshes += [(o["ref_bounds"], o["ref_index"], o["ref_prim_ids"], o["tris"]) for o in others]
    meshes.append(one_triangle(tris.dtype))
    rays = np.concatenate([g["rays"], extra_rays(tris, tris.dtype)])
    log = run_case(exe, tmp_path, meshes, rays)
    assert "empty batch ok, record count throws, small workspace throws, deep stack throws" in log, log
    assert "failures 0" in log, log
    t = table(log)
    assert len(t) == len(SCENES) * FILTERS * MODES, log
    for scene in SCENES:
        for mode in range(MODES):
            c = t[(scene, 0, mode)]
            assert c["hits"] > 0 and c["calls"] >= c["hits"], (scene, mode, log)
            assert 0 < c["occlusion"] < c["segments"], (scene, log)
    assert t[("identity", 0, 0)]["nan"] > 0, log


def test_one_primitive_mesh(exe, tmp_path):
    """A bottom tree whose root is a leaf, as the only mesh, with NaN-interval rays."""
    bounds, index, ids, tri = one_triangle(np.float32)
    rays = np.concatenate([np.array([[0.2, 0.2, 1, 0, 0, -1, 0, np.inf], [0.2, 0.2, 1, 0, 0, -1, np.nan, np.inf],
                                     [5, 5, 1, 0, 0, -1, 0, np.inf]], np.float32), extra_rays(tri, np.float32)])
    log = run_case(exe, tmp_path, [(bounds, index, ids, tri)], rays)
    t = table(log)
    for mode in range(MODES):
        assert t[("identity", 0, mode)]["hits"] >= 1, log
        assert t[("identity", 0, mode)]["nan"] >= 1, log
