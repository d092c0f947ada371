"""DeviceView::trace_instances and prepare_instances (include/bvh/v2/cuda/intersect.cuh) compiled by g++ as host code, no
GPU needed.

The golden trees of the unmodified reference (and a one-primitive tree) are the bottom meshes.  Placed by identity,
translation, power-of-two scale, axis permutation, general rotation and singular matrices, prepared with
prepare_instances and topped by a tree over the prepared boxes, a recording shader gets per ray the accept calls (instance,
original id, bits of t, u, v) and the record a nested loop over the C++ surface's Bvh<Node>::intersect makes, for
closest-hit, any-hit and robust rays under both tie rules and three filters, NaN-interval and axis-parallel rays included
(tests/device_instance_trace_host_test.cpp).  One identity instance equals trace_triangles; two copies at the same place
tie and the canonical rule takes the lower instance."""
import os
import subprocess

import numpy as np
import pytest

from tests.conftest import golden
from tests.test_device_api_host import extra_rays

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDES = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "bvh_b200", "csrc")]
FILTERS = 3
MODES = 8
SCENES = ["identity", "translate", "scale", "permute", "pair", "many"]


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "device_instance_trace_host_test")
    src = os.path.join(ROOT, "tests", "device_instance_trace_host_test.cpp")
    csrc = os.path.join(ROOT, "bvh_b200", "csrc")
    deps = [src, os.path.join(ROOT, "include", "bvh", "v2", "cuda", "intersect.cuh"),
            os.path.join(ROOT, "include", "bvh", "v2", "b200_surface.h"), os.path.join(ROOT, "include", "bvh_b200_device.h")]
    deps += [os.path.join(csrc, f) for f in ("traverse_core.cuh", "core.cuh", "persistent_core.cuh", "trace_plan.h")]
    if not os.path.exists(out) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(out):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["g++", "-std=gnu++20", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-Wall", *INCLUDES,
                               src, "-o", out])
    return out


def run_case(exe, tmp_path, meshes, rays):
    """meshes: (bounds, index, prim_ids, tris) of each bottom mesh, mesh 0 first"""
    dtype = rays.dtype
    rec = np.dtype([("bounds", dtype, 6), ("index", np.uint32 if dtype == np.float32 else np.uint64)])
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(np.array([len(meshes)], np.uint64).tobytes())
        for bounds, index, prim_ids, tris in meshes:
            nodes = np.zeros(bounds.shape[0], rec)
            nodes["bounds"], nodes["index"] = bounds, index
            f.write(np.array([nodes.shape[0], prim_ids.shape[0]], np.uint64).tobytes())
            f.write(nodes.tobytes())
            f.write(prim_ids.astype(np.uint64).tobytes())
            f.write(np.ascontiguousarray(tris, dtype).tobytes())
        f.write(np.array([rays.shape[0]], np.uint64).tobytes())
        f.write(np.ascontiguousarray(rays).tobytes())
    res = subprocess.run([exe, str(path), "d" if dtype == np.float64 else "f"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return res.stdout


def table(log):
    """(scene, filter, mode) -> dict of the line's counters"""
    out = {}
    for line in log.splitlines():
        w = line.split()
        if w and w[0] == "scene":
            out[(w[1], int(w[3]), int(w[5]))] = {"singular": int(w[12]), "ties": int(w[14]), "lower": int(w[16]),
                                                 "hits": int(w[18]), "calls": int(w[-1])}
    return out


def one_triangle(dtype):
    tri = np.array([[0, 0, 0, 1, 0, 0, 0, 1, 0]], dtype)
    return np.array([[0, 1, 0, 1, 0, 0]], dtype), np.array([1], np.uint64), np.array([0], np.uint64), tri


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "soup1k_f64"])
def test_trace_instances_matches_nested_loop(exe, tmp_path, name):
    g = golden(name)
    tris = g["tris"]
    others = [golden("box12_f32")] if tris.dtype == np.float32 else []
    meshes = [(g["ref_bounds"], g["ref_index"], g["ref_prim_ids"], tris)]
    meshes += [(o["ref_bounds"], o["ref_index"], o["ref_prim_ids"], o["tris"]) for o in others]
    meshes.append(one_triangle(tris.dtype))
    rays = np.concatenate([g["rays"], extra_rays(tris, tris.dtype)])
    log = run_case(exe, tmp_path, meshes, rays)
    assert "empty batch ok, record count throws, small workspace throws, deep stack throws" in log, log
    t = table(log)
    assert len(t) == len(SCENES) * FILTERS * MODES, log
    for scene in SCENES:
        for mode in range(MODES):
            c = t[(scene, 0, mode)]
            assert c["hits"] > 0 and c["calls"] >= c["hits"], (scene, mode, log)
            assert c["singular"] == (2 if scene == "many" else 0), (scene, log)
    for mode in (0, 2):                        # closest-hit, canonical rule: every tie goes to instance 0
        c = t[("pair", 0, mode)]
        assert c["ties"] > 0 and c["lower"] == c["ties"], (mode, log)
        assert t[("pair", 2, mode)]["hits"] > 0                 # odd instances rejected: instance 0 still hits
    for mode in (4, 6):                        # last visited: the second copy takes the ties
        c = t[("pair", 0, mode)]
        assert c["ties"] > 0 and c["lower"] == 0, (mode, log)


def test_one_primitive_meshes(exe, tmp_path):
    """Bottom trees whose root is a leaf, as the only mesh: NaN-interval rays get no accept call."""
    bounds, index, ids, tri = one_triangle(np.float32)
    rays = np.concatenate([np.array([[0.2, 0.2, 1, 0, 0, -1, 0, np.inf], [0.2, 0.2, 1, 0, 0, -1, np.nan, np.inf],
                                     [5, 5, 1, 0, 0, -1, 0, np.inf]], np.float32), extra_rays(tri, np.float32)])
    log = run_case(exe, tmp_path, [(bounds, index, ids, tri)], rays)
    t = table(log)
    for mode in range(MODES):
        assert t[("identity", 0, mode)]["hits"] >= 1, log
