"""The deforming forms of DeviceView::trace_instances and trace_instance_paths, make_deforming_instance and
prepare_deforming_instances (include/bvh/v2/cuda/intersect.cuh) compiled by g++ as host code, no GPU needed.

Each golden tree of the unmodified reference (and box12 and a one-triangle tree) is the bottom mesh in all three
kinds: static, deforming on shutter boxes and deforming with motion nodes, under the key pairs equal, jitter, ulps (at
1e4, keys a few ulps apart), non_finite and partial, at the times 0, 1, 0.5, 0.3, random, -1, 2 and NaN
(tests/device_deforming_instance_host_test.cpp).  For every flag, tie rule and three filters: static bottoms only equal
the motion trace_instances, one identity record equals the motion and motion-node trace_triangles, equal vertex keys
equal the static bottom, and path segments equal trace_instances; two copies tie to the lower instance; every world box
holds the blended, placed vertices at 65 uniform, adversarial and 1024 random times; in object space every blended
vertex lies in its leaf's motion-node keys and in the root's key boxes (the bottom box the world box rests on), while
the ulps pair's vertices leave the same leaf boxes recomputed without the widening; and the errors are thrown as
documented."""
import os
import subprocess

import numpy as np
import pytest

from tests.conftest import golden
from tests.test_device_api_host import extra_rays
from tests.test_device_instance_trace_host import INCLUDES, one_triangle, run_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = ["equal", "jitter", "ulps", "non_finite", "partial"]


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "device_deforming_instance_host_test")
    src = os.path.join(ROOT, "tests", "device_deforming_instance_host_test.cpp")
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


def check_log(log, hits=True):
    assert "failures 0" in log, log
    assert "empty batch ok, errors thrown 11 of 11" in log, log
    for pair in PAIRS:
        assert f"pair {pair} box misses 0 " in log, log
        assert f"pair {pair} leaf misses 0 root misses 0 " in log, log
    if hits:
        for line in log.splitlines():
            w = line.split()
            if w and w[0] == "rays" and w[3] == "0" and w[5] in ("0", "2"):
                assert int(w[-1]) > 0, line
        assert int(log.split("pair copies hits ")[1].split()[0]) > 0, log


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "soup1k_f64", "box12_f32"])
def test_deforming_instances_host(exe, tmp_path, name):
    g = golden(name)
    tris = g["tris"]
    rays = np.concatenate([g["rays"][:768], extra_rays(tris, tris.dtype)])
    log = run_case(exe, tmp_path, [(g["ref_bounds"], g["ref_index"], g["ref_prim_ids"], tris)], rays)
    check_log(log)
    if name != "soup1k_f64":
        # the rounding the widening is there for: blended vertices outside their leaves' key boxes recomputed without
        # the widening, inside the widened ones (so the leaf check fails when the widening is removed)
        assert int(log.split("pair ulps leaf misses 0 root misses 0 unwidened misses ")[1].split()[0]) > 0, log


def test_one_triangle_tree(exe, tmp_path):
    bounds, index, ids, tri = one_triangle(np.float32)
    rays = np.concatenate([np.array([[0.2, 0.2, 1, 0, 0, -1, 0, np.inf], [0.2, 0.2, 1, 0, 0, -1, np.nan, np.inf],
                                     [5, 5, 1, 0, 0, -1, 0, np.inf]], np.float32), extra_rays(tri, np.float32)])
    log = run_case(exe, tmp_path, [(bounds, index, ids, tri)], rays)
    check_log(log, hits=False)
