"""DeviceView::trace (include/bvh/v2/cuda/intersect.cuh) compiled by g++ as host code, no GPU needed.

On the golden trees of the unmodified reference and on a one-primitive tree, a recording tracer makes per ray the leaf
calls Bvh<Node>::intersect of the C++ surface makes, in the same order, and ends with the same hit and the same tmax, for
closest-hit, any-hit and robust rays, NaN-interval rays and a leaf that makes the interval NaN part-way through
(tests/device_trace_host_test.cpp).  The scheduling rules trace shares with bvhNN_intersect_rays (trace_plan.h) give the
values the batched call computed before they were shared."""
import os
import subprocess

import numpy as np
import pytest

from tests.conftest import golden
from tests.test_device_api_host import extra_rays

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDES = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "bvh_b200", "csrc")]


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "device_trace_host_test")
    src = os.path.join(ROOT, "tests", "device_trace_host_test.cpp")
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


def leaf_calls(log):
    """(mode, leaf) -> leaf calls of the whole batch"""
    out = {}
    for line in log.splitlines():
        w = line.split()
        if w and w[0] == "mode":
            out[(int(w[1]), int(w[3]))] = int(w[-1])
    return out


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "box12_f32", "soup1k_f64"])
def test_trace_matches_intersect(exe, tmp_path, name):
    g = golden(name)
    tris = g["tris"]
    rays = np.concatenate([g["rays"], extra_rays(tris, tris.dtype)])
    log = run_case(exe, tmp_path, g["ref_bounds"], g["ref_index"], g["ref_prim_ids"], tris, rays)
    assert "empty batch ok, small workspace throws, null workspace throws" in log, log
    calls = leaf_calls(log)
    assert len(calls) == 12, log
    assert " hits 0 " not in log.splitlines()[0], log          # the closest-hit triangle pass does hit something
    # the NaN-making leaf skips the box tests after its second call: no more leaf calls than the record-only leaf, and
    # fewer on the larger trees
    assert 0 < calls[(0, 2)] <= calls[(0, 1)], log
    if name != "box12_f32":
        assert calls[(0, 2)] < calls[(0, 1)], log


def test_one_primitive_tree(exe, tmp_path):
    """The root is a leaf: every ray, a NaN-interval one included, makes exactly one leaf call."""
    tri = np.array([[0, 0, 0, 1, 0, 0, 0, 1, 0]], np.float32)
    bounds = np.array([[0, 1, 0, 1, 0, 0]], np.float32)
    index = np.array([1], np.uint64)
    rays = np.concatenate([np.array([[0.2, 0.2, 1, 0, 0, -1, 0, np.inf], [0.2, 0.2, 1, 0, 0, -1, np.nan, np.inf],
                                     [5, 5, 1, 0, 0, -1, 0, np.inf]], np.float32), extra_rays(tri, np.float32)])
    log = run_case(exe, tmp_path, bounds, index, np.array([0], np.uint64), tri, rays)
    calls = leaf_calls(log)
    for mode in range(4):
        assert calls[(mode, 1)] == rays.shape[0], log


def old_run_rays(chunk, n, sms):
    """The run length trace_rays computed before the rule moved to trace_plan.h."""
    run = chunk
    fair = n // (sms * 32 * 8)
    if fair < run:
        run = fair
    run &= ~31 & 0xFFFFFFFF
    return 32 if run < 32 else run


def old_grid(sms, per_sm, n, rays_per_warp=32, block=128):
    """The grid launch_persistent computed before the rule moved to trace_plan.h."""
    per_sm = max(per_sm, 1)
    grid = sms * per_sm
    max_useful = (n + rays_per_warp - 1) // rays_per_warp // (block // 32) + 1
    return min(grid, max_useful)


def test_plan_rules_unchanged(exe):
    out = subprocess.run([exe, "plan"], capture_output=True, text=True, check=True).stdout.split("\n")
    rows = [list(map(int, line.split())) for line in out if line]
    assert len(rows) == 13 * 5 * 4 * 4
    for n, sms, chunk, per_sm, run, grid in rows:
        assert run == old_run_rays(chunk, n, sms), (n, sms, chunk)
        assert grid == old_grid(sms, per_sm, n), (n, sms, per_sm)
