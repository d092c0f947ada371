"""DeviceView::traverse_bottom_up and the three-argument node test without a GPU.

The header (include/bvh/v2/cuda/intersect.cuh) compiled by g++ runs its host pass on the golden trees of the unmodified
reference (tests/device_bottom_up_host_test.cpp): the same (leaf or inner, index) call sequence as
Bvh<Node>::traverse_bottom_up of the C++ surface, subtree counts and box unions equal to the C++ surface's (the boxes bit
for bit those of Bvh::refit), one call per node with the children first, and a three-argument node test that receives
the left_index sequence `&left - nodes.data()` gives on the C++ surface.  The mass, centre-of-mass and Barnes-Hut
functions of the GPU tests (tests/device_bottom_up.h) are checked here against a float64 brute force."""
import os
import re
import subprocess

import numpy as np
import pytest

from tests.conftest import golden
from tests.test_device_query_host import INCLUDES, ROOT, queries, tri_boxes

HARNESS = os.path.join(ROOT, "tests", "_build", "device_bottom_up_host_test")


def build_harness():
    """tests/_build/device_bottom_up_host_test, rebuilt when a source is newer."""
    src = os.path.join(ROOT, "tests", "device_bottom_up_host_test.cpp")
    deps = [src] + [os.path.join(ROOT, *p) for p in (("tests", "device_bottom_up.h"), ("tests", "device_queries.h"),
                                                     ("include", "bvh", "v2", "cuda", "intersect.cuh"),
                                                     ("include", "bvh", "v2", "b200_surface.h"), ("include", "bvh_b200_device.h"),
                                                     ("bvh_b200", "csrc", "traverse_core.cuh"), ("bvh_b200", "csrc", "refit_core.cuh"),
                                                     ("bvh_b200", "csrc", "build_core.cuh"), ("bvh_b200", "csrc", "core.cuh"))]
    if not os.path.exists(HARNESS) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(HARNESS):
        os.makedirs(os.path.dirname(HARNESS), exist_ok=True)
        subprocess.check_call(["g++", "-std=gnu++20", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-Wall", "-Werror",
                               *INCLUDES, src, "-o", HARNESS])
    return HARNESS


@pytest.fixture(scope="module")
def exe():
    return build_harness()


def node_records(bounds, index):
    dtype = bounds.dtype
    rec = np.dtype([("bounds", dtype, 6), ("index", np.uint32 if dtype == np.float32 else np.uint64)])
    nodes = np.zeros(bounds.shape[0], rec)
    nodes["bounds"], nodes["index"] = bounds, index
    return nodes


def run_check(exe, tmp_path, bounds, index, prim_ids, boxes, qs):
    """The `check` mode: {name: (mismatches, numbers...)} per output line."""
    path = tmp_path / "check.bin"
    with open(path, "wb") as f:
        f.write(np.array([bounds.shape[0], prim_ids.shape[0], qs.shape[0]], np.uint64).tobytes())
        f.write(node_records(bounds, index).tobytes())
        f.write(np.asarray(prim_ids, np.uint64).tobytes())
        f.write(np.ascontiguousarray(boxes, bounds.dtype).tobytes())
        f.write(np.ascontiguousarray(qs, bounds.dtype).tobytes())
    res = subprocess.run([exe, "check", str(path), "d" if bounds.dtype == np.float64 else "f"], capture_output=True, text=True)
    out = {}
    for line in res.stdout.splitlines():
        words = line.split()
        if words and words[0] in ("sequence", "counts", "boxes", "audit", "workspace"):
            out[words[0]] = {words[k]: int(words[k + 1]) for k in range(1, len(words) - 1, 2)}
        m = re.match(r"node_index kind (\d) start (\d) mismatches (\d+) node_calls (\d+) leaf_calls (\d+)", line)
        if m:
            out["node_index", int(m[1]), int(m[2])] = dict(zip(("mismatches", "node_calls", "leaf_calls"), map(int, m.groups()[2:])))
    assert res.returncode == 0, res.stdout + res.stderr
    assert len(out) == 11, res.stdout
    assert all(v["mismatches"] == 0 for v in out.values()), res.stdout
    return out


def run_physics(exe, tmp_path, bounds, index, prim_ids, pos, mass, points, theta, eps2):
    """The `physics` mode: (node_mass, node_centre, phi, approximated) from the header's host pass and traversal."""
    dtype = bounds.dtype
    path, out = tmp_path / "physics.bin", tmp_path / "physics.out"
    n, m = bounds.shape[0], points.shape[0]
    with open(path, "wb") as f:
        f.write(np.array([n, prim_ids.shape[0], m], np.uint64).tobytes())
        f.write(node_records(bounds, index).tobytes())
        f.write(np.asarray(prim_ids, np.uint64).tobytes())
        for a in (pos, mass, points, np.array([theta * theta, eps2])):
            f.write(np.ascontiguousarray(a, dtype).tobytes())
    subprocess.check_call([exe, "physics", str(path), "d" if dtype == np.float64 else "f", str(out)])
    raw = open(out, "rb").read()
    size = np.dtype(dtype).itemsize
    node_mass = np.frombuffer(raw, dtype, n)
    node_centre = np.frombuffer(raw, dtype, 3 * n, n * size).reshape(n, 3)
    phi = np.frombuffer(raw, dtype, m, 4 * n * size)
    approximated = np.frombuffer(raw, np.uint32, m, (4 * n + m) * size)
    return node_mass, node_centre, phi, approximated


def brute_potential(pos, mass, points, eps2):
    """-sum m / sqrt(d^2 + eps2) in float64."""
    pos, mass, points = (np.asarray(a, np.float64) for a in (pos, mass, points))
    out = np.empty(points.shape[0])
    for k in range(0, points.shape[0], 16):
        d2 = ((points[k:k + 16, None, :] - pos[None, :, :]) ** 2).sum(axis=2)
        out[k:k + 16] = -(mass[None, :] / np.sqrt(d2 + eps2)).sum(axis=1)
    return out


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "box12_f32", "soup1k_f64"])
def test_matches_cxx_surface(exe, tmp_path, name):
    g = golden(name)
    boxes = tri_boxes(g["tris"])
    index = g["ref_index"].astype(np.uint64)
    got = run_check(exe, tmp_path, g["ref_bounds"], index, g["ref_prim_ids"], boxes, queries(boxes, boxes.dtype, m=100))
    n, leaves = index.shape[0], int(((index & 15) != 0).sum())
    assert got["sequence"] == dict(calls=n, leaves=leaves, inners=n - leaves, mismatches=0)
    assert got["node_index", 1, 0]["node_calls"] == 100 * (leaves - 1)    # accept-all from the root: every inner node
    assert got["node_index", 1, 0]["leaf_calls"] == 100 * leaves
    assert got["node_index", 0, 0]["leaf_calls"] > 0
    for kind in range(2):                                              # a leaf start: one leaf call, no node test
        assert (got["node_index", kind, 2]["node_calls"], got["node_index", kind, 2]["leaf_calls"]) == (0, 100)


def test_one_primitive_tree(exe, tmp_path):
    """The root is a leaf: one leaf call, no inner call, no node test."""
    bounds = np.array([[0, 1, 0, 1, 0, 1]], np.float32)
    boxes = np.array([[0, 0, 0, 1, 1, 1]], np.float32)
    qs = queries(np.concatenate([boxes, boxes + 0.5]), np.float32, m=20)
    got = run_check(exe, tmp_path, bounds, np.array([1], np.uint64), np.array([0], np.uint64), boxes, qs)
    assert got["sequence"] == dict(calls=1, leaves=1, inners=0, mismatches=0)
    for kind in range(2):
        for start in range(3):
            assert (got["node_index", kind, start]["node_calls"], got["node_index", kind, start]["leaf_calls"]) == (0, 20)


@pytest.mark.parametrize("name", ["soup2k_f32", "soup1k_f64"])
def test_mass_and_barnes_hut(exe, tmp_path, name):
    """The GPU tests' functions on a golden tree, particles at the triangles' centroids: the root holds the total mass at
    the centre of mass, theta = 0 is the brute-force potential, theta = 0.5 approximates it and visits less."""
    g = golden(name)
    dtype = g["tris"].dtype
    pos = g["tris"].reshape(-1, 3, 3).mean(axis=1).astype(dtype)
    rng = np.random.default_rng(2)
    mass = (0.5 + rng.random(pos.shape[0])).astype(dtype)
    lo, hi = pos.min(axis=0), pos.max(axis=0)
    points = (lo + (hi - lo) * (rng.random((300, 3)) * 1.4 - 0.2)).astype(dtype)
    eps2 = float(((hi - lo).max() * 1e-3) ** 2)
    args = (g["ref_bounds"], g["ref_index"].astype(np.uint64), g["ref_prim_ids"], pos, mass, points)
    node_mass, node_centre, exact, none = run_physics(exe, tmp_path, *args, 0.0, eps2)
    assert np.isclose(node_mass[0], mass.astype(np.float64).sum(), rtol=1e-5)
    want_centre = (mass[:, None].astype(np.float64) * pos).sum(axis=0) / mass.astype(np.float64).sum()
    assert np.allclose(node_centre[0], want_centre, rtol=1e-5, atol=1e-5 * np.abs(hi - lo).max())
    brute = brute_potential(pos, mass, points, eps2)
    rtol = 1e-5 if dtype == np.float32 else 1e-12
    assert (none == 0).all() and np.allclose(exact, brute, rtol=rtol, atol=0)
    _, _, approx, used = run_physics(exe, tmp_path, *args, 0.5, eps2)
    assert used.min() > 0 and np.max(np.abs(approx - brute) / np.abs(brute)) < 2e-2
