"""The device traversal API (include/bvh/v2/cuda/intersect.cuh) compiled by g++ as host code, no GPU needed.

On the golden trees of the unmodified reference, DeviceView::intersect with the header's triangle leaf reproduces the
reference's ids and t bit for bit, and with recording leaves it makes the same leaf calls, in the same order, with the
same inner steps as Bvh<Node>::intersect of the C++ surface (tests/device_api_host_test.cpp)."""
import os
import subprocess

import numpy as np
import pytest

from tests.conftest import golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDES = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "bvh_b200", "csrc")]


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "device_api_host_test")
    src = os.path.join(ROOT, "tests", "device_api_host_test.cpp")
    deps = [src, os.path.join(ROOT, "include", "bvh", "v2", "cuda", "intersect.cuh"),
            os.path.join(ROOT, "include", "bvh", "v2", "b200_surface.h"), os.path.join(ROOT, "include", "bvh_b200.h"), os.path.join(ROOT, "include", "bvh_b200_device.h"),
            os.path.join(ROOT, "bvh_b200", "csrc", "traverse_core.cuh"), os.path.join(ROOT, "bvh_b200", "csrc", "core.cuh")]
    if not os.path.exists(out) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(out):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["g++", "-std=gnu++20", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-Wall", *INCLUDES,
                               src, "-o", out])
    return out


def test_header_compiles_as_host_cxx(tmp_path):
    src = tmp_path / "only_header.cpp"
    src.write_text("#include <bvh/v2/cuda/intersect.cuh>\n"
                   "template struct bvh::v2::cuda::DeviceView<float>;\n"
                   "template struct bvh::v2::cuda::DeviceView<double>;\n"
                   "int main() { return 0; }\n")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", *INCLUDES, str(src)])


def extra_rays(tris, dtype, seed=7):
    """Rays the golden sets lack: NaN intervals, zero and axis-parallel directions."""
    rng = np.random.default_rng(seed)
    lo, hi = tris.reshape(-1, 3).min(axis=0), tris.reshape(-1, 3).max(axis=0)
    centre = (lo + hi) / 2
    out = []
    for k in range(48):
        org = centre + (hi - lo) * (rng.random(3) - 0.5) * 2
        target = tris[rng.integers(tris.shape[0])].reshape(3, 3).mean(axis=0)
        d = target - org
        tmin, tmax = 0.0, np.inf
        kind = k % 6
        if kind == 0:
            tmin = np.nan
        elif kind == 1:
            tmax = np.nan
        elif kind == 2:
            d = np.zeros(3)
        elif kind == 3:
            axis = k % 3
            d = np.zeros(3)
            d[axis] = -1.0 if org[axis] > target[axis] else 1.0
            org = target.copy()
            org[axis] = lo[axis] - 1 if d[axis] > 0 else hi[axis] + 1
        elif kind == 4:
            d = np.array([d[0], 0.0, d[2]])
        else:
            tmax = 1e30
        out.append(np.concatenate([org, d, [tmin, tmax]]))
    return np.array(out, dtype)


def run_case(exe, tmp_path, nodes_bounds, nodes_index, prim_ids, tris, rays):
    dtype = tris.dtype
    rec = np.dtype([("bounds", dtype, 6), ("index", np.uint32 if dtype == np.float32 else np.uint64)])
    nodes = np.zeros(nodes_bounds.shape[0], rec)
    nodes["bounds"], nodes["index"] = nodes_bounds, nodes_index
    path, out_path = tmp_path / "case.bin", tmp_path / "out.bin"
    with open(path, "wb") as f:
        f.write(np.array([nodes.shape[0], prim_ids.shape[0], rays.shape[0]], np.uint64).tobytes())
        f.write(nodes.tobytes())
        f.write(prim_ids.astype(np.uint64).tobytes())
        f.write(np.ascontiguousarray(tris).tobytes())
        f.write(np.ascontiguousarray(rays).tobytes())
    res = subprocess.run([exe, str(path), "d" if dtype == np.float64 else "f", str(out_path)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    m = rays.shape[0]
    raw = out_path.read_bytes()
    ids = np.frombuffer(raw[:12 * m], np.uint32).reshape(3, m)
    t = np.frombuffer(raw[12 * m:], dtype).reshape(3, m)
    return ids, t, res.stdout


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "box12_f32", "soup1k_f64"])
def test_view_traversal_matches_reference(exe, tmp_path, name):
    g = golden(name)
    tris = g["tris"]
    rays = np.concatenate([g["rays"], extra_rays(tris, tris.dtype)])
    ids, t, log = run_case(exe, tmp_path, g["ref_bounds"], g["ref_index"], g["ref_prim_ids"], tris, rays)
    n = g["rays"].shape[0]
    bits = np.uint32 if tris.dtype == np.float32 else np.uint64
    for mode, key in enumerate(("last", "any", "robust")):
        assert (ids[mode, :n] == g[f"{key}_ids"]).all(), f"{name} {key}: ids"
        assert (t[mode, :n].view(bits) == g[f"{key}_t"].view(bits)).all(), f"{name} {key}: t"
    assert "hits 0 " not in log.splitlines()[0], log        # the closest-hit triangle pass does hit something


def test_one_primitive_tree(exe, tmp_path):
    """The root is a leaf: every ray, a NaN-interval one included, makes exactly the reference's single leaf call."""
    tri = np.array([[0, 0, 0, 1, 0, 0, 0, 1, 0]], np.float32)
    bounds = np.array([[0, 1, 0, 1, 0, 0]], np.float32)
    index = np.array([1], np.uint64)                          # first id 0, one primitive
    rays = np.concatenate([np.array([[0.2, 0.2, 1, 0, 0, -1, 0, np.inf], [0.2, 0.2, 1, 0, 0, -1, np.nan, np.inf],
                                     [5, 5, 1, 0, 0, -1, 0, np.inf]], np.float32), extra_rays(tri, np.float32)])
    ids, t, log = run_case(exe, tmp_path, bounds, index, np.array([0], np.uint64), tri, rays)
    assert ids[0, 0] == 0 and t[0, 0] == 1.0
    assert ids[0, 1] == 0xFFFFFFFF and ids[0, 2] == 0xFFFFFFFF
    # a record-only leaf is called once per ray whatever the ray: the root is a leaf and no box is tested before it
    for line in log.splitlines():
        if line.startswith("mode") and " leaf 1 " in line:
            assert line.endswith(f"leaf calls {rays.shape[0]}"), line
