"""DeviceView::traverse_bottom_up on the GPU (tests/device_bottom_up_kernels.cu): one call per node of the right kind with
both children first, subtree counts that add up, box unions bit for bit the tree's boxes after refit_boxes with the same
boxes, mass and centre of mass bit for bit those of the header's host pass (tests/device_bottom_up_host_test.cpp) on the
downloaded tree, the same result from a reused workspace, build -> pass -> refit -> pass on one torch stream, and a
Barnes-Hut potential through the three-argument node test that matches the host run bit for bit and, opening every node,
a float64 brute force."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes
from tests.conftest import golden
from tests.test_device_bottom_up_host import brute_potential, build_harness, run_physics
from tests.test_device_query_gpu import bits, cuda, sphere_boxes

pytestmark = pytest.mark.gpu

P, SZ = C.c_void_p, C.c_size_t


@pytest.fixture(scope="module")
def bu(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_bottom_up_tests())
    for s, t in (("3f", C.c_float), ("3d", C.c_double)):
        getattr(L, f"bu_workspace_bytes{s}").argtypes = [P, C.POINTER(C.c_size_t)]
        getattr(L, f"bu_count_box{s}").argtypes = [P, P, SZ, P, P, P]
        getattr(L, f"bu_audit{s}").argtypes = [P, P, SZ, P, P, P, P]
        getattr(L, f"bu_mass{s}").argtypes = [P, P, SZ, P, P, P, P]
        getattr(L, f"bu_potential{s}").argtypes = [P, P, P, P, P, P, SZ, t, t, P, P]
    L.bu_last_error.restype = C.c_char_p
    return L


@pytest.fixture(scope="module")
def harness():
    return build_harness()


class Pass:
    """The test entry points on one handle, with one workspace; outputs are torch tensors on the handle's stream.  With
    `sync`, torch's work is finished before each launch and the handle's after it."""

    def __init__(self, bu, bvh, sync=True):
        import torch
        self.bu, self.bvh, self.s, self.sync = bu, bvh, bvh.s, sync
        self.dt = torch.float32 if self.s == "3f" else torch.float64
        nbytes = C.c_size_t(0)
        self.call("workspace_bytes", C.byref(nbytes))
        self.bytes = nbytes.value
        assert self.bytes == 8 * (bvh.node_count + 1)
        self.ws = torch.empty(self.bytes, dtype=torch.uint8, device="cuda")
        self.ws.fill_(0xA5)                                   # not initialised: the pass sets up its own links and flags
        self.n = bvh.node_count

    def call(self, name, *args):
        import torch
        if self.sync:
            torch.cuda.synchronize()
        rc = getattr(self.bu, f"bu_{name}{self.s}")(C.c_void_p(self.bvh.handle), *args)
        assert rc == 0, self.bu.bu_last_error()
        if self.sync:
            self.bvh.sync()

    def count_box(self, d_boxes):
        import torch
        counts = torch.zeros(self.n, dtype=torch.int32, device="cuda")
        boxes = torch.full((self.n, 6), float("nan"), dtype=self.dt, device="cuda")
        self.call("count_box", self.ws.data_ptr(), self.bytes, d_boxes.data_ptr(), counts.data_ptr(), boxes.data_ptr())
        return counts, boxes

    def audit(self):
        import torch
        out = [torch.zeros(k, dtype=torch.int32, device="cuda") for k in (self.n, self.n, self.n, 1)]
        self.call("audit", self.ws.data_ptr(), self.bytes, *[o.data_ptr() for o in out])
        return out

    def mass(self, d_pos, d_mass):
        import torch
        node_mass = torch.zeros(self.n, dtype=self.dt, device="cuda")
        node_centre = torch.zeros((self.n, 3), dtype=self.dt, device="cuda")
        self.call("mass", self.ws.data_ptr(), self.bytes, d_pos.data_ptr(), d_mass.data_ptr(), node_mass.data_ptr(),
                  node_centre.data_ptr())
        return node_mass, node_centre

    def potential(self, d_pos, d_mass, node_mass, node_centre, d_points, theta, eps2):
        import torch
        m = d_points.shape[0]
        phi = torch.zeros(m, dtype=self.dt, device="cuda")
        used = torch.zeros(m, dtype=torch.int32, device="cuda")
        self.call("potential", d_pos.data_ptr(), d_mass.data_ptr(), node_mass.data_ptr(), node_centre.data_ptr(), d_points.data_ptr(),
                  m, theta * theta, eps2, phi.data_ptr(), used.data_ptr())
        return phi, used


def host(t):
    import torch
    torch.cuda.synchronize()
    a = t.cpu().numpy()
    return a.view(np.uint32) if a.dtype == np.int32 else a


def subtree_counts_ok(index, counts):
    """Every leaf counts its primitives, every inner node the sum of its children's."""
    first, own = (index >> np.uint64(4)).astype(np.int64), (index & np.uint64(15)).astype(np.int64)
    leaf = own != 0
    inner = np.nonzero(~leaf)[0]
    return (counts[leaf] == own[leaf]).all() and (counts[inner] == counts[first[inner]] + counts[first[inner] + 1]).all()


def check_tree(bu, harness, tmp_path, bvh, boxes, pos, mass):
    """The per-node checks on one tree; boxes, pos and mass in the original primitive order."""
    dtype = boxes.dtype
    run = Pass(bu, bvh)
    _, index, ids = bvh.arrays()
    leaf = (index & np.uint64(15)) != 0
    leaf_calls, inner_calls, marks, errors = (host(t) for t in run.audit())
    assert (leaf_calls == leaf).all() and (inner_calls == ~leaf).all(), "one call per node, of the node's kind"
    assert errors[0] == 0 and (marks == 1).all(), "an inner call came before a child's"

    d_boxes = cuda(boxes)
    counts, node_boxes = (host(t) for t in run.count_box(d_boxes))
    assert subtree_counts_ok(index, counts) and counts[0] == bvh.prim_count
    again = [host(t) for t in run.count_box(d_boxes)]                # the same workspace, again
    assert (again[0] == counts).all() and (bits(again[1]) == bits(node_boxes)).all()
    bvh.refit_boxes(boxes)
    assert (bits(node_boxes) == bits(bvh.arrays()[0])).all(), "box unions differ from refit_boxes"

    d_pos, d_mass = cuda(pos), cuda(mass)
    node_mass, node_centre = (host(t) for t in run.mass(d_pos, d_mass))
    bounds, _, _ = bvh.arrays()
    want_mass, want_centre, _, _ = run_physics(harness, tmp_path, bounds, index, ids, pos, mass, np.zeros((0, 3), dtype), 0.0, 0.0)
    assert (bits(node_mass) == bits(want_mass)).all() and (bits(node_centre) == bits(want_centre)).all()
    second = [host(t) for t in run.mass(d_pos, d_mass)]
    assert (bits(second[0]) == bits(node_mass)).all() and (bits(second[1]) == bits(node_centre)).all()
    return node_mass, node_centre


def particles(centers, dtype, seed=7):
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(centers, dtype), (0.5 + rng.random(centers.shape[0])).astype(dtype)


@pytest.mark.parametrize("n", [1, 2, 3, 1000, 100_000, 1_000_000])
@pytest.mark.parametrize("leaf", [(1, 1), (1, 8)], ids=["leaf1-1", "leaf1-8"])
@pytest.mark.parametrize("quality", ["low", "medium", "high"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
def test_spheres(bu, harness, gpu_lib, tmp_path, dtype, quality, leaf, n):
    api = gpu_lib
    import torch
    boxes, centers = sphere_boxes(n, dtype, seed=n + 11)
    d_boxes, d_centers = cuda(boxes), cuda(centers)
    torch.cuda.synchronize()
    bvh = api.Bvh.build_boxes(d_boxes.data_ptr(), d_centers.data_ptr(), count=n, dtype=dtype, flags=api.DEVICE_POINTERS,
                              quality=quality, min_leaf_size=leaf[0], max_leaf_size=leaf[1])
    pos, mass = particles(centers, dtype)
    node_mass, node_centre = check_tree(bu, harness, tmp_path, bvh, boxes, pos, mass)
    assert np.isclose(node_mass[0], mass.astype(np.float64).sum(), rtol=1e-4)
    bvh.destroy()


def test_triangle_soup(bu, harness, gpu_lib, tmp_path):
    tris = scenes.soup(200_000)
    v = tris.reshape(-1, 3, 3)
    boxes = np.ascontiguousarray(np.concatenate([v.min(axis=1), v.max(axis=1)], axis=1))
    bvh = gpu_lib.Bvh.build_triangles(tris)
    check_tree(bu, harness, tmp_path, bvh, boxes, *particles(v.mean(axis=1), np.float32))
    bvh.destroy()


@pytest.mark.parametrize("name", ["soup2k_f32", "soup1k_f64"])
def test_reference_tree(bu, harness, gpu_lib, tmp_path, name):
    """The reference's own tree, uploaded through bvhNN_load."""
    g = golden(name)
    dtype = g["tris"].dtype
    path = tmp_path / "ref.bvh"
    path.write_bytes(g["ref_serialized"].tobytes())
    bvh = gpu_lib.Bvh.load(str(path), dtype=dtype)
    v = g["tris"].reshape(-1, 3, 3)
    boxes = np.ascontiguousarray(np.concatenate([v.min(axis=1), v.max(axis=1)], axis=1), dtype)
    check_tree(bu, harness, tmp_path, bvh, boxes, *particles(v.mean(axis=1), dtype))
    bvh.destroy()


def test_build_pass_refit_pass_on_one_stream(bu, harness, gpu_lib, tmp_path):
    """torch writes the boxes, build_boxes, the passes, torch moves the spheres, refit_boxes, the passes again: one torch
    stream, no synchronisation but the build's own.  The second results are those of the moved spheres."""
    api = gpu_lib
    import torch
    n = 100_000
    rng = np.random.default_rng(5)
    c0 = rng.random((n, 3)).astype(np.float32)
    r = (0.002 + 0.004 * rng.random(n)).astype(np.float32)
    step = (0.05 * (rng.random((n, 3)) - 0.5)).astype(np.float32)
    mass = (0.5 + rng.random(n)).astype(np.float32)
    stream = torch.cuda.Stream()
    api.set_stream(stream.cuda_stream)
    results = []
    try:
        with torch.cuda.stream(stream):
            c, d_r, d_mass, d_step = cuda(c0), cuda(r)[:, None], cuda(mass), cuda(step)
            boxes = torch.cat([c - d_r, c + d_r], dim=1)
            bvh = api.Bvh.build_boxes(boxes.data_ptr(), c.data_ptr(), count=n, dtype=np.float32, flags=api.DEVICE_POINTERS)
            run = Pass(bu, bvh, sync=False)
            for frame in range(2):
                if frame:
                    c.add_(d_step)
                    torch.cat([c - d_r, c + d_r], dim=1, out=boxes)
                    bvh.refit_boxes(boxes.data_ptr(), api.DEVICE_POINTERS)
                results.append((c.clone(), boxes.clone()) + run.count_box(boxes) + run.mass(c, d_mass))
    finally:
        api.set_stream(None)
    stream.synchronize()
    bounds, index, ids = bvh.arrays()
    for frame, (pos, b, counts, node_boxes, node_mass, node_centre) in enumerate(results):
        pos, b = host(pos), host(b)
        assert subtree_counts_ok(index, host(counts))
        want_mass, want_centre, _, _ = run_physics(harness, tmp_path, bounds, index, ids, pos, mass, np.zeros((0, 3), np.float32), 0.0, 0.0)
        assert (bits(host(node_mass)) == bits(want_mass)).all() and (bits(host(node_centre)) == bits(want_centre)).all(), frame
        if frame:
            assert (bits(host(node_boxes)) == bits(bounds)).all(), "the second pass sees the refitted tree's boxes"
        else:
            assert not (host(node_boxes) == bounds).all(), "the first pass ran before the move"
    assert not np.allclose(host(results[0][5]), host(results[1][5]))
    bvh.destroy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
def test_barnes_hut(bu, harness, gpu_lib, tmp_path, dtype):
    """theta = 0.5: bit for bit the host run of the same header, within 2% of the brute force.  theta = 0 opens every
    node: the float64 brute force within rtol 2e-4 (float32: 100K positive terms summed one by one in tree order) or
    1e-11 (float64)."""
    boxes, centers = sphere_boxes(100_000, dtype, seed=8)
    bvh = gpu_lib.Bvh.build(boxes, centers)
    pos, mass = particles(centers, dtype)
    rng = np.random.default_rng(9)
    points = (rng.random((2000, 3)) * 1.2 - 0.1).astype(dtype)
    eps2 = 1e-6
    run = Pass(bu, bvh)
    d_pos, d_mass, d_points = cuda(pos), cuda(mass), cuda(points)
    node_mass, node_centre = run.mass(d_pos, d_mass)
    bounds, index, ids = bvh.arrays()
    want_mass, want_centre, want_phi, want_used = run_physics(harness, tmp_path, bounds, index, ids, pos, mass, points, 0.5, eps2)
    assert (bits(host(node_mass)) == bits(want_mass)).all() and (bits(host(node_centre)) == bits(want_centre)).all()
    phi, used = (host(t) for t in run.potential(d_pos, d_mass, node_mass, node_centre, d_points, 0.5, eps2))
    assert (bits(phi) == bits(want_phi)).all() and (used == want_used).all()
    assert used.min() > 0
    exact, none = (host(t) for t in run.potential(d_pos, d_mass, node_mass, node_centre, d_points, 0.0, eps2))
    assert (none == 0).all()
    brute = brute_potential(pos, mass, points, eps2)
    assert np.allclose(exact, brute, rtol=2e-4 if dtype == np.float32 else 1e-11, atol=0)
    assert np.max(np.abs(phi - brute) / np.abs(brute)) < 2e-2
    bvh.destroy()


def test_errors(bu, gpu_lib):
    """A workspace one byte too small, or none, is refused before anything is launched."""
    boxes, centers = sphere_boxes(1000, np.float32)
    bvh = gpu_lib.Bvh.build(boxes, centers)
    run = Pass(bu, bvh)
    import torch
    counts = torch.zeros(bvh.node_count, dtype=torch.int32, device="cuda")
    out = torch.zeros((bvh.node_count, 6), dtype=torch.float32, device="cuda")
    d_boxes = cuda(boxes)
    for ws, nbytes in ((run.ws.data_ptr(), run.bytes - 1), (None, run.bytes)):
        assert bu.bu_count_box3f(C.c_void_p(bvh.handle), ws, nbytes, d_boxes.data_ptr(), counts.data_ptr(), out.data_ptr()) == -1
        assert b"too small" in bu.bu_last_error()
    assert (host(counts) == 0).all()
    assert bu.bu_count_box3f(None, run.ws.data_ptr(), run.bytes, d_boxes.data_ptr(), counts.data_ptr(), out.data_ptr()) == -1
    bvh.destroy()
