"""The device traversal API on the GPU: DeviceView::intersect in test kernels (tests/device_api_kernels.cu) against the
library's batched kernels, the C++ surface's Bvh::intersect on the host mirror and a NumPy brute force."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes

pytestmark = pytest.mark.gpu

P, SZ, U = C.c_void_p, C.c_size_t, C.c_uint
LEAF_NONE, LEAF_TRI, LEAF_SPHERE = 0, 1, 2
NO_START = C.c_size_t(-1).value


@pytest.fixture(scope="module")
def dapi(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_api_tests())
    for s in ("3f", "3d"):
        getattr(L, f"dapi_trace{s}").argtypes = [P, P, SZ, U, P, P, P, P, P]
        getattr(L, f"dapi_record{s}").argtypes = [P, C.c_int, P, SZ, P, SZ, U, P, P, P, P, P]
        getattr(L, f"dapi_host_record{s}").argtypes = [P, C.c_int, P, SZ, P, P, SZ, U, P, P, P, P, P]
        getattr(L, f"dapi_accel_capacity_check{s}").argtypes = [P, SZ, SZ, C.POINTER(C.c_size_t)]
    L.dapi_last_error.restype = C.c_char_p
    return L


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def sfx(dtype):
    return "3f" if np.dtype(dtype) == np.float32 else "3d"


def dev_trace(dapi, bvh, rays, flags):
    n = rays.shape[0]
    ids, inner = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    t, u, v = (np.zeros(n, rays.dtype) for _ in range(3))
    rc = getattr(dapi, f"dapi_trace{sfx(rays.dtype)}")(C.c_void_p(bvh.handle), _p(rays), n, flags, _p(ids), _p(t), _p(u), _p(v), _p(inner))
    assert rc == 0, dapi.dapi_last_error()
    return ids, t, u, v, inner


def record(dapi, bvh, leaf, rays, flags, spheres=None, start=NO_START, host=False, verts=None):
    n = rays.shape[0]
    ids, leaves, inner = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    t, hashes = np.zeros(n, rays.dtype), np.zeros(n, np.uint64)
    s = sfx(rays.dtype)
    if host:
        rc = getattr(dapi, f"dapi_host_record{s}")(C.c_void_p(bvh.handle), leaf, _p(rays), n, _p(verts), _p(spheres), start, flags,
                                                   _p(ids), _p(t), _p(leaves), _p(hashes), _p(inner))
    else:
        rc = getattr(dapi, f"dapi_record{s}")(C.c_void_p(bvh.handle), leaf, _p(rays), n, _p(spheres), start, flags,
                                              _p(ids), _p(t), _p(leaves), _p(hashes), _p(inner))
    assert rc == 0, dapi.dapi_last_error()
    return ids, t, leaves, hashes, inner


def bits(a):
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def special_rays(tris, dtype):
    from tests.test_device_api_host import extra_rays
    return extra_rays(tris, dtype)


SCENES = [("soup", 1_000_000, 3163, np.float32), ("grid", 1_000_000, 3163, np.float32), ("soup", 100_000, 1000, np.float64)]


@pytest.fixture(scope="module", params=SCENES, ids=["c2-soup", "c2-grid", "c5"])
def scene(request, gpu_lib):
    kind, n, img, dtype = request.param
    tris = scenes.make_mesh(kind, n, dtype=dtype)
    rays = scenes.make_primary(kind, img, img, dtype=dtype)
    bvh = gpu_lib.Bvh.build_triangles(tris)
    yield tris, rays, bvh
    bvh.destroy()


@pytest.mark.parametrize("flags", [0, 2, 1], ids=["closest", "robust", "any"])
def test_triangles_equal_batched_kernel(dapi, gpu_lib, scene, flags):
    """The triangle leaf through DeviceView::intersect equals bvhNN_intersect_rays(BVH_TIE_LAST_VISITED | flags) bit for
    bit, and its inner-hook count equals the statistics kernel's inner steps."""
    api = gpu_lib
    tris, rays, bvh = scene
    want, stats = bvh.intersect_rays(rays, flags=flags | api.TIE_LAST_VISITED, stats=True)
    ids, t, u, v, inner = dev_trace(dapi, bvh, rays, flags)
    assert (ids.astype(np.uint64) == want["prim_id"].astype(np.uint64) & 0xFFFFFFFF).all()
    for got, key in ((t, "t"), (u, "u"), (v, "v")):
        assert (bits(got) == bits(np.ascontiguousarray(want[key]))).all(), key
    assert (inner == stats["inner_steps"]).all()
    assert (ids != 0xFFFFFFFF).sum() > rays.shape[0] // 10


@pytest.mark.parametrize("flags", [0, 2, 1, 3], ids=["closest", "robust", "any", "any-robust"])
@pytest.mark.parametrize("leaf", [LEAF_TRI, LEAF_NONE], ids=["tri", "record-only"])
def test_leaf_order_equals_host(dapi, scene, flags, leaf):
    """Per ray: the same leaf calls in the same order, the same inner steps and the same hit as Bvh::intersect on the
    host mirror, from the root and from a node below it, NaN-interval and degenerate rays included."""
    tris, rays, bvh = scene
    rng = np.random.default_rng(5)
    m = 100_000 if leaf == LEAF_TRI else 20_000         # a leaf that never shrinks tmax visits every leaf the ray's line crosses
    sub = np.concatenate([rays[np.sort(rng.choice(rays.shape[0], m, replace=False))], special_rays(tris, rays.dtype)])
    for start in (NO_START, 2):
        dev = record(dapi, bvh, leaf, sub, flags, start=start)
        host = record(dapi, bvh, leaf, sub, flags, start=start, host=True, verts=tris)
        for name, a, b in zip(("ids", "t", "leaves", "hashes", "inner"), dev, host):
            same = bits(a) == bits(b) if a.dtype.kind == "f" else a == b
            assert same.all(), f"{name} differs at {np.nonzero(~same)[0][:8]} (start {start})"


def sphere_scene(n=100_000, seed=3):
    rng = np.random.default_rng(seed)
    centers = rng.random((n, 3), dtype=np.float32)
    radii = (0.002 + 0.004 * rng.random(n)).astype(np.float32)
    bboxes = np.concatenate([centers - radii[:, None], centers + radii[:, None]], axis=1).astype(np.float32)
    spheres = np.ascontiguousarray(np.concatenate([centers, radii[:, None]], axis=1), np.float32)
    # rays from outside the unit cube towards random points inside it
    m = 50_000
    org = np.stack([rng.random(m), rng.random(m), np.full(m, -1.0)], axis=1).astype(np.float32)
    target = rng.random((m, 3)).astype(np.float32)
    rays = np.zeros((m, 8), np.float32)
    rays[:, :3], rays[:, 3:6], rays[:, 6], rays[:, 7] = org, target - org, 0.0, np.inf
    return centers, bboxes, spheres, rays


def sphere_brute_force(spheres, rays, chunk=64):
    """sphere_hit of tests/device_api_kernels.cu in float32, same operation order, over every sphere: (ids, t, whether the
    closest distance is unique)."""
    parts = [_sphere_brute_force(spheres, rays[k:k + chunk]) for k in range(0, rays.shape[0], chunk)]
    return tuple(np.concatenate(p) for p in zip(*parts))


def _sphere_brute_force(spheres, rays):
    f = np.float32
    c, r = spheres[None, :, :3], spheres[None, :, 3]
    org, d = rays[:, None, :3], rays[:, None, 3:6]
    oc = org - c

    def dot(a, b):
        return ((f(0) + a[..., 0] * b[..., 0]) + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]
    a = dot(d, d)
    b = f(2) * dot(d, oc)
    cc = dot(oc, oc) - r * r
    delta = b * b - f(4) * a * cc
    with np.errstate(invalid="ignore", divide="ignore"):
        inv = -f(0.5) / a
        sq = np.sqrt(np.maximum(delta, f(0)))
        n0, n1 = (b + sq) * inv, (b - sq) * inv
    tmin, tmax = rays[:, None, 6], rays[:, None, 7]
    t0 = np.where(n0 > tmin, n0, tmin)
    t1 = np.where(n1 < tmax, n1, tmax)
    t0 = np.where((delta >= 0) & (t0 <= t1), t0, np.inf).astype(np.float32)
    best = t0.argmin(axis=1)
    tb = t0[np.arange(rays.shape[0]), best]
    unique = (t0 == tb[:, None]).sum(axis=1) == 1
    return np.where(np.isfinite(tb), best, 0xFFFFFFFF).astype(np.uint32), tb, unique


def test_spheres_from_boxes(dapi, gpu_lib):
    """A tree built from sphere boxes (no triangles: view.tris is NULL) traced with the reference's sphere test as the
    leaf: bit-identical to Bvh::intersect with the same leaf on the host mirror, and the ids of a NumPy brute force."""
    centers, bboxes, spheres, rays = sphere_scene()
    bvh = gpu_lib.Bvh.build(bboxes, centers)
    assert bvh.device_view()["tris"] == 0
    for flags in (0, 2):
        dev = record(dapi, bvh, LEAF_SPHERE, rays, flags, spheres=spheres)
        host = record(dapi, bvh, LEAF_SPHERE, rays, flags, spheres=spheres, host=True)
        assert (dev[0] == host[0]).all() and (bits(dev[1]) == bits(host[1])).all()
        assert (dev[2] == host[2]).all() and (dev[3] == host[3]).all() and (dev[4] == host[4]).all()
    ids = dev[0]
    assert (ids != 0xFFFFFFFF).sum() > 1000
    sub = slice(0, 2000)
    want, t, unique = sphere_brute_force(spheres, rays[sub])
    assert (ids[sub][unique] == want[unique]).all()
    assert (bits(dev[1][sub][unique & (want != 0xFFFFFFFF)]) == bits(t[unique & (want != 0xFFFFFFFF)])).all()
    bvh.destroy()


def test_view_follows_mirror_edits(dapi, gpu_lib):
    """An edited leaf box (bvh_node3f_set_bbox) plus bvh3f_refit: a fresh view traces the edited tree."""
    api = gpu_lib
    tris = scenes.make_mesh("soup", 20_000)
    rays = scenes.make_primary("soup", 200, 200)
    bvh = api.Bvh.build_triangles(tris)
    before = bvh.device_view()
    bounds, index_values, prim_ids = bvh.arrays()
    # the leaf holding the triangle the most rays hit
    hit_ids = bvh.intersect_rays(rays)["prim_id"]
    top = np.bincount(hit_ids[hit_ids != 0xFFFFFFFF].astype(np.int64)).argmax()
    slot = int(np.nonzero(prim_ids == top)[0][0])
    first, count = (index_values >> 4).astype(np.int64), (index_values & 15).astype(np.int64)
    leaf = int(np.nonzero((count > 0) & (first <= slot) & (slot < first + count))[0][0])
    # shrink one leaf's box to a point far away: its triangles can no longer be reached
    L = api.lib()
    L.bvh_node3f_set_bbox.argtypes = [P, P]
    box = (C.c_float * 6)(50, 50, 50, 50.5, 50.5, 50.5)         # struct bvh_bbox3f {min xyz, max xyz}
    node = bvh._f("get_node")(bvh.handle, leaf)
    L.bvh_node3f_set_bbox(C.c_void_p(node), box)
    bvh.refit()
    after = bvh.device_view()
    assert after["nodes"] != 0 and after["node_count"] == before["node_count"]      # the edited mirror was uploaded
    dev = record(dapi, bvh, LEAF_TRI, rays, 0)
    host = record(dapi, bvh, LEAF_TRI, rays, 0, host=True, verts=tris)
    for a, b in zip(dev, host):
        assert (bits(a) == bits(b)).all() if a.dtype.kind == "f" else (a == b).all()
    unedited = api.Bvh.build_triangles(tris)
    base = record(dapi, unedited, LEAF_TRI, rays, 0)
    assert (base[0] != dev[0]).any(), "the edit changed nothing: pick another leaf"
    bvh.destroy(); unedited.destroy()


def test_errors(dapi, gpu_lib):
    api = gpu_lib
    L = api.lib()
    v = api.DeviceView()
    assert L.bvh3f_get_device_view(None, C.byref(v)) != 0 and "null handle" in api.last_error()
    tris = scenes.make_mesh("soup", 1000)
    bvh = api.Bvh.build_triangles(tris)
    assert L.bvh3f_get_device_view(C.c_void_p(bvh.handle), None) != 0 and "null view" in api.last_error()
    view = bvh.device_view()
    assert view["prim_count"] == 1000 and view["tris"] != 0 and view["node_count"] == bvh.node_count
    depth = C.c_size_t(0)
    assert dapi.dapi_accel_capacity_check3f(_p(tris), 1000, 1, C.byref(depth)) == 1          # too small: throws
    assert depth.value == view["depth"]
    assert dapi.dapi_accel_capacity_check3f(_p(tris), 1000, depth.value + 1, C.byref(depth)) == 0
    bvh.destroy()
