"""bvhNN_refit_boxes on the GPU: bit-identical to the host path (leaf boxes written into the mirror, then bvhNN_refit) and
to the reference's refit, traces of the moved scene, a triangle handle with the wide tree, stream order with torch, and
the error cases."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes
from tests.helpers import assert_hits_equal, hits_tuple
from tests.test_device_api_gpu import LEAF_SPHERE, bits, dapi, record, sphere_brute_force, sphere_scene  # noqa: F401
from tests.test_refit_boxes_host import fold_leaf_boxes

pytestmark = pytest.mark.gpu

DTYPES = pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])


def moved_spheres(spheres, seed, dtype):
    """Centres moved and radii rescaled; (n, 4) spheres and their (n, 6) boxes in `dtype`."""
    rng = np.random.default_rng(seed)
    n = spheres.shape[0]
    c = spheres[:, :3] + (0.02 * (rng.random((n, 3)) - 0.5)).astype(np.float32)
    r = spheres[:, 3] * (0.5 + rng.random(n)).astype(np.float32)
    out = np.concatenate([c, r[:, None]], axis=1).astype(dtype)
    boxes = np.concatenate([out[:, :3] - out[:, 3:], out[:, :3] + out[:, 3:]], axis=1)
    return np.ascontiguousarray(out), np.ascontiguousarray(boxes)


def host_path_refit(api, bvh, leaf_bounds, index_values):
    """The way without this entry point: every leaf box through bvh_nodeNN_set_bbox, then bvhNN_refit."""
    s = bvh.s
    ct = C.c_float if s == "3f" else C.c_double
    L = api.lib()
    set_bbox = getattr(L, f"bvh_node{s}_set_bbox")
    set_bbox.argtypes = [C.c_void_p, C.c_void_p]
    for i in np.nonzero((index_values & 15) != 0)[0]:
        b = leaf_bounds[i]
        box = (ct * 6)(b[0], b[2], b[4], b[1], b[3], b[5])          # struct bvh_bboxNN {min xyz, max xyz}
        set_bbox(C.c_void_p(bvh._f("get_node")(bvh.handle, int(i))), box)
    bvh.refit()


@DTYPES
def test_bit_identical_to_host_path(gpu_lib, oracle, tmp_path, dtype):
    api = gpu_lib
    import torch
    centers, bboxes, spheres, _ = sphere_scene()
    a = api.Bvh.build(bboxes.astype(dtype), centers.astype(dtype))
    path = str(tmp_path / "tree.bin")
    a.save(path)
    b = api.Bvh.load(path, dtype)                       # the same tree, refitted the host way
    _, index0, ids0 = a.arrays()
    view0 = a.device_view()
    for frame, pointers in enumerate(("host", "device")):
        _, boxes = moved_spheres(spheres, seed=frame, dtype=dtype)
        if pointers == "host":
            a.refit_boxes(boxes)
        else:
            d = torch.from_numpy(boxes).cuda()
            torch.cuda.synchronize()
            a.refit_boxes(d.data_ptr(), api.DEVICE_POINTERS)
            a.sync()
        bounds, index_values, ids = a.arrays()
        assert (index_values == index0).all() and (ids == ids0).all()
        folded = fold_leaf_boxes(index_values, ids, boxes, dtype)
        tree = oracle.from_arrays(folded, index_values, ids)
        oracle.refit(tree)
        assert (bits(bounds) == bits(tree.arrays()[0])).all(), f"{pointers}: differs from the reference's refit"
        host_path_refit(api, b, folded, index_values)
        assert (bits(bounds) == bits(b.arrays()[0])).all(), f"{pointers}: differs from the host path"
        assert a.device_view()["nodes"] == view0["nodes"]
    a.destroy(); b.destroy()


@DTYPES
def test_traces_after_refit(dapi, gpu_lib, dtype):  # noqa: F811
    """The sphere leaf through DeviceView::intersect on the refitted tree equals Bvh::intersect on the refreshed mirror,
    and (float) the ids of a brute force over the moved spheres wherever the closest hit is unique."""
    api = gpu_lib
    centers, bboxes, spheres, rays = sphere_scene()
    bvh = api.Bvh.build(bboxes.astype(dtype), centers.astype(dtype))
    moved, boxes = moved_spheres(spheres, seed=7, dtype=dtype)
    view = bvh.device_view()
    bvh.refit_boxes(boxes)
    assert bvh.device_view()["nodes"] == view["nodes"]
    rays = rays.astype(dtype)
    for flags in (0, api.ROBUST):
        dev = record(dapi, bvh, LEAF_SPHERE, rays, flags, spheres=moved)
        host = record(dapi, bvh, LEAF_SPHERE, rays, flags, spheres=moved, host=True)
        assert (dev[0] == host[0]).all() and (bits(dev[1]) == bits(host[1])).all()
        assert (dev[2] == host[2]).all() and (dev[3] == host[3]).all() and (dev[4] == host[4]).all()
    ids = dev[0]
    assert (ids != 0xFFFFFFFF).sum() > 1000
    if dtype == np.float32:
        sub = slice(0, 2000)
        want, _, unique = sphere_brute_force(moved, rays[sub])
        assert (ids[sub][unique] == want[unique]).all()
    bvh.destroy()


def test_triangle_handle_with_wide_tree(gpu_lib, oracle):
    """Triangles stay attached and untouched; boxes grown by a margin still enclose them, so every kernel finds the
    brute-force hits, and the wide companion tree is rebuilt from the refitted boxes."""
    api = gpu_lib
    api.set_option("use_wide", 1)
    try:
        tris = scenes.soup(20_000)
        bvh = api.Bvh.build_triangles(tris)
        assert bvh.get_property("wide_nodes") > 0
        bb, _ = oracle.tri_bboxes_centers(tris)
        grown = bb + np.array([-1, -1, -1, 1, 1, 1], np.float32) * np.float32(0.01)
        bvh.refit_boxes(grown)
        assert bvh.get_property("wide_nodes") > 0
        bounds, index_values, ids = bvh.arrays()
        leaf = (index_values & 15) != 0
        assert (bits(bounds[leaf]) == bits(fold_leaf_boxes(index_values, ids, grown, np.float32)[leaf])).all()
        rays = scenes.make_primary("soup", 120, 120)
        want = oracle.brute_force(tris, rays)
        assert (want[0] != 0xFFFFFFFF).sum() > 1000
        for flags in (0, api.ROBUST, api.KERNEL_WIDE):
            assert_hits_equal(hits_tuple(bvh.intersect_rays(rays, flags=flags)), want, f"flags {flags}")
        bvh.destroy()
    finally:
        api.set_option("use_wide", 0)


def test_stream_order_with_torch(gpu_lib, oracle):
    """Frames of (torch op rewrites the boxes in place, refit_boxes, intersect_rays) on one stream, no synchronisation
    in between.  Frames alternate between boxes moved far away (every ray misses) and boxes grown around the triangles
    (the brute-force hits): a refit that read another frame's boxes, or a trace that ran before its refit, shows."""
    api = gpu_lib
    import torch
    stream = torch.cuda.Stream()
    api.set_stream(stream.cuda_stream)
    try:
        tris = scenes.soup(20_000)
        bvh = api.Bvh.build_triangles(tris)
        assert bvh.get_property("stream") == stream.cuda_stream
    finally:
        api.set_stream(None)
    rays = scenes.make_primary("soup", 100, 100)
    bb, _ = oracle.tri_bboxes_centers(tris)
    want = oracle.brute_force(tris, rays)
    m = rays.shape[0]
    with torch.cuda.stream(stream):
        base = torch.from_numpy(bb).cuda()
        d_rays = torch.from_numpy(rays).cuda()
        boxes = torch.empty_like(base)
        far = torch.full((6,), 100.0, device="cuda")
        grow = torch.tensor([-0.01, -0.01, -0.01, 0.01, 0.01, 0.01], device="cuda")
        hits = [torch.empty((m, 16), dtype=torch.uint8, device="cuda") for _ in range(6)]
        for frame in range(6):
            torch.add(base, far if frame % 2 == 0 else grow, out=boxes)
            bvh.refit_boxes(boxes.data_ptr(), api.DEVICE_POINTERS)
            bvh.intersect_rays(d_rays.data_ptr(), m, hits[frame].data_ptr(), flags=api.DEVICE_POINTERS)
    stream.synchronize()
    for frame, h in enumerate(hits):
        got = h.cpu().numpy().view(api.HIT3F).reshape(m)
        if frame % 2 == 0:
            assert (got["prim_id"] == 0xFFFFFFFF).all(), f"frame {frame}"
        else:
            assert_hits_equal(hits_tuple(got), want, f"frame {frame}")
    bvh.destroy()


@DTYPES
def test_errors_leave_the_tree_as_it_was(dapi, gpu_lib, tmp_path, dtype):  # noqa: F811
    api = gpu_lib
    import torch
    centers, bboxes, spheres, rays = sphere_scene(n=20_000)
    bvh = api.Bvh.build(bboxes.astype(dtype), centers.astype(dtype))
    spheres, rays = spheres.astype(dtype), rays.astype(dtype)
    before = record(dapi, bvh, LEAF_SPHERE, rays, 0, spheres=spheres)
    bounds_before = bvh.arrays()[0]
    _, moved = moved_spheres(spheres.astype(np.float32), seed=3, dtype=dtype)
    d = torch.from_numpy(moved).cuda()
    torch.cuda.synchronize()
    f = getattr(api.lib(), f"bvh{bvh.s}_refit_boxes")
    n = bvh.prim_count
    h = C.c_void_p(bvh.handle)
    cases = [((None, moved.ctypes.data, n, 0), "null handle"), ((h, None, n, 0), "null boxes"),
             ((h, moved.ctypes.data, n - 1, 0), "prim_count"), ((h, d.data_ptr(), n + 1, api.DEVICE_POINTERS), "prim_count")]
    for args, message in cases:
        assert f(*args) != 0 and message in api.last_error(), message
    assert (bits(bvh.arrays()[0]) == bits(bounds_before)).all()
    after = record(dapi, bvh, LEAF_SPHERE, rays, 0, spheres=spheres)
    for a, b in zip(before, after):
        assert (bits(a) == bits(b)).all() if a.dtype.kind == "f" else (a == b).all()
    bvh.destroy()
    # a handle loaded from a file without nodes holds no tree
    empty = tmp_path / "empty.bin"
    empty.write_bytes(bytes(16))
    e = api.Bvh.load(str(empty), dtype)
    assert f(C.c_void_p(e.handle), moved.ctypes.data, 0, 0) != 0 and "no BVH" in api.last_error()
    e.destroy()
