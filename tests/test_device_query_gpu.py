"""bvhNN_build_boxes and DeviceView::traverse_top_down on the GPU: trees built from device-resident boxes are bit for bit
those of bvhNN_build, queries written with the caller's node test (tests/device_query_kernels.cu) make the same leaf
calls as Bvh::traverse_top_down on the host mirror and find what a brute force finds, and build, query, refit and query
again run in order on one torch stream."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes
from tests.test_device_api_gpu import sphere_scene

pytestmark = pytest.mark.gpu

P, SZ, U = C.c_void_p, C.c_size_t, C.c_uint
ARRAY_STACK, SHARED_STACK = 0, 1


@pytest.fixture(scope="module")
def dq(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_query_tests())
    for s in ("3f", "3d"):
        getattr(L, f"dq_overlap{s}").argtypes = [P, P, P, SZ, C.c_int, P, P, P, P, P]
        getattr(L, f"dq_nearest{s}").argtypes = [P, P, P, SZ, C.c_int, P, P, P, P, P]
        getattr(L, f"dq_host_overlap{s}").argtypes = [P, P, P, SZ, P, P, P, P, P]
        getattr(L, f"dq_host_nearest{s}").argtypes = [P, P, P, SZ, P, P, P, P, P]
        getattr(L, f"dq_accel_from_boxes{s}").argtypes = [P, P, SZ, U, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    L.dq_last_error.restype = C.c_char_p
    return L


def bits(a):
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def sphere_boxes(n, dtype, seed=1):
    """n spheres in the unit cube, radii about half the mean spacing: (boxes (n, 6) min3 max3, centres (n, 3))."""
    rng = np.random.default_rng(seed)
    c = rng.random((n, 3))
    r = (0.5 + rng.random(n)) * 0.5 / np.cbrt(n)
    return np.concatenate([c - r[:, None], c + r[:, None]], axis=1).astype(dtype), c.astype(dtype)


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def id_hash(ids):
    """dq::id_hash (tests/device_queries.h), vectorised."""
    x = ids.astype(np.uint64) + np.uint64(0x9E3779B97F4A7C15)
    with np.errstate(over="ignore"):
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def brute_overlap(boxes, queries, chunk=16):
    """Per query box: the count of primitive boxes overlapping it and the sum of their id hashes (mod 2^64)."""
    h = id_hash(np.arange(boxes.shape[0]))
    counts, sums = [], []
    for k in range(0, queries.shape[0], chunk):
        q = queries[k:k + chunk, None, :]
        hit = ((boxes[None, :, 0] <= q[..., 3]) & (q[..., 0] <= boxes[None, :, 3]) & (boxes[None, :, 1] <= q[..., 4]) &
               (q[..., 1] <= boxes[None, :, 4]) & (boxes[None, :, 2] <= q[..., 5]) & (q[..., 2] <= boxes[None, :, 5]))
        counts.append(hit.sum(axis=1))
        with np.errstate(over="ignore"):
            sums.append(np.array([h[row].sum(dtype=np.uint64) for row in hit], np.uint64))
    return np.concatenate(counts).astype(np.uint32), np.concatenate(sums)


def query_boxes(boxes, m, seed):
    """Boxes of random primitives grown by up to their own size, a few large boxes, inverted ones and NaN ones."""
    rng = np.random.default_rng(seed)
    b = boxes[rng.integers(boxes.shape[0], size=m)].astype(np.float64)
    size = (b[:, 3:] - b[:, :3]) * rng.random((m, 1)) * 2
    q = np.concatenate([b[:, :3] - size, b[:, 3:] + size], axis=1)
    q[::97, :3] -= 0.05
    q[::97, 3:] += 0.05
    q[1::101] = q[1::101][:, [3, 4, 5, 0, 1, 2]]                      # inverted
    q[2::103, 1] = np.nan
    return q.astype(boxes.dtype)


class Run:
    """The query kernels on device buffers (torch), the host traversal on the mirror, and their outputs as numpy."""

    def __init__(self, dq, bvh):
        self.dq, self.bvh, self.s = dq, bvh, bvh.s

    def overlap(self, d_boxes, d_queries, m, stack, record=True):
        import torch
        out = [torch.zeros(m, dtype=t, device="cuda") for t in (torch.int32, torch.int64, torch.int32, torch.int64, torch.int32)]
        ptrs = [o.data_ptr() for o in out] if record else [out[0].data_ptr(), out[1].data_ptr(), None, None, None]
        rc = getattr(self.dq, f"dq_overlap{self.s}")(C.c_void_p(self.bvh.handle), d_boxes.data_ptr(), d_queries.data_ptr(), m,
                                                     stack, *ptrs)
        assert rc == 0, self.dq.dq_last_error()
        return out

    def nearest(self, d_centers, d_points, m, stack):
        import torch
        dt = torch.float32 if self.s == "3f" else torch.float64
        out = [torch.zeros(m, dtype=torch.int32, device="cuda"), torch.zeros(m, dtype=dt, device="cuda")] + \
              [torch.zeros(m, dtype=t, device="cuda") for t in (torch.int32, torch.int64, torch.int32)]
        rc = getattr(self.dq, f"dq_nearest{self.s}")(C.c_void_p(self.bvh.handle), d_centers.data_ptr(), d_points.data_ptr(), m,
                                                     stack, *[o.data_ptr() for o in out])
        assert rc == 0, self.dq.dq_last_error()
        return out

    def host(self, name, a, b, dtype2):
        m = b.shape[0]
        out = [np.zeros(m, np.uint32), np.zeros(m, dtype2), np.zeros(m, np.uint32), np.zeros(m, np.uint64), np.zeros(m, np.uint32)]
        rc = getattr(self.dq, f"dq_host_{name}{self.s}")(C.c_void_p(self.bvh.handle), a.ctypes.data, b.ctypes.data, m,
                                                         *[o.ctypes.data for o in out])
        assert rc == 0, self.dq.dq_last_error()
        return out


def to_numpy(outs):
    import torch
    torch.cuda.synchronize()
    res = [o.cpu().numpy() for o in outs]
    return [r.view(np.uint32) if r.dtype == np.int32 else r.view(np.uint64) if r.dtype == np.int64 else r for r in res]


# -- build parity -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 2, 1000, 1_000_000])
@pytest.mark.parametrize("leaf", [(1, 8), (2, 4)], ids=["leaf1-8", "leaf2-4"])
@pytest.mark.parametrize("quality", ["low", "medium", "high"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
def test_build_boxes_equals_build(gpu_lib, dtype, quality, leaf, n):
    api = gpu_lib
    import torch
    boxes, centers = sphere_boxes(n, dtype, seed=n)
    cfg = dict(quality=quality, min_leaf_size=leaf[0], max_leaf_size=leaf[1])
    want = api.Bvh.build(boxes, centers, **cfg)
    d_boxes, d_centers = cuda(boxes), cuda(centers)
    torch.cuda.synchronize()                            # the handle's private stream reads what torch wrote
    got = api.Bvh.build_boxes(d_boxes.data_ptr(), d_centers.data_ptr(), count=n, dtype=dtype, flags=api.DEVICE_POINTERS, **cfg)
    host = api.Bvh.build_boxes(boxes, centers, **cfg)
    wb, wi, wids = want.arrays()
    for b in (got, host):
        bb, bi, bids = b.arrays()
        assert (bits(bb) == bits(wb)).all() and (bi == wi).all() and (bids == wids).all()
        assert b.depth == want.depth and b.device_view()["depth"] == want.device_view()["depth"]
        b.destroy()
    want.destroy()


def test_accel_from_boxes(dq, gpu_lib):
    """bvh::v2::cuda::Accel::from_boxes on device pointers: the device view of the tree Bvh.build gives."""
    api = gpu_lib
    import torch
    boxes, centers = sphere_boxes(5000, np.float32)
    want = api.Bvh.build(boxes, centers).device_view()
    d_boxes, d_centers = cuda(boxes), cuda(centers)
    torch.cuda.synchronize()
    nodes, depth = C.c_size_t(0), C.c_size_t(0)
    assert dq.dq_accel_from_boxes3f(d_boxes.data_ptr(), d_centers.data_ptr(), 5000, api.DEVICE_POINTERS, C.byref(nodes), C.byref(depth)) == 0
    assert (nodes.value, depth.value) == (want["node_count"], want["depth"])
    assert dq.dq_accel_from_boxes3f(d_boxes.data_ptr(), None, 5000, api.DEVICE_POINTERS, C.byref(nodes), C.byref(depth)) == -1
    assert b"Accel::from_boxes: build_boxes: null centres" in dq.dq_last_error()


# -- query parity ------------------------------------------------------------------------------------------------------

def soup_boxes():
    tris = scenes.make_mesh("soup", 1_000_000).reshape(-1, 3, 3)
    return np.concatenate([tris.min(axis=1), tris.max(axis=1)], axis=1), tris.mean(axis=1, dtype=np.float32)


@pytest.fixture(scope="module", params=["spheres-100k", "c2-soup"])
def scene(request, gpu_lib):
    import torch
    if request.param == "spheres-100k":
        centers, boxes, _, _ = sphere_scene()
    else:
        boxes, centers = soup_boxes()
    boxes, centers = np.ascontiguousarray(boxes, np.float32), np.ascontiguousarray(centers, np.float32)
    d_boxes, d_centers = cuda(boxes), cuda(centers)
    torch.cuda.synchronize()
    bvh = gpu_lib.Bvh.build_boxes(d_boxes.data_ptr(), d_centers.data_ptr(), count=boxes.shape[0], dtype=np.float32,
                                  flags=gpu_lib.DEVICE_POINTERS)
    yield boxes, centers, d_boxes, d_centers, bvh
    bvh.destroy()


def test_overlap_queries(dq, scene):
    """Both stacks make the host traversal's leaf calls; the overlap sets equal a brute force."""
    boxes, centers, d_boxes, _, bvh = scene
    run = Run(dq, bvh)
    queries = query_boxes(boxes, 3000, seed=5)
    d_q = cuda(queries)
    host = run.host("overlap", boxes, queries, np.uint64)
    for stack in (ARRAY_STACK, SHARED_STACK):
        dev = to_numpy(run.overlap(d_boxes, d_q, queries.shape[0], stack))
        for name, a, b in zip(("count", "ids", "leaves", "hash", "nodes"), dev, host):
            assert (a == b).all(), f"{name} differs at {np.nonzero(a != b)[0][:8]} (stack {stack})"
    m = 3000 if boxes.shape[0] <= 100_000 else 300
    count, ids = brute_overlap(boxes, queries[:m])
    assert (dev[0][:m] == count).all() and (dev[1][:m] == ids).all()
    assert count.sum() > m and (count == 0).any()


def test_nearest_queries(dq, scene):
    """Both stacks make the host traversal's leaf calls; the nearest centre is the k-d tree's."""
    from scipy.spatial import cKDTree
    boxes, centers, _, d_centers, bvh = scene
    run = Run(dq, bvh)
    rng = np.random.default_rng(9)
    lo, hi = boxes[:, :3].min(axis=0), boxes[:, 3:].max(axis=0)
    points = (lo + (hi - lo) * (rng.random((5000, 3)) * 1.2 - 0.1)).astype(np.float32)
    d_p = cuda(points)
    host = run.host("nearest", centers, points, np.float32)
    for stack in (ARRAY_STACK, SHARED_STACK):
        dev = to_numpy(run.nearest(d_centers, d_p, points.shape[0], stack))
        for name, a, b in zip(("id", "dist2", "leaves", "hash", "nodes"), dev, host):
            same = bits(a) == bits(b) if a.dtype.kind == "f" else a == b
            assert same.all(), f"{name} differs at {np.nonzero(~same)[0][:8]} (stack {stack})"
    dist, idx = cKDTree(centers.astype(np.float64)).query(points.astype(np.float64), k=2)
    got = np.sqrt(dev[1].astype(np.float64))
    assert np.allclose(got, dist[:, 0], rtol=1e-5, atol=1e-6)
    clear = dist[:, 1] - dist[:, 0] > 1e-4 * (1 + dist[:, 0])
    assert clear.mean() > 0.9 and (dev[0][clear] == idx[clear, 0]).all()
    assert dev[2].max() < centers.shape[0] // 8                    # a search, not a scan


# -- one stream ----------------------------------------------------------------------------------------------------------

def test_build_query_refit_query_on_one_stream(dq, gpu_lib):
    """torch writes the boxes, build_boxes, an overlap query, torch moves the spheres, refit_boxes, the query again:
    every frame on one torch stream with no synchronisation but the build's own, each checked against a brute force."""
    api = gpu_lib
    import torch
    n, m = 100_000, 2000
    rng = np.random.default_rng(4)
    c0 = rng.random((n, 3)).astype(np.float32)
    r0 = (0.002 + 0.004 * rng.random(n)).astype(np.float32)
    steps = [(0.02 * (rng.random((n, 3)) - 0.5)).astype(np.float32) for _ in range(3)]
    queries = query_boxes(np.concatenate([c0 - r0[:, None], c0 + r0[:, None]], axis=1), m, seed=6)
    stream = torch.cuda.Stream()
    api.set_stream(stream.cuda_stream)
    frames, outs = [], []
    try:
        with torch.cuda.stream(stream):
            c, r = cuda(c0), cuda(r0)[:, None]
            d_q, moves = cuda(queries), [cuda(s) for s in steps]
            boxes = torch.cat([c - r, c + r], dim=1)
            bvh = api.Bvh.build_boxes(boxes.data_ptr(), c.data_ptr(), count=n, dtype=np.float32, flags=api.DEVICE_POINTERS)
            run = Run(dq, bvh)
            for frame in range(4):
                if frame:
                    c.add_(moves[frame - 1])
                    torch.cat([c - r, c + r], dim=1, out=boxes)
                    bvh.refit_boxes(boxes.data_ptr(), api.DEVICE_POINTERS)
                outs.append(run.overlap(boxes, d_q, m, SHARED_STACK if frame % 2 else ARRAY_STACK, record=False))
                frames.append(boxes.clone())
    finally:
        api.set_stream(None)
    assert bvh.get_property("stream") == stream.cuda_stream
    stream.synchronize()
    for frame, (out, b) in enumerate(zip(outs, frames)):
        count, ids = brute_overlap(b.cpu().numpy(), queries)
        got = to_numpy(out[:2])
        assert (got[0] == count).all() and (got[1] == ids).all(), f"frame {frame}"
        assert count.sum() > m
    bvh.destroy()


# -- errors --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
def test_errors(gpu_lib, dtype):
    api = gpu_lib
    import torch
    boxes, centers = sphere_boxes(100, dtype)
    d_boxes, d_centers = cuda(boxes), cuda(centers)
    torch.cuda.synchronize()
    f = getattr(api.lib(), f"bvh{api._sfx(dtype)}_build_boxes")
    D = api.DEVICE_POINTERS
    cases = [((None, d_centers.data_ptr(), 100, None, D), "null boxes"), ((d_boxes.data_ptr(), None, 100, None, D), "null centres"),
             ((None, centers.ctypes.data, 100, None, 0), "null boxes"), ((boxes.ctypes.data, None, 100, None, 0), "null centres"),
             ((d_boxes.data_ptr(), d_centers.data_ptr(), 0, None, D), "prim_count out of range"),
             ((boxes.ctypes.data, centers.ctypes.data, 0, None, 0), "prim_count out of range"),
             ((d_boxes.data_ptr(), d_centers.data_ptr(), 1 << 32, None, D), "prim_count out of range")]
    if dtype == np.float32:                             # first ids of 2n - 1 nodes must fit 28 bits; nothing is read
        cases.append(((d_boxes.data_ptr(), d_centers.data_ptr(), (1 << 27) + 1, None, D), "too many primitives"))
    for args, message in cases:
        assert not f(*args) and message in api.last_error(), (message, api.last_error())
    with pytest.raises(api.BvhError, match="null centres"):
        api.Bvh.build_boxes(d_boxes.data_ptr(), 0, count=100, dtype=dtype, flags=D)
    ok = api.Bvh.build_boxes(d_boxes.data_ptr(), d_centers.data_ptr(), count=100, dtype=dtype, flags=D)
    assert ok.prim_count == 100
    ok.destroy()
