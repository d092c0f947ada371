"""DeviceView::query on the GPU (test queriers in tests/device_query_batch_kernels.cu): per query the same results, leaf
calls and node calls as one thread per query through traverse_top_down (the kernels of libdevice_query_kernels.so and
libdevice_bottom_up_kernels.so, loaded as they are), answers equal to a brute force and a k-d tree, every query finished
exactly once at the scheduler's edges, build -> query -> refit -> query on one torch stream, and the errors."""
import ctypes as C

import numpy as np
import pytest

from tests.test_device_bottom_up_gpu import Pass, particles
from tests.test_device_query_gpu import brute_overlap, bits, cuda, query_boxes, sphere_boxes
from tests.test_device_trace_gpu import load_chain

pytestmark = pytest.mark.gpu

P, SZ = C.c_void_p, C.c_size_t
OVERLAP, NEAREST, CONTAINS = 0, 1, 2


@pytest.fixture(scope="module")
def dqb(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_query_batch_tests())
    for s, t in (("3f", C.c_float), ("3d", C.c_double)):
        getattr(L, f"dqb_query{s}").argtypes = [P, C.c_int, C.c_int, C.c_int, P, P, SZ, P, P, P, P, P, P, P, SZ, P]
        getattr(L, f"dqb_potential{s}").argtypes = [P, P, P, P, P, P, SZ, t, t, P, P, P, SZ, P]
        getattr(L, f"dqb_workspace_bytes{s}").argtypes = [P]
        getattr(L, f"dqb_workspace_bytes{s}").restype = SZ
    L.dqb_last_error.restype = C.c_char_p
    return L


@pytest.fixture(scope="module")
def dq(gpu_lib):
    """libdevice_query_kernels.so: the one-thread-per-query overlap and nearest kernels."""
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_query_tests())
    for s in ("3f", "3d"):
        getattr(L, f"dq_overlap{s}").argtypes = [P, P, P, SZ, C.c_int, P, P, P, P, P]
        getattr(L, f"dq_nearest{s}").argtypes = [P, P, P, SZ, C.c_int, P, P, P, P, P]
    L.dq_last_error.restype = C.c_char_p
    return L


@pytest.fixture(scope="module")
def bu(gpu_lib):
    """libdevice_bottom_up_kernels.so: mass and centre per node, and the one-thread-per-point potential."""
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_bottom_up_tests())
    for s, t in (("3f", C.c_float), ("3d", C.c_double)):
        getattr(L, f"bu_workspace_bytes{s}").argtypes = [P, C.POINTER(C.c_size_t)]
        getattr(L, f"bu_mass{s}").argtypes = [P, P, SZ, P, P, P, P]
        getattr(L, f"bu_potential{s}").argtypes = [P, P, P, P, P, P, SZ, t, t, P, P]
    L.bu_last_error.restype = C.c_char_p
    return L


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def to_host(outs):
    import torch
    torch.cuda.synchronize()
    res = [o.cpu().numpy() for o in outs]
    return [r.view(np.uint32) if r.dtype == np.int32 else r.view(np.uint64) if r.dtype == np.int64 else r for r in res]


class Batch:
    """dqb_query on one handle with one workspace; outputs are torch tensors (r0, r1, leaves, hashes, nodes)."""

    def __init__(self, dqb, bvh):
        import torch
        self.dqb, self.bvh, self.s = dqb, bvh, bvh.s
        self.bytes = getattr(dqb, f"dqb_workspace_bytes{self.s}")(C.c_void_p(bvh.handle))
        assert self.bytes == 8
        self.ws = torch.empty(self.bytes, dtype=torch.uint8, device="cuda")

    def __call__(self, kind, d_prims, d_queries, m, any_hit=False, per_thread=False, record=True, counts=None, stream=None,
                 ws=None, ws_bytes=None):
        import torch
        r1_type = torch.int64 if kind == OVERLAP else torch.int32 if kind == CONTAINS else \
            (torch.float32 if self.s == "3f" else torch.float64)
        k = max(m, 1)                                            # (an empty tensor's address is null)
        out = [torch.zeros(k, dtype=torch.int32, device="cuda"), torch.zeros(k, dtype=r1_type, device="cuda")]
        if record:
            out += [torch.zeros(k, dtype=t, device="cuda") for t in (torch.int32, torch.int64, torch.int32)]
        rec = [ptr(o) for o in out[2:]] if record else [None, None, None]
        ws = self.ws if ws is None else ws
        rc = getattr(self.dqb, f"dqb_query{self.s}")(C.c_void_p(self.bvh.handle), kind, int(per_thread), int(any_hit), ptr(d_prims),
                                                     ptr(d_queries), m, ptr(out[0]), ptr(out[1]), *rec, ptr(counts), ptr(ws),
                                                     self.bytes if ws_bytes is None else ws_bytes, stream)
        if rc:
            raise (ValueError if rc == -2 else RuntimeError)(self.dqb.dqb_last_error().decode())
        return out


def per_thread_reference(dq, bvh, kind, d_prims, d_queries, m):
    """The same query one thread per query, through libdevice_query_kernels.so (array stack)."""
    import torch
    dt = torch.int64 if kind == OVERLAP else (torch.float32 if bvh.s == "3f" else torch.float64)
    out = [torch.zeros(m, dtype=torch.int32, device="cuda"), torch.zeros(m, dtype=dt, device="cuda")] + \
          [torch.zeros(m, dtype=t, device="cuda") for t in (torch.int32, torch.int64, torch.int32)]
    f = getattr(dq, f"dq_{'overlap' if kind == OVERLAP else 'nearest'}{bvh.s}")
    rc = f(C.c_void_p(bvh.handle), d_prims.data_ptr(), d_queries.data_ptr(), m, 0, *[o.data_ptr() for o in out])
    assert rc == 0, dq.dq_last_error()
    return out


def assert_same(got, want, what):
    for name, a, b in zip(("r0", "r1", "leaves", "hash", "nodes"), got, want):
        same = bits(a) == bits(b) if a.dtype.kind == "f" else a == b
        assert same.all(), f"{what}: {name} differs at {np.nonzero(~same)[0][:8]}"


def points_in(boxes, m, seed):
    rng = np.random.default_rng(seed)
    lo, hi = boxes[:, :3].min(axis=0).astype(np.float64), boxes[:, 3:].max(axis=0).astype(np.float64)
    return (lo + (hi - lo) * (rng.random((m, 3)) * 1.2 - 0.1)).astype(boxes.dtype)


def build(api, boxes, centers, quality="medium", leaf=(1, 8)):
    import torch
    d_boxes, d_centers = cuda(boxes), cuda(centers)
    torch.cuda.synchronize()
    bvh = api.Bvh.build_boxes(d_boxes.data_ptr(), d_centers.data_ptr(), count=boxes.shape[0], dtype=boxes.dtype,
                              flags=api.DEVICE_POINTERS, quality=quality, min_leaf_size=leaf[0], max_leaf_size=leaf[1])
    return bvh, d_boxes, d_centers


# -- the same as one thread per query -----------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 1000, 1_000_000])
@pytest.mark.parametrize("leaf", [(1, 1), (1, 8)], ids=["leaf1-1", "leaf1-8"])
@pytest.mark.parametrize("quality", ["low", "medium", "high"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
def test_same_as_per_thread(dqb, dq, gpu_lib, dtype, quality, leaf, n):
    """Overlap and nearest through query equal the one-thread-per-query kernels of libdevice_query_kernels.so per query:
    count and id hash / nearest id and squared distance, leaf calls, the hash of the leaf ranges, node calls.
    Containment, IsAnyHit both ways, equals the same querier one thread per query."""
    boxes, centers = sphere_boxes(n, dtype, seed=n + 3)
    bvh, d_boxes, d_centers = build(gpu_lib, boxes, centers, quality, leaf)
    run = Batch(dqb, bvh)
    m = min(max(4 * n, 1000), 200_000)
    qb, pts = query_boxes(boxes, m, seed=n), points_in(boxes, m, seed=n + 1)
    d_qb, d_pts = cuda(qb), cuda(pts)
    for kind, prims, queries in ((OVERLAP, d_boxes, d_qb), (NEAREST, d_centers, d_pts)):
        got = to_host(run(kind, prims, queries, m))
        want = to_host(per_thread_reference(dq, bvh, kind, prims, queries, m))
        assert_same(got, want, f"kind {kind}")
        assert got[2].sum() > 0
    every = None
    for any_hit in (False, True):
        got = to_host(run(CONTAINS, d_boxes, d_pts, m, any_hit=any_hit))
        want = to_host(run(CONTAINS, d_boxes, d_pts, m, any_hit=any_hit, per_thread=True))
        assert_same(got, want, f"contains any_hit={any_hit}")
        if any_hit:
            # the query ends in the first leaf that finds a containing box: found iff the full search finds one, with
            # no more finds and no more leaf calls than it
            assert ((got[1] > 0) == (every[1] > 0)).all()
            assert (got[1] <= every[1]).all() and (got[2] <= every[2]).all()
        else:
            every = got
        if n > 1:
            assert (got[1] > 0).any()
    bvh.destroy()


# -- correct answers ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
def test_answers(dqb, gpu_lib, dtype):
    """Overlap sets equal a brute force on a sample; nearest centres are the k-d tree's."""
    from scipy.spatial import cKDTree
    boxes, centers = sphere_boxes(200_000, dtype, seed=21)
    bvh, d_boxes, d_centers = build(gpu_lib, boxes, centers)
    run = Batch(dqb, bvh)
    qb = query_boxes(boxes, 20_000, seed=22)
    count, ids = to_host(run(OVERLAP, d_boxes, cuda(qb), qb.shape[0], record=False))
    bf_count, bf_ids = brute_overlap(boxes, qb[:500])
    assert (count[:500] == bf_count).all() and (ids[:500] == bf_ids).all()
    assert bf_count.sum() > 500 and (bf_count == 0).any()
    pts = points_in(boxes, 20_000, seed=23)
    nid, d2 = to_host(run(NEAREST, d_centers, cuda(pts), pts.shape[0], record=False))
    dist, idx = cKDTree(centers.astype(np.float64)).query(pts.astype(np.float64), k=2)
    assert np.allclose(np.sqrt(d2.astype(np.float64)), dist[:, 0], rtol=1e-5, atol=1e-6)
    clear = dist[:, 1] - dist[:, 0] > 1e-4 * (1 + dist[:, 0])
    assert clear.mean() > 0.9 and (nid[clear] == idx[clear, 0]).all()
    bvh.destroy()


# -- Barnes-Hut ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
def test_barnes_hut(dqb, bu, gpu_lib, dtype):
    """The three-argument node test reads mass and centre written by traverse_bottom_up: the potential through query
    equals the per-thread kernel of libdevice_bottom_up_kernels.so bit for bit, with the particles in their original order
    and in BVH order."""
    import torch
    boxes, centers = sphere_boxes(300_000, dtype, seed=31)
    bvh = gpu_lib.Bvh.build(boxes, centers)
    pos, mass = particles(centers, dtype)
    run = Pass(bu, bvh)
    d_pos, d_mass = cuda(pos), cuda(mass)
    node_mass, node_centre = run.mass(d_pos, d_mass)
    ids = bvh.arrays()[2].astype(np.int64)
    ws = torch.empty(8, dtype=torch.uint8, device="cuda")
    eps2 = 1e-6
    for order in (np.arange(pos.shape[0]), ids):
        d_points = cuda(pos[order])
        for theta in (0.5, 0.0):
            want_phi, want_used = run.potential(d_pos, d_mass, node_mass, node_centre, d_points, theta, eps2)
            phi = torch.zeros_like(want_phi)
            used = torch.zeros_like(want_used)
            rc = getattr(dqb, f"dqb_potential{bvh.s}")(C.c_void_p(bvh.handle), d_pos.data_ptr(), d_mass.data_ptr(),
                                                       node_mass.data_ptr(), node_centre.data_ptr(), d_points.data_ptr(),
                                                       d_points.shape[0], theta * theta, eps2, phi.data_ptr(), used.data_ptr(),
                                                       ws.data_ptr(), 8, None)
            assert rc == 0, dqb.dqb_last_error()
            got_phi, got_used, w_phi, w_used = to_host([phi, used, want_phi, want_used])
            assert (bits(got_phi) == bits(w_phi)).all() and (got_used == w_used).all(), theta
            assert (got_used > 0).all() if theta else (got_used == 0).all()
    bvh.destroy()


# -- every query finished exactly once -------------------------------------------------------------------------------------

def test_every_query_once(dqb, gpu_lib):
    """finish is called once per query at the sizes where the scheduling changes; nothing past n is written."""
    import torch
    boxes, centers = sphere_boxes(100_000, np.float32, seed=41)
    bvh, d_boxes, _ = build(gpu_lib, boxes, centers)
    run = Batch(dqb, bvh)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    warps = sms * 9 * 4                                          # one resident wave: 9 blocks of 4 warps per SM
    run_len = 64                                                 # persistent_run_rays for large batches
    big = (1 << 20) + 7
    qb = cuda(query_boxes(boxes, big, seed=42))
    guard = 1000
    sizes = [0, 1, 31, 32, 33, 63, 64, 65, run_len - 1, run_len + 1, warps * 32 + 1, warps * run_len - 1, warps * run_len + 1,
             warps * run_len * 3 + 17, big]
    for n in sizes:
        counts = torch.zeros(n + guard, dtype=torch.int32, device="cuda")
        run(OVERLAP, d_boxes, qb, n, record=False, counts=counts)
        got = to_host([counts])[0]
        assert (got[:n] == 1).all(), (n, np.nonzero(got[:n] != 1)[0][:8])
        assert (got[n:] == 0).all(), n
    bvh.destroy()


# -- one stream ---------------------------------------------------------------------------------------------------------

def test_build_query_refit_query_on_one_stream(dqb, dq, gpu_lib):
    """torch writes the boxes, build_boxes, query, torch moves the spheres, refit_boxes, query again: one torch stream with
    no host synchronisation between the steps.  The results after the refit equal the per-thread kernel's on the
    refitted tree; the first frame's equal a brute force."""
    import torch
    api = gpu_lib
    n, m = 100_000, 5000
    rng = np.random.default_rng(51)
    c0 = rng.random((n, 3)).astype(np.float32)
    r0 = (0.002 + 0.004 * rng.random(n)).astype(np.float32)
    step = (0.03 * (rng.random((n, 3)) - 0.5)).astype(np.float32)
    qb = query_boxes(np.concatenate([c0 - r0[:, None], c0 + r0[:, None]], axis=1), m, seed=52)
    stream = torch.cuda.Stream()
    api.set_stream(stream.cuda_stream)
    outs = []
    try:
        with torch.cuda.stream(stream):
            c, r, d_step, d_q = cuda(c0), cuda(r0)[:, None], cuda(step), cuda(qb)
            boxes = torch.cat([c - r, c + r], dim=1)
            bvh = api.Bvh.build_boxes(boxes.data_ptr(), c.data_ptr(), count=n, dtype=np.float32, flags=api.DEVICE_POINTERS)
            run = Batch(dqb, bvh)
            first_boxes = boxes.clone()
            outs.append(run(OVERLAP, boxes, d_q, m, stream=C.c_void_p(stream.cuda_stream)))
            c.add_(d_step)
            torch.cat([c - r, c + r], dim=1, out=boxes)
            bvh.refit_boxes(boxes.data_ptr(), api.DEVICE_POINTERS)
            outs.append(run(OVERLAP, boxes, d_q, m, stream=C.c_void_p(stream.cuda_stream)))
    finally:
        api.set_stream(None)
    stream.synchronize()
    first, second = to_host(outs[0]), to_host(outs[1])
    count, ids = brute_overlap(first_boxes.cpu().numpy(), qb)
    assert (first[0] == count).all() and (first[1] == ids).all()
    torch.cuda.synchronize()
    want = to_host(per_thread_reference(dq, bvh, OVERLAP, boxes, d_q, m))
    assert_same(second, want, "after refit")
    assert (second[0] != first[0]).any(), "moving the spheres changed no overlap"
    bvh.destroy()


# -- errors -------------------------------------------------------------------------------------------------------------

def test_workspace(dqb, gpu_lib):
    """A workspace that is too small is refused with its message; a reused workspace gives the same results."""
    import torch
    boxes, centers = sphere_boxes(50_000, np.float32, seed=61)
    bvh, d_boxes, _ = build(gpu_lib, boxes, centers)
    run = Batch(dqb, bvh)
    d_q = cuda(query_boxes(boxes, 50_000, seed=62))
    ws = torch.empty(8, dtype=torch.uint8, device="cuda")
    first = to_host(run(OVERLAP, d_boxes, d_q, 50_000, ws=ws))
    second = to_host(run(OVERLAP, d_boxes, d_q, 50_000, ws=ws))
    assert_same(first, second, "reused workspace")
    with pytest.raises(ValueError, match="DeviceView::query: a workspace of 7 bytes is too small"):
        run(OVERLAP, d_boxes, d_q, 50_000, ws=ws, ws_bytes=7)
    bvh.destroy()


def test_too_deep_tree_throws(dqb, gpu_lib, tmp_path):
    """A chain tree of depth 399 (float) needs more than 200 KB of shared-memory stack per block: query throws before
    it launches anything; depth 398 runs, and an accept-everything box visits every leaf."""
    import torch
    q = np.array([[-1, -1, -1, 2, 2, 2]] * 40, np.float32)
    for depth, ok in ((398, True), (399, False)):
        bvh = load_chain(gpu_lib, tmp_path, depth)
        run = Batch(dqb, bvh)
        prims = cuda(np.tile(np.array([[0, 0, 0, 1, 1, 1]], np.float32), (bvh.prim_count, 1)))
        counts = torch.zeros(40, dtype=torch.int32, device="cuda")
        if ok:
            out = to_host(run(OVERLAP, prims, cuda(q), 40, counts=counts))
            assert (to_host([counts])[0] == 1).all()
            assert (out[2] == bvh.node_count // 2 + 1).all() and (out[0] == bvh.prim_count).all()
        else:
            with pytest.raises(ValueError, match="DeviceView::query: a tree of depth 399 needs .* shared-memory stack"):
                run(OVERLAP, prims, cuda(q), 40, counts=counts)
            assert (to_host([counts])[0] == 0).all()
        bvh.destroy()
