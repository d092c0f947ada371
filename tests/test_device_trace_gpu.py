"""DeviceView::trace on the GPU (test tracers in tests/device_trace_kernels.cu): the triangle leaf bit for bit equal to
bvhNN_intersect_rays, leaf-call sequences equal to one thread per ray through DeviceView::intersect, every ray finished
exactly once, spheres from device boxes, trees at the edges, and a one-stream torch pipeline."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes

pytestmark = pytest.mark.gpu

P, SZ, U = C.c_void_p, C.c_size_t, C.c_uint
LEAF_NONE, LEAF_TRI, LEAF_SPHERE, LEAF_TRI_NAN = 0, 1, 2, 3
FLAGS = [0, 2, 1, 3]
FLAG_IDS = ["closest", "robust", "any", "any-robust"]


@pytest.fixture(scope="module")
def dtr(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_trace_tests())
    for s in ("3f", "3d"):
        getattr(L, f"dtr_run{s}").argtypes = [P, C.c_int, C.c_int, U, P, SZ, P, P, P, P, P, P, P, P, P, SZ, P]
        getattr(L, f"dtr_workspace_bytes{s}").argtypes = [P]
        getattr(L, f"dtr_workspace_bytes{s}").restype = SZ
    L.dtr_last_error.restype = C.c_char_p
    return L


def sfx(dtype):
    return "3f" if np.dtype(dtype) == np.float32 else "3d"


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def bits(a):
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class Run:
    """One dtr_run call over device-resident rays; outputs are torch tensors."""

    def __init__(self, dtr, bvh, dtype):
        import torch
        self.dtr, self.bvh, self.s = dtr, bvh, sfx(dtype)
        self.tdtype = torch.float32 if self.s == "3f" else torch.float64
        self.ws = torch.empty(64, dtype=torch.uint8, device="cuda")

    def __call__(self, d_rays, n, leaf, flags, per_thread=False, spheres=None, stream=None, counts=None, ws=None, ws_bytes=None,
                 sync=True):
        import torch
        dev = "cuda"
        ids = torch.empty(n, dtype=torch.int32, device=dev)
        t, u, v = (torch.empty(n, dtype=self.tdtype, device=dev) for _ in range(3))
        calls = torch.empty(n, dtype=torch.int32, device=dev)
        hashes = torch.empty(n, dtype=torch.int64, device=dev)
        ws = self.ws if ws is None else ws
        ws_bytes = ws.numel() if ws_bytes is None else ws_bytes
        rc = getattr(self.dtr, f"dtr_run{self.s}")(C.c_void_p(self.bvh.handle), int(per_thread), leaf, flags, ptr(d_rays), n,
                                                   ptr(spheres), ptr(ids), ptr(t), ptr(u), ptr(v), ptr(calls), ptr(hashes),
                                                   ptr(counts), ptr(ws), ws_bytes, stream)
        if rc:
            raise (ValueError if rc == -2 else RuntimeError)(self.dtr.dtr_last_error().decode())
        out = (ids, t, u, v, calls, hashes)
        if not sync:
            return out
        torch.cuda.synchronize()
        return tuple(host(x) for x in out)


def special_rays(tris, dtype):
    from tests.test_device_api_host import extra_rays
    return extra_rays(tris, dtype)


SCENES = [("soup", 1_000_000, 3163, np.float32), ("grid", 1_000_000, 1000, np.float32), ("soup", 100_000, 1000, np.float64)]


@pytest.fixture(scope="module", params=SCENES, ids=["c2-soup", "c2-grid", "c5"])
def scene(request, gpu_lib):
    kind, n, img, dtype = request.param
    tris = scenes.make_mesh(kind, n, dtype=dtype)
    rays = np.concatenate([scenes.make_primary(kind, img, img, dtype=dtype), special_rays(tris, dtype)])
    bvh = gpu_lib.Bvh.build_triangles(tris)
    yield tris, rays, bvh
    bvh.destroy()


@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
def test_triangles_equal_batched_kernel(dtr, gpu_lib, scene, flags):
    """The triangle leaf through trace equals bvhNN_intersect_rays(BVH_TIE_LAST_VISITED | flags) bit for bit (the full
    c2 soup batch; 1M rays elsewhere), special rays included."""
    api = gpu_lib
    tris, rays, bvh = scene
    want = bvh.intersect_rays(rays, flags=flags | api.TIE_LAST_VISITED)
    ids, t, u, v, _, _ = Run(dtr, bvh, rays.dtype)(cuda(rays), rays.shape[0], LEAF_TRI, flags)
    assert (ids.view(np.uint32).astype(np.uint64) == want["prim_id"].astype(np.uint64) & 0xFFFFFFFF).all()
    for got, key in ((t, "t"), (u, "u"), (v, "v")):
        assert (bits(got) == bits(np.ascontiguousarray(want[key]))).all(), key
    assert (ids != -1).sum() > rays.shape[0] // 10


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
@pytest.mark.parametrize("leaf", [LEAF_NONE, LEAF_TRI, LEAF_TRI_NAN], ids=["none", "tri", "tri-nan"])
def test_leaf_calls_equal_per_thread(dtr, gpu_lib, dtype, flags, leaf):
    """Per ray the leaf-call count, the hash of the (begin, end) sequence, the id and tmax equal one thread per ray
    through DeviceView::intersect with the same leaf."""
    kind = "soup"
    tris = scenes.make_mesh(kind, 200_000, dtype=dtype)
    rays = np.concatenate([scenes.make_primary(kind, 1000, 1000, dtype=dtype), special_rays(tris, dtype)])
    bvh = gpu_lib.Bvh.build_triangles(tris)
    run, d_rays, n = Run(dtr, bvh, dtype), cuda(rays), rays.shape[0]
    got = run(d_rays, n, leaf, flags)
    want = run(d_rays, n, leaf, flags, per_thread=True)
    for name, a, b in zip(("ids", "t", "u", "v", "calls", "hashes"), got, want):
        same = bits(a) == bits(b) if a.dtype.kind == "f" else a == b
        assert same.all(), f"{name} differs at {np.nonzero(~same)[0][:8]}"
    assert got[4].sum() > n
    bvh.destroy()


def sphere_scene(n, m, seed=3):
    rng = np.random.default_rng(seed)
    centers = rng.random((n, 3), dtype=np.float32)
    radii = (0.0005 + 0.001 * rng.random(n)).astype(np.float32)
    spheres = np.ascontiguousarray(np.concatenate([centers, radii[:, None]], axis=1), np.float32)
    org = np.stack([rng.random(m), rng.random(m), np.full(m, -1.0)], axis=1).astype(np.float32)
    target = rng.random((m, 3)).astype(np.float32)
    rays = np.zeros((m, 8), np.float32)
    rays[:, :3], rays[:, 3:6], rays[:, 6], rays[:, 7] = org, target - org, 0.0, np.inf
    return centers, radii, spheres, rays


def sphere_boxes(c, r):
    import torch
    return torch.cat([c - r, c + r], dim=1).contiguous()


@pytest.mark.parametrize("flags", [0, 2, 1], ids=["closest", "robust", "any"])
def test_spheres(dtr, gpu_lib, flags):
    """1M spheres built with build_boxes from device arrays: trace equals the per-thread sphere kernel bit for bit, and a
    brute force on a subset of rays wherever the closest hit is unique."""
    import torch
    from tests.test_device_api_gpu import sphere_brute_force
    api = gpu_lib
    centers, radii, spheres, rays = sphere_scene(1_000_000, 1_000_000)
    c, r, d_spheres, d_rays = cuda(centers), cuda(radii)[:, None], cuda(spheres), cuda(rays)
    boxes = sphere_boxes(c, r)
    torch.cuda.synchronize()
    bvh = api.Bvh.build_boxes(boxes.data_ptr(), c.data_ptr(), count=centers.shape[0], dtype=np.float32, flags=api.DEVICE_POINTERS)
    run = Run(dtr, bvh, np.float32)
    got = run(d_rays, rays.shape[0], LEAF_SPHERE, flags, spheres=d_spheres)
    want = run(d_rays, rays.shape[0], LEAF_SPHERE, flags, spheres=d_spheres, per_thread=True)
    for name, a, b in zip(("ids", "t", "u", "v", "calls", "hashes"), got, want):
        assert (bits(a) == bits(b)).all() if a.dtype.kind == "f" else (a == b).all(), name
    ids = got[0].view(np.uint32)
    assert (ids != 0xFFFFFFFF).sum() > 10_000
    if flags == 0:
        sub = slice(0, 200)
        bf_ids, bf_t, unique = sphere_brute_force(spheres, rays[sub], chunk=4)
        assert (ids[sub][unique] == bf_ids[unique]).all()
        hit = unique & (bf_ids != 0xFFFFFFFF)
        assert (bits(got[1][sub][hit]) == bits(bf_t[hit])).all()
    bvh.destroy()


def test_every_ray_once(dtr, gpu_lib):
    """finish is called once per ray for batch sizes around the scheduler's edges; nothing past n is written."""
    import torch
    tris = scenes.make_mesh("soup", 100_000)
    rays = scenes.make_primary("soup", 1001, 1001)
    bvh = gpu_lib.Bvh.build_triangles(tris)
    run = Run(dtr, bvh, np.float32)
    props = torch.cuda.get_device_properties(0)
    wave = props.multi_processor_count * 9 * 4 * 32           # one resident wave of warps (9 blocks of 4 warps per SM), in rays
    d_rays = cuda(np.resize(rays, (max(wave + 1, 1_000_003), 8)))
    guard = 1000
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 4097, wave - 1, wave, wave + 1, 1_000_003):
        counts = torch.zeros(n + guard, dtype=torch.int32, device="cuda")
        run(d_rays, n, LEAF_NONE, 0, counts=counts)
        got = host(counts)
        assert (got[:n] == 1).all(), (n, np.nonzero(got[:n] != 1)[0][:8])
        assert (got[n:] == 0).all(), n
    bvh.destroy()


def test_one_primitive_tree(dtr, gpu_lib):
    """The root is a leaf: every ray, NaN-interval ones included, gets exactly one leaf call."""
    tri = np.array([[0, 0, 0, 1, 0, 0, 0, 1, 0]], np.float32)
    bvh = gpu_lib.Bvh.build_triangles(tri)
    rays = np.concatenate([np.array([[0.2, 0.2, 1, 0, 0, -1, 0, np.inf], [0.2, 0.2, 1, 0, 0, -1, np.nan, np.inf],
                                     [5, 5, 1, 0, 0, -1, 0, np.inf]], np.float32), special_rays(tri, np.float32)])
    run = Run(dtr, bvh, np.float32)
    for flags in FLAGS:
        ids, t, _, _, calls, _ = run(cuda(rays), rays.shape[0], LEAF_TRI, flags)
        assert (calls == 1).all()
        assert ids[0] == 0 and t[0] == 1.0 and ids[1] == -1 and ids[2] == -1
    bvh.destroy()


def save_chain(path, inner):
    """A chain of `inner` inner nodes in the reference's serialized float format (u32 node and primitive counts, then
    per node six bounds and the u32 index first_id << 4 | count, then the u32 primitive ids): inner node k is node 2k,
    its left child 2k + 1 is a one-primitive leaf and its right child 2k + 2 is the next inner node (the last one a leaf)."""
    import struct
    nodes, prim = [], 0
    for k in range(inner):
        nodes.append(((2 * k + 1) << 4) | 0)
        nodes.append((prim << 4) | 1)
        prim += 1
    nodes.append((prim << 4) | 1)
    prim += 1
    with open(path, "wb") as f:
        f.write(struct.pack("<II", len(nodes), prim))
        for index in nodes:
            f.write(struct.pack("<6fI", 0, 1, 0, 1, 0, 1, index))
        f.write(struct.pack(f"<{prim}I", *range(prim)))


def load_chain(api, tmp_path, depth):
    """A loaded chain tree whose reported depth is `depth`."""
    path = tmp_path / f"chain{depth}.bvh"
    save_chain(path, depth)
    bvh = api.Bvh.load(str(path), dtype=np.float32)
    if bvh.depth != depth:                              # (whether the root counts)
        inner = 2 * depth - bvh.depth
        bvh.destroy()
        save_chain(path, inner)
        bvh = api.Bvh.load(str(path), dtype=np.float32)
    assert bvh.depth == depth
    return bvh


def test_too_deep_tree_throws(dtr, gpu_lib, tmp_path):
    """A chain tree deeper than 398 (float) needs more than 200 KB of shared-memory stack per block: trace throws
    std::length_error before it launches anything; depth 398 runs, and every ray visits every leaf."""
    import torch
    rays = np.array([[0.5, 0.5, -1, 0, 0, 1, 0, np.inf]] * 40, np.float32)
    for depth, ok in ((398, True), (399, False)):
        bvh = load_chain(gpu_lib, tmp_path, depth)
        run = Run(dtr, bvh, np.float32)
        counts = torch.zeros(40, dtype=torch.int32, device="cuda")
        if ok:
            calls = run(cuda(rays), 40, LEAF_NONE, 0, counts=counts)[4]
            assert (host(counts) == 1).all()
            assert (calls == bvh.node_count // 2 + 1).all()
        else:
            with pytest.raises(ValueError, match="shared-memory stack"):
                run(cuda(rays), 40, LEAF_NONE, 0, counts=counts)
            torch.cuda.synchronize()
            assert (host(counts) == 0).all()
        bvh.destroy()


def test_workspace(dtr, gpu_lib):
    """A reused workspace gives the same results; one that is too small is refused with a message."""
    import torch
    tris = scenes.make_mesh("soup", 100_000)
    rays = scenes.make_primary("soup", 500, 500)
    bvh = gpu_lib.Bvh.build_triangles(tris)
    run, d_rays, n = Run(dtr, bvh, np.float32), cuda(rays), rays.shape[0]
    assert dtr.dtr_workspace_bytes3f(C.c_void_p(bvh.handle)) == 8
    ws = torch.empty(8, dtype=torch.uint8, device="cuda")
    first = run(d_rays, n, LEAF_TRI, 0, ws=ws)
    second = run(d_rays, n, LEAF_TRI, 0, ws=ws)
    for a, b in zip(first, second):
        assert (bits(a) == bits(b)).all() if a.dtype.kind == "f" else (a == b).all()
    with pytest.raises(ValueError, match="workspace of 7 bytes is too small"):
        run(d_rays, n, LEAF_TRI, 0, ws=ws, ws_bytes=7)
    bvh.destroy()


def test_build_trace_refit_trace_on_one_stream(dtr, gpu_lib):
    """torch writes the boxes, build_boxes, trace, torch moves the spheres, refit_boxes, trace again: one torch stream, no
    synchronisation between the steps.  Both results equal the same steps run synchronously."""
    import torch
    api = gpu_lib
    centers, radii, spheres, rays = sphere_scene(200_000, 200_000, seed=9)
    step = (0.02 * (np.random.default_rng(4).random((centers.shape[0], 3)) - 0.5)).astype(np.float32)
    d_rays = cuda(rays)
    torch.cuda.synchronize()

    def frames(sync):
        stream = torch.cuda.Stream()
        api.set_stream(stream.cuda_stream)
        out = []
        try:
            with torch.cuda.stream(stream):
                c, r, d_step = cuda(centers), cuda(radii)[:, None], cuda(step)
                boxes = sphere_boxes(c, r)
                bvh = api.Bvh.build_boxes(boxes.data_ptr(), c.data_ptr(), count=centers.shape[0], dtype=np.float32,
                                          flags=api.DEVICE_POINTERS)
                run = Run(dtr, bvh, np.float32)
                for frame in range(2):
                    if frame:
                        c.add_(d_step)
                        torch.cat([c - r, c + r], dim=1, out=boxes)
                        bvh.refit_boxes(boxes.data_ptr(), api.DEVICE_POINTERS)
                        if sync:
                            stream.synchronize()
                    sph = torch.cat([c, r], dim=1).contiguous()
                    res = run(d_rays, rays.shape[0], LEAF_SPHERE, 0, spheres=sph, stream=C.c_void_p(stream.cuda_stream), sync=False)
                    out.append(tuple(x.clone() for x in res))
                    if sync:
                        stream.synchronize()
        finally:
            api.set_stream(None)
        stream.synchronize()
        bvh.destroy()
        return [tuple(host(x) for x in f) for f in out]

    fast, slow = frames(False), frames(True)
    for a, b in zip(fast, slow):
        for x, y in zip(a, b):
            assert (bits(x) == bits(y)).all() if x.dtype.kind == "f" else (x == y).all()
    assert (fast[0][1] != fast[1][1]).any(), "moving the spheres changed no hit"
