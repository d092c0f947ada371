"""DeviceView::trace_triangles on the GPU (test shaders in tests/device_triangle_trace_kernels.cu): accept-all bit for bit
equal to bvhNN_intersect_rays under every flag and both tie rules, filters equal to one thread per ray through
DeviceView::intersect, secondary rays that skip their origin triangle equal to a brute force, in-kernel camera rays,
every ray finished once, the errors, and a one-stream torch pipeline."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes

pytestmark = pytest.mark.gpu

P, SZ, U = C.c_void_p, C.c_size_t, C.c_uint
ALL, REJECT_ALL, EVEN_IDS, ALPHA, NOT_ORIGIN = range(5)
ANY, ROBUST, LAST = 1, 2, 4
MODES = [0, ROBUST, ANY, ANY | ROBUST]
MODE_IDS = ["closest", "robust", "any", "any-robust"]


@pytest.fixture(scope="module")
def dtt(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_triangle_trace_tests())
    for s in ("3f", "3d"):
        getattr(L, f"dtt_run{s}").argtypes = [P, C.c_int, C.c_int, U, P, SZ, P, P, P, P, P, P, P, P, P, SZ, P]
    L.dtt_camera3f.argtypes = [P, P, C.c_uint32, C.c_uint32, P, P, SZ, P]
    L.dtt_camera_rays3f.argtypes = [P, C.c_uint32, C.c_uint32, P, P]
    L.dtt_workspace_bytes3f.argtypes = [P]
    L.dtt_workspace_bytes3f.restype = SZ
    L.dtt_last_error.restype = C.c_char_p
    return L


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def bits(a):
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def check(dtt, rc):
    if rc:
        msg = dtt.dtt_last_error().decode()
        raise {-2: ValueError, -3: TypeError}.get(rc, RuntimeError)(msg)


class Run:
    """One dtt_run call over device-resident rays; outputs are (ids, t, u, v, calls, hashes)."""

    def __init__(self, dtt, bvh, dtype):
        import torch
        self.dtt, self.bvh = dtt, bvh
        self.s = "3f" if np.dtype(dtype) == np.float32 else "3d"
        self.tdtype = torch.float32 if self.s == "3f" else torch.float64
        self.ws = torch.empty(64, dtype=torch.uint8, device="cuda")

    def __call__(self, d_rays, n, filt, flags, per_thread=False, origins=None, counts=None, ws=None, ws_bytes=None,
                 stream=None, sync=True):
        import torch
        ids = torch.empty(n, dtype=torch.int32, device="cuda")
        t, u, v = (torch.empty(n, dtype=self.tdtype, device="cuda") for _ in range(3))
        calls = torch.empty(n, dtype=torch.int32, device="cuda")
        hashes = torch.empty(n, dtype=torch.int64, device="cuda")
        ws = self.ws if ws is None else ws
        ws_bytes = ws.numel() if ws_bytes is None else ws_bytes
        check(self.dtt, getattr(self.dtt, f"dtt_run{self.s}")(C.c_void_p(self.bvh.handle), int(per_thread), filt, flags,
                                                              ptr(d_rays), n, ptr(origins), ptr(ids), ptr(t), ptr(u), ptr(v),
                                                              ptr(calls), ptr(hashes), ptr(counts), ptr(ws), ws_bytes, stream))
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
    yield tris, rays, bvh, cuda(rays)
    bvh.destroy()


@pytest.mark.parametrize("last", [False, True], ids=["lowest-id", "last-visited"])
@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
def test_accept_all_equals_library(dtt, gpu_lib, scene, flags, last):
    """Every hit accepted, rays from an array and records to an array: bit for bit bvhNN_intersect_rays(flags) in id, t, u
    and v, the full c2 soup batch (10M rays) included, special rays included."""
    tris, rays, bvh, d_rays = scene
    lib_flags = flags | (gpu_lib.TIE_LAST_VISITED if last else 0)
    want = bvh.intersect_rays(rays, flags=lib_flags)
    ids, t, u, v, calls, _ = Run(dtt, bvh, rays.dtype)(d_rays, rays.shape[0], ALL, flags | (LAST if last else 0))
    assert (ids.view(np.uint32).astype(np.uint64) == want["prim_id"].astype(np.uint64) & 0xFFFFFFFF).all()
    for got, key in ((t, "t"), (u, "u"), (v, "v")):
        assert (bits(got) == bits(np.ascontiguousarray(want[key]))).all(), key
    assert (ids != -1).sum() > rays.shape[0] // 10
    assert (calls[ids != -1] >= 1).all() and (calls[ids == -1] == 0).all()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
@pytest.mark.parametrize("mode", range(8), ids=[f"{m}-{t}" for t in ("lowest", "last") for m in MODE_IDS])
def test_filters_equal_per_thread(dtt, gpu_lib, dtype, mode):
    """Filters on odd ids, an alpha cut-out and the origin triangle: per ray the record, the accept-call count and the hash
    of the accept sequence equal one thread per ray through DeviceView::intersect with the same leaf, tie rule and filter."""
    import torch
    flags = MODES[mode % 4] | (LAST if mode >= 4 else 0)
    tris = scenes.make_mesh("soup", 200_000, dtype=dtype)
    rays = np.concatenate([scenes.make_primary("soup", 700, 700, dtype=dtype), special_rays(tris, dtype)])
    bvh = gpu_lib.Bvh.build_triangles(tris)
    run, d_rays, n = Run(dtt, bvh, dtype), cuda(rays), rays.shape[0]
    origins = torch.from_numpy(run(d_rays, n, ALL, 0)[0].view(np.uint32).copy()).cuda()
    for filt in (REJECT_ALL, EVEN_IDS, ALPHA, NOT_ORIGIN):
        got = run(d_rays, n, filt, flags, origins=origins)
        want = run(d_rays, n, filt, flags, per_thread=True, origins=origins)
        for name, a, b in zip(("ids", "t", "u", "v", "calls", "hashes"), got, want):
            same = bits(a) == bits(b) if a.dtype.kind == "f" else a == b
            assert same.all(), f"filter {filt}: {name} differs at {np.nonzero(~same)[0][:8]}"
        assert got[4].sum() > n // 10, filt
        if filt == REJECT_ALL:
            assert (got[0] == -1).all()
    bvh.destroy()


def brute_force_closest(tris, rays, origins, chunk=16):
    """Closest hit of every ray over every triangle, the origin triangle skipped, lowest id at equal t: PrecomputedTri
    (the oracle's triangle test, reference tri.h:30-37,55-74) in float32, one IEEE operation per torch call."""
    import torch
    v = torch.from_numpy(tris).cuda().view(-1, 3, 3)
    p0, p1, p2 = v[:, 0], v[:, 1], v[:, 2]
    e1, e2 = p0 - p1, p2 - p0

    def cross(a, b):
        return torch.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                            a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], dim=-1)

    def dot(a, b):
        return ((0 + a[..., 0] * b[..., 0]) + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]

    nrm = cross(e1, e2)
    eps = -np.finfo(np.float32).eps
    ids = np.full(rays.shape[0], 0xFFFFFFFF, np.uint32)
    ts = np.full(rays.shape[0], np.inf, np.float32)
    prim = torch.arange(v.shape[0], device="cuda", dtype=torch.int64)
    for s in range(0, rays.shape[0], chunk):
        r = torch.from_numpy(rays[s:s + chunk]).cuda()
        org, d = r[:, None, 0:3], r[:, None, 3:6]
        c = p0[None] - org
        rr = cross(d.expand_as(c), c)
        inv_det = 1 / dot(nrm[None], d)
        u = dot(rr, e2[None]) * inv_det
        w_v = dot(rr, e1[None]) * inv_det
        w = (1 - u) - w_v
        t = dot(nrm[None], c) * inv_det
        ok = (u >= eps) & (w_v >= eps) & (w >= eps) & (t >= r[:, None, 6]) & (t <= r[:, None, 7])
        ok &= prim[None] != torch.from_numpy(origins[s:s + chunk].astype(np.int64)).cuda()[:, None]
        tm = torch.where(ok, t, torch.full_like(t, np.inf))
        best = tm.min(dim=1).values
        cand = ok & (tm == best[:, None])
        first = torch.where(cand, prim[None].expand_as(tm), torch.full_like(tm, 2 ** 40, dtype=torch.int64)).min(dim=1).values
        hit = cand.any(dim=1)
        ids[s:s + chunk] = np.where(host(hit), host(first), 0xFFFFFFFF).astype(np.uint32)
        ts[s:s + chunk] = host(best)
    return ids, ts


def test_secondary_rays_skip_origin(dtt, gpu_lib):
    """Rays spawned at the soup's primary hits with tmin = 0 and the hit triangle as origin: with the origin filter (robust
    box test), a 10k-ray sample equals a brute force that skips the origin; without it, a noticeable fraction of them hits
    its own triangle again."""
    tris = scenes.make_mesh("soup", 1_000_000)
    primary = scenes.make_primary("soup", 1000, 1000)
    bvh = gpu_lib.Bvh.build_triangles(tris)
    hits = bvh.intersect_rays(primary)
    keep = hits["prim_id"] != 0xFFFFFFFF
    rng = np.random.default_rng(5)
    sel = np.nonzero(keep)[0]
    sel = sel[rng.permutation(sel.shape[0])[:200_000]]
    org = primary[sel, 0:3] + hits["t"][sel, None] * primary[sel, 3:6]
    d = rng.normal(size=(sel.shape[0], 3)).astype(np.float32)
    rays = np.zeros((sel.shape[0], 8), np.float32)
    rays[:, 0:3], rays[:, 3:6], rays[:, 6], rays[:, 7] = org, d, 0.0, np.inf
    origins = hits["prim_id"][sel].astype(np.uint32)
    run, d_rays, n = Run(dtt, bvh, np.float32), cuda(rays), rays.shape[0]
    d_origins = cuda(origins)
    ids, t, _, _, _, _ = run(d_rays, n, NOT_ORIGIN, ROBUST, origins=d_origins)
    plain = run(d_rays, n, ALL, ROBUST)[0].view(np.uint32)
    self_hits = (plain == origins).mean()
    assert self_hits > 0.01, f"only {self_hits:.4f} of the secondary rays hit their origin: the test would prove nothing"
    assert not (ids.view(np.uint32) == origins).any()
    sample = rng.permutation(n)[:10_000]
    bf_ids, bf_t = brute_force_closest(tris, rays[sample], origins[sample])
    assert (ids.view(np.uint32)[sample] == bf_ids).all(), np.nonzero(ids.view(np.uint32)[sample] != bf_ids)[0][:8]
    hit = bf_ids != 0xFFFFFFFF
    assert (t[sample][hit] == bf_t[hit]).all()
    assert hit.mean() > 0.1
    bvh.destroy()


def test_camera_rays_in_kernel(dtt, gpu_lib):
    """A camera shader computes ray i from i and writes only t: equal to the t of bvh3f_intersect_rays on the rays a
    separate kernel writes with the same generator."""
    import torch
    tris = scenes.make_mesh("soup", 1_000_000)
    bvh = gpu_lib.Bvh.build_triangles(tris)
    lo, hi = tris.reshape(-1, 3).min(axis=0), tris.reshape(-1, 3).max(axis=0)
    cam = np.array([(lo[0] + hi[0]) / 2, (lo[1] + hi[1]) / 2, lo[2] - 1.0, lo[0] - 0.5, hi[0] + 0.5, lo[1] - 0.5, hi[1] + 0.5],
                   np.float32)
    w, h = 1500, 1100
    n = w * h
    depth = torch.empty(n, dtype=torch.float32, device="cuda")
    ws = torch.empty(8, dtype=torch.uint8, device="cuda")
    rays = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    check(dtt, dtt.dtt_camera3f(C.c_void_p(bvh.handle), cam.ctypes.data, w, h, ptr(depth), ptr(ws), 8, None))
    check(dtt, dtt.dtt_camera_rays3f(cam.ctypes.data, w, h, ptr(rays), None))
    torch.cuda.synchronize()
    want = bvh.intersect_rays(host(rays))
    got = host(depth)
    assert (bits(got) == bits(np.ascontiguousarray(want["t"]))).all()
    assert np.isfinite(got).mean() > 0.1
    bvh.destroy()


def test_every_ray_once(dtt, gpu_lib):
    """finish is called once per ray for batch sizes around the scheduler's edges; nothing past n is written; n = 0
    launches nothing."""
    import torch
    tris = scenes.make_mesh("soup", 100_000)
    rays = scenes.make_primary("soup", 1001, 1001)
    bvh = gpu_lib.Bvh.build_triangles(tris)
    run = Run(dtt, bvh, np.float32)
    props = torch.cuda.get_device_properties(0)
    wave = props.multi_processor_count * 9 * 4 * 32           # one resident wave of warps (9 blocks of 4 warps per SM), in rays
    big = 1_000_007
    d_rays = cuda(np.resize(rays, (max(wave + 1, big), 8)))
    guard = 1000
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 4097, wave - 1, wave, wave + 1, big):
        counts = torch.zeros(n + guard, dtype=torch.int32, device="cuda")
        run(d_rays, n, ALL, 0, counts=counts)
        got = host(counts)
        assert (got[:n] == 1).all(), (n, np.nonzero(got[:n] != 1)[0][:8])
        assert (got[n:] == 0).all(), n
    bvh.destroy()


def test_errors_leave_tree_usable(dtt, gpu_lib):
    """A view without triangles (build_boxes) raises invalid_argument, a short workspace length_error; neither launches
    anything, and the tree traces as before afterwards."""
    import torch
    api = gpu_lib
    tris = scenes.make_mesh("soup", 100_000)
    rays = scenes.make_primary("soup", 300, 300)
    bvh = api.Bvh.build_triangles(tris)
    run, d_rays, n = Run(dtt, bvh, np.float32), cuda(rays), rays.shape[0]
    assert dtt.dtt_workspace_bytes3f(C.c_void_p(bvh.handle)) == 8
    first = run(d_rays, n, ALL, 0)
    counts = torch.zeros(n, dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="workspace of 7 bytes is too small"):
        run(d_rays, n, ALL, 0, counts=counts, ws_bytes=7)
    centres = tris.reshape(-1, 3, 3).mean(axis=1).astype(np.float32)
    boxes = np.concatenate([tris.reshape(-1, 3, 3).min(axis=1), tris.reshape(-1, 3, 3).max(axis=1)], axis=1).astype(np.float32)
    d_boxes, d_centres = cuda(boxes), cuda(centres)
    torch.cuda.synchronize()
    box_bvh = api.Bvh.build_boxes(d_boxes.data_ptr(), d_centres.data_ptr(), count=centres.shape[0], dtype=np.float32,
                                  flags=api.DEVICE_POINTERS)
    with pytest.raises(TypeError, match="no triangles"):
        Run(dtt, box_bvh, np.float32)(d_rays, n, ALL, 0, counts=counts)
    box_bvh.destroy()
    torch.cuda.synchronize()
    assert (host(counts) == 0).all()
    second = run(d_rays, n, ALL, 0)
    for a, b in zip(first, second):
        assert (bits(a) == bits(b)).all() if a.dtype.kind == "f" else (a == b).all()
    bvh.destroy()


def test_build_trace_refit_trace_on_one_stream(dtt, gpu_lib):
    """build_triangles, trace_triangles, refit_triangles with moved vertices, trace_triangles again: one torch stream, no
    synchronisation between the steps.  Both results equal the same steps run synchronously."""
    import torch
    api = gpu_lib
    tris = scenes.make_mesh("soup", 200_000)
    moved = (tris + 0.01 * (np.random.default_rng(4).random(tris.shape) - 0.5)).astype(np.float32)
    rays = scenes.make_primary("soup", 700, 700)
    d_rays = cuda(rays)
    torch.cuda.synchronize()

    def frames(sync):
        stream = torch.cuda.Stream()
        api.set_stream(stream.cuda_stream)
        out = []
        try:
            with torch.cuda.stream(stream):
                d_tris, d_moved = cuda(tris), cuda(moved)
                bvh = api.Bvh.build_triangles(d_tris.data_ptr(), count=tris.shape[0], dtype=np.float32, flags=api.DEVICE_POINTERS)
                run = Run(dtt, bvh, np.float32)
                for frame in range(2):
                    if frame:
                        bvh.refit_triangles(d_moved.data_ptr(), api.DEVICE_POINTERS)
                        if sync:
                            stream.synchronize()
                    res = run(d_rays, rays.shape[0], ALL, 0, stream=C.c_void_p(stream.cuda_stream), sync=False)
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
    assert (fast[0][1] != fast[1][1]).any(), "moving the triangles changed no hit"
