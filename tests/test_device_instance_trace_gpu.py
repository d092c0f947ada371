"""DeviceView::trace_instances and prepare_instances on the GPU (test shaders in tests/device_instance_trace_kernels.cu):
one identity instance bit for bit equal to trace_triangles under every flag and both tie rules, many transformed
instances equal to one thread per ray nesting DeviceView::intersect by hand, closest hits equal to a float64 brute force
over the world-space triangles, the boxes and inverses of prepare_instances, every ray finished once, the errors, and a
rigid animation on one torch stream."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes

pytestmark = pytest.mark.gpu

P, SZ, U = C.c_void_p, C.c_size_t, C.c_uint
ANY, ROBUST, LAST = 1, 2, 4
MODES = [m | t for t in (0, LAST) for m in (0, ROBUST, ANY, ANY | ROBUST)]
MODE_IDS = [f"{m}-{t}" for t in ("lowest", "last") for m in ("closest", "robust", "any", "any-robust")]
NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def dit(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_instance_trace_tests())
    for s in ("3f", "3d"):
        getattr(L, f"dit_records{s}").argtypes = [P, P, P, SZ, P, C.POINTER(SZ), P]
        getattr(L, f"dit_set_matrices{s}").argtypes = [P, P, SZ, P]
        getattr(L, f"dit_prepare{s}").argtypes = [P, SZ, SZ, P, P, P]
        getattr(L, f"dit_run{s}").argtypes = [P, P, SZ, SZ, C.c_int, C.c_int, U, P, SZ] + [P] * 8 + [P, SZ, P]
        getattr(L, f"dit_triangles{s}").argtypes = [P, U, P, SZ] + [P] * 7 + [P, SZ, P]
        getattr(L, f"dit_record_bytes{s}").restype = SZ
    L.dit_plain3f.argtypes = [P, P, SZ, SZ, P, SZ, P, P, P, SZ, P]
    L.dit_plain_triangles3f.argtypes = [P, P, SZ, P, P, SZ, P]
    L.dit_nested_trace3f.argtypes = [P, P, SZ, P, SZ, P, P, P, SZ, P]
    L.dit_last_error.restype = C.c_char_p
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


def check(dit, rc):
    if rc:
        msg = dit.dit_last_error().decode()
        raise {-2: ValueError, -3: TypeError}.get(rc, RuntimeError)(msg)


def rotations(rng, k):
    """k random rotation matrices (QR of Gaussian matrices, determinant +1)"""
    q, r = np.linalg.qr(rng.normal(size=(k, 3, 3)))
    q = q * np.sign(np.diagonal(r, axis1=1, axis2=2))[:, None, :]
    q[np.linalg.det(q) < 0, :, 0] *= -1
    return q


def placements(count, seed=3, spacing=1.5, singular=()):
    """count 3 x 4 matrices: copies of a unit-cube mesh on a square grid of cells `spacing` apart, each rotated about the
    cube's centre and scaled by 0.6 .. 1.2; the indices in `singular` get a matrix that flattens y."""
    rng = np.random.default_rng(seed)
    side = int(np.ceil(np.sqrt(count)))
    a = rotations(rng, count) * rng.uniform(0.6, 1.2, size=(count, 1, 1))
    for k in singular:
        a[k] = np.diag([1.0, 0.0, 1.0])
    k = np.arange(count)
    cell = np.stack([(k % side) * spacing, (k // side) * spacing, np.zeros(count)], axis=1)
    c = np.full(3, 0.5)
    b = cell + c - a @ c
    return np.concatenate([a, b[:, :, None]], axis=2).reshape(count, 12)


def world_rays(mats, w, h, dtype, seed=9):
    """w x h rays in pixel order from below the placed copies (z = -3), almost along +z, over their cells"""
    t = mats.reshape(-1, 3, 4)[:, :, 3]
    lo, hi = t.min(axis=0) - 1.0, t.max(axis=0) + 1.0
    px, py = np.meshgrid((np.arange(w) + 0.5) / w, (np.arange(h) + 0.5) / h)
    rays = np.zeros((w * h, 8))
    rays[:, 0] = lo[0] + px.ravel() * (hi[0] - lo[0])
    rays[:, 1] = lo[1] + py.ravel() * (hi[1] - lo[1])
    rays[:, 2] = -3.0
    rng = np.random.default_rng(seed)
    rays[:, 3:5] = rng.uniform(-0.05, 0.05, size=(w * h, 2))
    rays[:, 5] = 1.0
    rays[:, 7] = np.inf
    return rays.astype(dtype)


def special_rays(tris, dtype):
    from tests.test_device_api_host import extra_rays
    return extra_rays(tris, dtype)


class Scene:
    """Bottom meshes, instance records in device memory, prepare_instances' boxes and a top tree built from them."""

    def __init__(self, dit, api, meshes, mesh_of, mats, dtype, stream=None):
        import torch
        self.dit, self.api = dit, api
        self.s = "3f" if np.dtype(dtype) == np.float32 else "3d"
        self.dtype = np.dtype(dtype)
        self.tdtype = torch.float32 if self.s == "3f" else torch.float64
        self.meshes = [m if isinstance(m, api.Bvh) else api.Bvh.build_triangles(np.ascontiguousarray(m, dtype)) for m in meshes]
        self.own = [not isinstance(m, api.Bvh) for m in meshes]
        self.count = len(mesh_of)
        self.rec_bytes = getattr(dit, f"dit_record_bytes{self.s}")()
        self.records = torch.zeros(self.count * self.rec_bytes, dtype=torch.uint8, device="cuda")
        handles = (C.c_void_p * len(self.meshes))(*[m.handle for m in self.meshes])
        mesh_of = np.ascontiguousarray(mesh_of, np.uint32)
        mats = np.ascontiguousarray(mats, dtype)
        depth = SZ(0)
        torch.cuda.synchronize()
        check(dit, getattr(dit, f"dit_records{self.s}")(handles, mesh_of.ctypes.data, mats.ctypes.data, self.count, ptr(self.records),
                                                        C.byref(depth), stream))
        self.max_depth = depth.value
        self.boxes = torch.empty((self.count, 6), dtype=self.tdtype, device="cuda")
        self.centres = torch.empty((self.count, 3), dtype=self.tdtype, device="cuda")
        self.prepare(stream)
        torch.cuda.synchronize()
        self.top = api.Bvh.build_boxes(self.boxes.data_ptr(), self.centres.data_ptr(), count=self.count, dtype=self.dtype,
                                       flags=api.DEVICE_POINTERS)
        self.ws = torch.empty(64, dtype=torch.uint8, device="cuda")

    def prepare(self, stream=None):
        check(self.dit, getattr(self.dit, f"dit_prepare{self.s}")(ptr(self.records), self.count, self.max_depth, ptr(self.boxes),
                                                                  ptr(self.centres), stream))

    def world_to_object(self):
        """(count, 12) world_to_object of every record, float64"""
        raw = host(self.records).reshape(self.count, self.rec_bytes)
        off = 32 if self.s == "3f" else 40
        size = self.dtype.itemsize
        m = raw[:, off + 12 * size: off + 24 * size].copy().view(self.dtype)
        return m.astype(np.float64)

    def run(self, d_rays, n, filt, flags, per_thread=False, counts=None, ws_bytes=None, count=None, max_depth=None,
            stream=None, sync=True):
        import torch
        ids = torch.empty(n, dtype=torch.int32, device="cuda")
        t, u, v = (torch.empty(n, dtype=self.tdtype, device="cuda") for _ in range(3))
        inst, calls = (torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2))
        hashes = torch.empty(n, dtype=torch.int64, device="cuda")
        check(self.dit, getattr(self.dit, f"dit_run{self.s}")(
            C.c_void_p(self.top.handle), ptr(self.records), self.count if count is None else count,
            self.max_depth if max_depth is None else max_depth, int(per_thread), filt, flags, ptr(d_rays), n, ptr(ids), ptr(t),
            ptr(u), ptr(v), ptr(inst), ptr(calls), ptr(hashes), ptr(counts), ptr(self.ws),
            self.ws.numel() if ws_bytes is None else ws_bytes, stream))
        out = (ids, t, u, v, inst, calls, hashes)
        if not sync:
            return out
        torch.cuda.synchronize()
        return tuple(host(x) for x in out)

    def destroy(self):
        self.top.destroy()
        for m, own in zip(self.meshes, self.own):
            if own:
                m.destroy()


def assert_same(got, want, what=""):
    names = ("ids", "t", "u", "v", "inst", "calls", "hashes")
    for name, a, b in zip(names, got, want):
        same = bits(a) == bits(b) if a.dtype.kind == "f" else a == b
        assert same.all(), f"{what} {name} differs at {np.nonzero(~same)[0][:8]}"


IDENTITY = np.array([[1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]], np.float64)
SCENES = [("soup", 1_000_000, 1000, np.float32), ("grid", 1_000_000, 1000, np.float32), ("soup", 100_000, 700, np.float64)]


@pytest.fixture(scope="module", params=SCENES, ids=["c2-soup", "c2-grid", "c5"])
def identity_scene(request, dit, gpu_lib):
    kind, n, img, dtype = request.param
    tris = scenes.make_mesh(kind, n, dtype=dtype)
    rays = np.concatenate([scenes.make_primary(kind, img, img, dtype=dtype), special_rays(tris, dtype)])
    scene = Scene(dit, gpu_lib, [tris], [0], IDENTITY, dtype)
    yield scene, rays, cuda(rays)
    scene.destroy()


@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
def test_identity_instance_equals_trace_triangles(dit, identity_scene, flags):
    """One instance with the identity matrix: records, instance, accept-call counts and accept-sequence hashes equal
    trace_triangles on the mesh, bit for bit."""
    import torch
    scene, rays, d_rays = identity_scene
    n = rays.shape[0]
    got = scene.run(d_rays, n, 0, flags)
    outs = [torch.empty(n, dtype=dt, device="cuda") for dt in (torch.int32, scene.tdtype, scene.tdtype, scene.tdtype, torch.int32,
                                                               torch.int32, torch.int64)]
    check(dit, getattr(dit, f"dit_triangles{scene.s}")(C.c_void_p(scene.meshes[0].handle), flags, ptr(d_rays), n,
                                                       *[ptr(x) for x in outs], ptr(scene.ws), scene.ws.numel(), None))
    torch.cuda.synchronize()
    want = tuple(host(x) for x in outs)
    assert_same(got, want, "identity")
    assert (got[0] != -1).sum() > n // 10
    assert ((got[4] == 0) == (got[0] != -1)).all()


def many_scene(dit, api, dtype, count=60, singular=()):
    meshes = [scenes.make_mesh("soup", 20_000, dtype=dtype), scenes.make_mesh("grid", 20_000, dtype=dtype)]
    mats = placements(count, singular=singular)
    mesh_of = np.arange(count) % 2
    return Scene(dit, api, meshes, mesh_of, mats, dtype), meshes, mesh_of, mats


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
def test_many_instances_equal_nested_intersect(dit, gpu_lib, dtype, flags):
    """60 rotated and scaled copies of two meshes: per ray the record, instance, accept-call count and accept-sequence
    hash equal one thread per ray nesting DeviceView::intersect by hand, with every candidate accepted and with odd
    instances rejected."""
    scene, meshes, _, mats = many_scene(dit, gpu_lib, dtype)
    rays = np.concatenate([world_rays(mats, 500, 500, dtype), special_rays(meshes[0], dtype)])
    d_rays, n = cuda(rays), rays.shape[0]
    for filt in (0, 1):
        got = scene.run(d_rays, n, filt, flags)
        want = scene.run(d_rays, n, filt, flags, per_thread=True)
        assert_same(got, want, f"filter {filt}")
        assert (got[0] != -1).sum() > n // 10
        if filt == 1:
            assert ((got[4][got[0] != -1] & 1) == 0).all()
        else:
            assert len(np.unique(got[4][got[0] != -1])) > 30
    scene.destroy()


def world_triangles(meshes, mesh_of, mats):
    """(count * tris, 3, 3) float64 world-space vertices, instance-major"""
    out = []
    for k, m in enumerate(mats.reshape(-1, 3, 4)):
        v = meshes[mesh_of[k]].reshape(-1, 3, 3).astype(np.float64)
        out.append(v @ m[:, :3].T + m[:, 3])
    return np.concatenate(out)


def test_closest_equals_float64_brute_force(dit, gpu_lib):
    """Closest (instance, id) of 4000 sampled rays equal a float64 brute force over the world-space triangles, except
    rays whose two best float64 distances differ by less than 1e-4 relative or whose hit lies within 1e-4 of a
    triangle's edge (where float32 rounding may decide)."""
    import torch
    count = 24
    meshes = [scenes.make_mesh("soup", 5_000), scenes.make_mesh("grid", 5_000)]
    mats = placements(count, seed=11)
    mesh_of = np.arange(count) % 2
    scene = Scene(dit, gpu_lib, meshes, mesh_of, mats, np.float32)
    rays = world_rays(mats, 300, 300, np.float32)
    sample = np.random.default_rng(2).permutation(rays.shape[0])[:4000]
    ids, t, _, _, inst, _, _ = scene.run(cuda(rays[sample]), sample.shape[0], 0, 0)
    tris = torch.from_numpy(world_triangles(meshes, mesh_of, mats)).cuda()
    per = meshes[0].shape[0]
    p0, e1, e2 = tris[:, 0], tris[:, 1] - tris[:, 0], tris[:, 2] - tris[:, 0]
    checked = 0
    for s in range(0, sample.shape[0], 50):
        r = torch.from_numpy(rays[sample[s:s + 50]].astype(np.float64)).cuda()
        o, d = r[:, None, 0:3], r[:, None, 3:6]
        pv = torch.cross(d.expand(-1, p0.shape[0], -1), e2[None].expand(d.shape[0], -1, -1), dim=-1)
        det = (e1[None] * pv).sum(-1)
        tv = o - p0[None]
        a = (tv * pv).sum(-1) / det
        qv = torch.cross(tv, e1[None].expand_as(tv), dim=-1)
        b = (d * qv).sum(-1) / det
        tt = (e2[None] * qv).sum(-1) / det
        edge = torch.minimum(torch.minimum(a, b), 1 - a - b)
        ok = (edge >= 0) & (tt >= 0)
        near = (edge.abs() < 1e-4) & (tt >= 0)
        tm = torch.where(ok, tt, torch.full_like(tt, np.inf))
        two = torch.topk(tm, 2, dim=1, largest=False)
        best, second, arg = two.values[:, 0], two.values[:, 1], two.indices[:, 0]
        for j in range(r.shape[0]):
            i = s + j
            bt, st = float(best[j]), float(second[j])
            close = np.isfinite(bt) and (st - bt) <= 1e-4 * max(abs(bt), 1.0)
            reach = bt + 1e-3 * max(abs(bt), 1.0) if np.isfinite(bt) else np.inf
            hit_near = bool((near[j] & (tt[j] <= reach)).any())          # an edge in front of the hit: float32 may decide
            if close or hit_near:
                continue
            checked += 1
            if not np.isfinite(bt):
                assert ids[i] == -1, i
            else:
                k = int(arg[j])
                assert (int(inst[i]), int(ids[i])) == (k // per, k % per), (i, bt, float(t[i]))
                assert abs(float(t[i]) - bt) <= 1e-4 * max(abs(bt), 1.0)
    assert checked > 3000
    assert (ids != -1).mean() > 0.2
    scene.destroy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
def test_prepare_instances(dit, gpu_lib, dtype):
    """Every world box contains every transformed vertex (float64); world_to_object is within 1e-5 (float) / 1e-13
    (double) of numpy.linalg.inv relative to the matrix's size; singular matrices get an empty box, a NaN inverse and no
    hits, even in a leaf they share, and an instance alone at a singular matrix gets none either."""
    count = 40
    singular = (3, 17)
    scene, meshes, mesh_of, mats = many_scene(dit, gpu_lib, dtype, count=count, singular=singular)
    boxes = host(scene.boxes).astype(np.float64)
    verts = world_triangles(meshes, mesh_of, mats).reshape(count, -1, 3)
    w2o = scene.world_to_object()
    tol = 1e-5 if dtype == np.float32 else 1e-13
    for k in range(count):
        if k in singular:
            assert (boxes[k, :3] == np.inf).all() and (boxes[k, 3:] == -np.inf).all()
            assert np.isnan(w2o[k]).all()
            continue
        lo, hi = verts[k].min(axis=0), verts[k].max(axis=0)
        assert (boxes[k, :3] <= lo).all() and (boxes[k, 3:] >= hi).all(), k
        assert (hi - lo > 0.3 * (boxes[k, 3:] - boxes[k, :3])).all()      # not needlessly large
        m = np.vstack([mats[k].reshape(3, 4), [0, 0, 0, 1]])
        want = np.linalg.inv(m)[:3].ravel()
        assert np.abs(w2o[k] - want).max() <= tol * max(1.0, np.abs(want).max()), k
    rays = world_rays(mats, 400, 400, dtype)
    d_rays, n = cuda(rays), rays.shape[0]
    for flags in (0, ANY):
        got = scene.run(d_rays, n, 0, flags)
        assert (got[0] != -1).sum() > n // 10
        assert not np.isin(got[4], singular).any()
        assert_same(got, scene.run(d_rays, n, 0, flags, per_thread=True))
    scene.destroy()
    alone = Scene(dit, gpu_lib, [meshes[0]], [0], placements(1, singular=(0,)), dtype)
    got = alone.run(d_rays, n, 0, 0)
    assert (got[0] == -1).all() and (got[5] == 0).all() and (got[4] == -1).all()
    alone.destroy()


def test_every_ray_once(dit, gpu_lib):
    """finish is called once per ray at batch sizes around the scheduler's edges and at 1M rays; nothing past n is
    written; n = 0 launches nothing."""
    import torch
    scene, _, _, mats = many_scene(dit, gpu_lib, np.float32, count=16)
    props = torch.cuda.get_device_properties(0)
    wave = props.multi_processor_count * 9 * 4 * 32
    big = 1_000_007
    rays = world_rays(mats, 1001, 1001, np.float32)
    d_rays = cuda(np.resize(rays, (max(wave + 1, big), 8)))
    guard = 1000
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 4097, wave - 1, wave, wave + 1, big):
        counts = torch.zeros(n + guard, dtype=torch.int32, device="cuda")
        scene.run(d_rays, n, 0, 0, counts=counts)
        got = host(counts)
        assert (got[:n] == 1).all(), (n, np.nonzero(got[:n] != 1)[0][:8])
        assert (got[n:] == 0).all(), n
    scene.destroy()


def test_errors_leave_trees_usable(dit, gpu_lib):
    """A record count other than the top tree's raises invalid_argument; a short workspace and a bottom depth that
    overflows the 200 KB stack raise length_error; none launches anything, and the trees trace as before afterwards."""
    import torch
    scene, _, _, mats = many_scene(dit, gpu_lib, np.float32, count=20)
    rays = world_rays(mats, 300, 300, np.float32)
    d_rays, n = cuda(rays), rays.shape[0]
    first = scene.run(d_rays, n, 0, 0)
    counts = torch.zeros(n, dtype=torch.int32, device="cuda")
    with pytest.raises(TypeError, match="19 instance records for a top tree of 20"):
        scene.run(d_rays, n, 0, 0, counts=counts, count=19)
    with pytest.raises(ValueError, match="workspace of 7 bytes is too small"):
        scene.run(d_rays, n, 0, 0, counts=counts, ws_bytes=7)
    with pytest.raises(ValueError, match="shared-memory stack"):
        scene.run(d_rays, n, 0, 0, counts=counts, max_depth=400)
    torch.cuda.synchronize()
    assert (host(counts) == 0).all()
    assert_same(scene.run(d_rays, n, 0, 0), first, "after the errors")
    scene.destroy()


def test_rigid_animation_on_one_stream(dit, gpu_lib):
    """Four frames on one torch stream, with no synchronisation between the steps: new matrices written on the device,
    prepare_instances, refit_boxes of the top tree, trace_instances.  Each frame equals the per-thread reference run
    on that frame's records afterwards, and the motion changes the hits."""
    import torch
    api = gpu_lib
    count = 30
    meshes = [scenes.make_mesh("soup", 20_000), scenes.make_mesh("grid", 20_000)]
    mesh_of = np.arange(count) % 2
    frames = [placements(count, seed=20 + f) for f in range(4)]
    rays = world_rays(frames[0], 400, 400, np.float32)
    d_rays, n = cuda(rays), rays.shape[0]
    scene = Scene(dit, api, meshes, mesh_of, frames[0], np.float32)
    stream = torch.cuda.Stream()
    api.set_stream(stream.cuda_stream)
    got = []
    try:
        top = api.Bvh.build_boxes(scene.boxes.data_ptr(), scene.centres.data_ptr(), count=count, dtype=np.float32,
                                  flags=api.DEVICE_POINTERS)
        scene.top.destroy()
        scene.top = top
        s = C.c_void_p(stream.cuda_stream)
        with torch.cuda.stream(stream):
            d_frames = [cuda(f.astype(np.float32)) for f in frames]
            for f in range(4):
                check(dit, dit.dit_set_matrices3f(ptr(scene.records), ptr(d_frames[f]), count, s))
                scene.prepare(s)
                top.refit_boxes(scene.boxes.data_ptr(), api.DEVICE_POINTERS)
                out = scene.run(d_rays, n, 0, 0, stream=s, sync=False)
                got.append(tuple(x.clone() for x in out))
        stream.synchronize()
        got = [tuple(host(x) for x in f) for f in got]
        for f in range(4):
            check(dit, dit.dit_set_matrices3f(ptr(scene.records), ptr(d_frames[f]), count, s))
            scene.prepare(s)
            top.refit_boxes(scene.boxes.data_ptr(), api.DEVICE_POINTERS)
            stream.synchronize()
            want = scene.run(d_rays, n, 0, 0, per_thread=True, stream=s)
            assert_same(got[f], want, f"frame {f}")
    finally:
        api.set_stream(None)
    assert all((got[f][0] != -1).sum() > n // 10 for f in range(4))
    assert (got[0][1] != got[1][1]).any()
    scene.destroy()
