"""The motion forms of DeviceView::trace_instances and trace_instance_paths, prepare_motion_instances and instance_at on
the GPU (test shaders in tests/device_motion_instance_kernels.cu; the static calls they are compared with in
tests/device_instance_trace_kernels.cu and tests/device_instance_path_trace_kernels.cu): with equal keys the static
calls bit for bit at random times; at one time the static call over static records set to the placement at that time,
on the same top tree; at random times one thread per ray calling instance_at and nesting DeviceView::intersect by hand;
closest hits against a float64 brute force over the moved vertices; one path-tracing launch against its wavefront loop;
every ray and path finished once; the errors; and four animated frames on one torch stream."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes
from tests.test_device_instance_trace_gpu import assert_same, dit, placements, special_rays, world_rays  # noqa: F401
from tests.test_device_instance_path_trace_gpu import dipt  # noqa: F401

pytestmark = pytest.mark.gpu

P, SZ, U, U32 = C.c_void_p, C.c_size_t, C.c_uint, C.c_uint32
ANY, ROBUST, LAST = 1, 2, 4
MODES = [m | t for t in (0, LAST) for m in (0, ROBUST, ANY, ANY | ROBUST)]
MODE_IDS = [f"{m}-{t}" for t in ("lowest", "last") for m in ("closest", "robust", "any", "any-robust")]
PATH_FLAGS = [0, ROBUST, LAST, ROBUST | LAST]
PATH_IDS = ["fast-lowest", "robust-lowest", "fast-last", "robust-last"]
TRACER_NAMES = ("radiance", "segments", "hashes")


@pytest.fixture(scope="module")
def dmi(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_motion_instance_tests())
    for s in ("3f", "3d"):
        real = C.c_float if s == "3f" else C.c_double
        getattr(L, f"dmi_records{s}").argtypes = [P, P, P, P, SZ, P, C.POINTER(SZ), P]
        getattr(L, f"dmi_set_keys{s}").argtypes = [P, P, P, SZ, P]
        getattr(L, f"dmi_static_at{s}").argtypes = [P, SZ, real, P, P]
        getattr(L, f"dmi_placement{s}").argtypes = [P, P, SZ, P, P]
        getattr(L, f"dmi_prepare{s}").argtypes = [P, SZ, SZ, P, P, P]
        getattr(L, f"dmi_run{s}").argtypes = [P, P, SZ, SZ, C.c_int, C.c_int, U, P, P, SZ] + [P] * 8 + [P, SZ, P]
        getattr(L, f"dmi_tracer{s}").argtypes = [P, P, SZ, SZ, C.c_int, U, SZ, P, P, P, P, U32, P, P, P, P, P, P, SZ, P]
        getattr(L, f"dmi_wavefront_bytes{s}").argtypes = [SZ]
        getattr(L, f"dmi_wavefront_bytes{s}").restype = SZ
        getattr(L, f"dmi_record_bytes{s}").restype = SZ
    L.dmi_last_error.restype = C.c_char_p
    return L


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def assert_fields(got, want, names, what=""):
    for name, a, b in zip(names, got, want):
        same = a.view(np.uint32 if a.dtype.itemsize == 4 else np.uint64) == b.view(np.uint32 if b.dtype.itemsize == 4 else np.uint64)
        assert same.all(), f"{what} {name} differs at {np.nonzero(~same)[0][:8]}"


def check(lib, rc, prefix="dmi"):
    if rc:
        msg = getattr(lib, f"{prefix}_last_error")().decode()
        raise {-2: ValueError, -3: TypeError}.get(rc, RuntimeError)(msg)


def moving_keys(count, seed=3, spacing=1.5, singular=()):
    """(key0, key1): placements() at time 0, and each copy moved by up to one cell width and turned by up to 30 degrees
    about the cube's centre at time 1.  The copies in `singular` mirror y over the shutter, so that their placement
    has no inverse at time 0.5."""
    rng = np.random.default_rng(seed + 100)
    key0 = placements(count, seed=seed, spacing=spacing).reshape(count, 3, 4)
    key1 = key0.copy()
    axis = rng.normal(size=(count, 3))
    axis /= np.linalg.norm(axis, axis=1, keepdims=True)
    angle = rng.uniform(-np.pi / 6, np.pi / 6, size=count)
    c = np.full(3, 0.5)
    for k in range(count):
        x, y, z = axis[k]
        kx = np.array([[0, -z, y], [z, 0, -x], [-y, x, 0]])
        turn = np.eye(3) + np.sin(angle[k]) * kx + (1 - np.cos(angle[k])) * kx @ kx
        a = turn @ key0[k, :, :3]
        centre = key0[k, :, :3] @ c + key0[k, :, 3]
        shift = rng.uniform(-1.0, 1.0, size=3) * np.array([spacing, spacing, 0.25])
        key1[k, :, :3] = a
        key1[k, :, 3] = centre + shift - a @ c
    for k in singular:
        key0[k, :, :3] = np.eye(3)
        key1[k, :, :3] = np.diag([1.0, -1.0, 1.0])
        key0[k, :, 3] = key1[k, :, 3] = [(k % 8) * spacing, (k // 8) * spacing, 0.0]
        key1[k, 1, 3] += 1.0                                    # (y mirrored about the cube's centre)
    return key0.reshape(count, 12), key1.reshape(count, 12)


class MotionScene:
    """Bottom meshes, motion records in device memory, prepare_motion_instances' boxes and a top tree built from them."""

    def __init__(self, dmi, api, meshes, mesh_of, keys0, keys1, dtype):
        import torch
        self.dmi, self.api = dmi, api
        self.s = "3f" if np.dtype(dtype) == np.float32 else "3d"
        self.dtype = np.dtype(dtype)
        self.tdtype = torch.float32 if self.s == "3f" else torch.float64
        self.meshes = [m if isinstance(m, api.Bvh) else api.Bvh.build_triangles(np.ascontiguousarray(m, dtype)) for m in meshes]
        self.tris = [None if isinstance(m, api.Bvh) else np.ascontiguousarray(m, dtype) for m in meshes]
        self.mesh_of = list(mesh_of)
        self.count = len(mesh_of)
        self.rec_bytes = getattr(dmi, f"dmi_record_bytes{self.s}")()
        self.records = torch.zeros(self.count * self.rec_bytes, dtype=torch.uint8, device="cuda")
        handles = (C.c_void_p * len(self.meshes))(*[m.handle for m in self.meshes])
        mesh_of = np.ascontiguousarray(mesh_of, np.uint32)
        k0, k1 = np.ascontiguousarray(keys0, dtype), np.ascontiguousarray(keys1, dtype)
        depth = SZ(0)
        torch.cuda.synchronize()
        check(dmi, getattr(dmi, f"dmi_records{self.s}")(handles, mesh_of.ctypes.data, k0.ctypes.data, k1.ctypes.data, self.count,
                                                        ptr(self.records), C.byref(depth), None))
        self.max_depth = depth.value
        self.boxes = torch.empty((self.count, 6), dtype=self.tdtype, device="cuda")
        self.centres = torch.empty((self.count, 3), dtype=self.tdtype, device="cuda")
        self.prepare()
        torch.cuda.synchronize()
        self.top = api.Bvh.build_boxes(self.boxes.data_ptr(), self.centres.data_ptr(), count=self.count, dtype=self.dtype,
                                       flags=api.DEVICE_POINTERS)
        self.ws = torch.empty(64, dtype=torch.uint8, device="cuda")

    def prepare(self, stream=None):
        check(self.dmi, getattr(self.dmi, f"dmi_prepare{self.s}")(ptr(self.records), self.count, self.max_depth, ptr(self.boxes),
                                                                  ptr(self.centres), stream))

    def run(self, d_rays, d_times, n, filt, flags, per_thread=False, counts=None, ws_bytes=None, count=None, max_depth=None,
            stream=None, sync=True):
        import torch
        ids = torch.empty(n, dtype=torch.int32, device="cuda")
        t, u, v = (torch.empty(n, dtype=self.tdtype, device="cuda") for _ in range(3))
        inst, calls = (torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2))
        hashes = torch.empty(n, dtype=torch.int64, device="cuda")
        check(self.dmi, getattr(self.dmi, f"dmi_run{self.s}")(
            C.c_void_p(self.top.handle), ptr(self.records), self.count if count is None else count,
            self.max_depth if max_depth is None else max_depth, int(per_thread), filt, flags, ptr(d_rays), ptr(d_times), n, ptr(ids),
            ptr(t), ptr(u), ptr(v), ptr(inst), ptr(calls), ptr(hashes), ptr(counts), ptr(self.ws),
            self.ws.numel() if ws_bytes is None else ws_bytes, stream))
        out = (ids, t, u, v, inst, calls, hashes)
        if not sync:
            return out
        torch.cuda.synchronize()
        return tuple(host(x) for x in out)

    def placement(self, times):
        """(count, 2, 12) float64: instance_at(records[k], times[k])'s object_to_world and world_to_object"""
        import torch
        d_times = cuda(np.asarray(times, self.dtype))
        out = torch.empty((self.count, 24), dtype=self.tdtype, device="cuda")
        check(self.dmi, getattr(self.dmi, f"dmi_placement{self.s}")(ptr(self.records), ptr(d_times), self.count, ptr(out), None))
        torch.cuda.synchronize()
        return host(out).astype(np.float64).reshape(self.count, 2, 12)

    def destroy(self):
        self.top.destroy()
        for m in self.meshes:
            m.destroy()


class StaticAt:
    """Static records set to instance_at(records[k], tau), prepared by prepare_instances, traced through
    trace_instances (dit_run) and trace_instance_paths (dipt_tracer) on the motion scene's own top tree."""

    def __init__(self, dit, scene, tau):
        import torch
        self.dit, self.scene = dit, scene
        self.rec_bytes = getattr(dit, f"dit_record_bytes{scene.s}")()
        self.records = torch.zeros(scene.count * self.rec_bytes, dtype=torch.uint8, device="cuda")
        check(scene.dmi, getattr(scene.dmi, f"dmi_static_at{scene.s}")(ptr(scene.records), scene.count, tau, ptr(self.records), None))
        boxes = torch.empty((scene.count, 6), dtype=scene.tdtype, device="cuda")
        centres = torch.empty((scene.count, 3), dtype=scene.tdtype, device="cuda")
        check(dit, getattr(dit, f"dit_prepare{scene.s}")(ptr(self.records), scene.count, scene.max_depth, ptr(boxes), ptr(centres),
                                                         None), "dit")
        torch.cuda.synchronize()

    def run(self, d_rays, n, filt, flags):
        import torch
        sc = self.scene
        outs = [torch.empty(n, dtype=dt, device="cuda") for dt in (torch.int32, sc.tdtype, sc.tdtype, sc.tdtype, torch.int32,
                                                                   torch.int32, torch.int64)]
        check(self.dit, getattr(self.dit, f"dit_run{sc.s}")(
            C.c_void_p(sc.top.handle), ptr(self.records), sc.count, sc.max_depth, 0, filt, flags, ptr(d_rays), n, *[ptr(x) for x in outs],
            None, ptr(sc.ws), sc.ws.numel(), None), "dit")
        torch.cuda.synchronize()
        return tuple(host(x) for x in outs)


class Tracer:
    """The path tracer over a motion scene (dmi_tracer) and, for equal keys, over static records (dipt_tracer)."""

    def __init__(self, scene, primary, times, light, bounces):
        import torch
        self.scene, self.bounces = scene, bounces
        self.primary, self.times = cuda(primary), cuda(np.asarray(times, scene.dtype))
        self.n = primary.shape[0]
        self.light = np.asarray(light, scene.dtype)
        self.d_verts = [cuda(t.reshape(-1)) for t in scene.tris]
        self.verts = torch.tensor([self.d_verts[k].data_ptr() for k in scene.mesh_of], dtype=torch.int64, device="cuda")
        self.scratch = torch.empty(getattr(scene.dmi, f"dmi_wavefront_bytes{scene.s}")(self.n), dtype=torch.uint8, device="cuda")
        self.ws = torch.empty(8, dtype=torch.uint8, device="cuda")

    def outputs(self):
        import torch
        return (torch.full((self.n,), float("nan"), dtype=self.scene.tdtype, device="cuda"),
                torch.full((self.n,), -1, dtype=torch.int32, device="cuda"), torch.zeros(self.n, dtype=torch.int32, device="cuda"))

    def __call__(self, mode, flags, counts=None, n=None, ws_bytes=8, count=None, max_depth=None):
        import torch
        sc = self.scene
        out = self.outputs()
        check(sc.dmi, getattr(sc.dmi, f"dmi_tracer{sc.s}")(
            C.c_void_p(sc.top.handle), ptr(sc.records), sc.count if count is None else count,
            sc.max_depth if max_depth is None else max_depth, mode, flags, self.n if n is None else n, ptr(self.primary),
            ptr(self.times), self.light.ctypes.data, ptr(self.verts), self.bounces, *[ptr(x) for x in out], ptr(counts),
            ptr(self.scratch), ptr(self.ws), ws_bytes, None))
        torch.cuda.synchronize()
        return tuple(host(x) for x in out)

    def static(self, dipt, static_at, flags):
        import torch
        sc = self.scene
        out = self.outputs()
        check(dipt, getattr(dipt, f"dipt_tracer{sc.s}")(
            C.c_void_p(sc.top.handle), ptr(static_at.records), sc.count, sc.max_depth, 0, flags, self.n, ptr(self.primary),
            self.light.ctypes.data, ptr(self.verts), self.bounces, *[ptr(x) for x in out], None, ptr(self.ws), 8, None), "dipt")
        torch.cuda.synchronize()
        return tuple(host(x) for x in out)


def random_times(n, seed=5, dtype=np.float32):
    return np.random.default_rng(seed).uniform(0.0, 1.0, size=n).astype(dtype)


EQUAL_SCENES = [("soup", 1_000_000, 700, np.float32), ("grid", 1_000_000, 700, np.float32), ("soup", 200_000, 400, np.float64)]


@pytest.fixture(scope="module", params=EQUAL_SCENES, ids=["c2-soup-3f", "c2-grid-3f", "soup-3d"])
def equal_scene(request, dmi, dit, gpu_lib):
    """Four overlapping copies of one c2 mesh whose two keys are equal, the static records at their placement, primary
    rays with random times and a path tracer over them."""
    kind, n, img, dtype = request.param
    tris = scenes.make_mesh(kind, n, dtype=dtype)
    keys = placements(4, seed=7, spacing=0.6)
    scene = MotionScene(dmi, gpu_lib, [tris], [0] * 4, keys, keys, dtype)
    static = StaticAt(dit, scene, 0.25)
    rays = np.concatenate([world_rays(keys, img, img, dtype), special_rays(tris, dtype)])
    times = random_times(rays.shape[0], dtype=dtype)
    centre = keys.reshape(-1, 3, 4)[:, :, 3].mean(axis=0)
    tracer = Tracer(scene, world_rays(keys, img // 2, img // 2, dtype), random_times((img // 2) ** 2, 6, dtype),
                    centre + np.array([0.3, -0.2, -4.0]), 4)
    yield scene, static, rays, cuda(rays), cuda(times), tracer
    scene.destroy()


@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
def test_equal_keys_equal_trace_instances(dit, equal_scene, flags):
    """Equal keys: at random per-ray times, records, instances, accept-call counts and accept-sequence hashes equal
    trace_instances over the static records on the same top tree, bit for bit."""
    scene, static, rays, d_rays, d_times, _ = equal_scene
    n = rays.shape[0]
    for filt in (0, 1):
        got = scene.run(d_rays, d_times, n, filt, flags)
        assert_same(got, static.run(d_rays, n, filt, flags), f"equal keys, filter {filt}")
        assert (got[0] != -1).sum() > n // 20


@pytest.mark.parametrize("flags", PATH_FLAGS, ids=PATH_IDS)
def test_equal_keys_equal_trace_instance_paths(dipt, equal_scene, flags):
    """Equal keys: a path tracer with shadow segments, one time per path, equals trace_instance_paths over the static
    records on the same top tree, bit for bit."""
    scene, static, _, _, _, tracer = equal_scene
    got = tracer(0, flags)
    assert_fields(got, tracer.static(dipt, static, flags), TRACER_NAMES, "equal keys paths")
    rad, segs, _ = got
    assert (segs >= 1).all() and segs.max() >= 4 and np.isfinite(rad).all()


def moving_scene(dmi, api, dtype, count=60, singular=(7,), seed=3):
    meshes = [scenes.make_mesh("soup", 20_000, dtype=dtype), scenes.make_mesh("grid", 20_000, dtype=dtype)]
    keys0, keys1 = moving_keys(count, seed=seed, singular=singular)
    mesh_of = np.arange(count) % 2
    return MotionScene(dmi, api, meshes, mesh_of, keys0, keys1, dtype), keys0, keys1


def scene_rays(keys0, keys1, w, h, dtype):
    return world_rays(np.concatenate([keys0, keys1]), w, h, dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
def test_one_time_equals_static_records(dmi, dit, gpu_lib, dtype):
    """60 moving copies, one of them mirrored over the shutter (no inverse at 0.5): all rays at one time tau equal
    trace_instances over static records set to instance_at(records[k], tau) and prepared by prepare_instances, on the
    same top tree, bit for bit, under every flag."""
    scene, keys0, keys1 = moving_scene(dmi, gpu_lib, dtype)
    rays = np.concatenate([scene_rays(keys0, keys1, 400, 400, dtype), special_rays(scene.tris[0], dtype)])
    d_rays, n = cuda(rays), rays.shape[0]
    hits = {}
    for tau in (0.0, 0.37, 0.5, 1.0):
        d_times = cuda(np.full(n, tau, dtype))
        static = StaticAt(dit, scene, tau)
        for flags in MODES:
            got = scene.run(d_rays, d_times, n, 0, flags)
            assert_same(got, static.run(d_rays, n, 0, flags), f"tau {tau} flags {flags}")
        hits[tau] = got
        assert (got[0] != -1).sum() > n // 10
        if tau == 0.5:
            assert not (hits[tau][4] == 7).any()
        else:
            assert (hits[tau][4] == 7).any()
    assert (hits[0.0][1] != hits[1.0][1]).any()
    scene.destroy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
def test_random_times_equal_nested_instance_at(dmi, gpu_lib, dtype, flags):
    """60 moving copies, random per-ray times: per ray the record, instance, accept-call count and accept-sequence hash
    equal one thread per ray that builds instance_at on each entry and nests DeviceView::intersect by hand, with every
    candidate accepted and with odd instances rejected."""
    scene, keys0, keys1 = moving_scene(dmi, gpu_lib, dtype)
    rays = np.concatenate([scene_rays(keys0, keys1, 400, 400, dtype), special_rays(scene.tris[0], dtype)])
    d_rays, n = cuda(rays), rays.shape[0]
    times = random_times(n, dtype=dtype)
    times[::97] = np.array([np.nan, -1.0, 2.0, 0.0, 1.0], dtype)[np.arange(times[::97].shape[0]) % 5]
    d_times = cuda(times)
    for filt in (0, 1):
        got = scene.run(d_rays, d_times, n, filt, flags)
        assert_same(got, scene.run(d_rays, d_times, n, filt, flags, per_thread=True), f"filter {filt}")
        assert (got[0] != -1).sum() > n // 10
        if filt == 1:
            assert ((got[4][got[0] != -1] & 1) == 0).all()
    scene.destroy()


def test_closest_equals_float64_brute_force(dmi, gpu_lib):
    """Closest (instance, id) of 4000 sampled rays at eight times equal a float64 brute force over the vertices moved by
    each record's rounded placement at the ray's time, except rays whose two best float64 distances differ by less than
    1e-4 relative or whose hit lies within 1e-4 of a triangle's edge (where float32 rounding may decide)."""
    import torch
    count = 24
    meshes = [scenes.make_mesh("soup", 5_000), scenes.make_mesh("grid", 5_000)]
    keys0, keys1 = moving_keys(count, seed=11)
    mesh_of = np.arange(count) % 2
    scene = MotionScene(dmi, gpu_lib, meshes, mesh_of, keys0, keys1, np.float32)
    rays = scene_rays(keys0, keys1, 300, 300, np.float32)
    rng = np.random.default_rng(2)
    sample = rng.permutation(rays.shape[0])[:4000]
    palette = rng.uniform(0, 1, size=8).astype(np.float32)
    which = np.arange(sample.shape[0]) % 8
    ids, t, _, _, inst, _, _ = scene.run(cuda(rays[sample]), cuda(palette[which]), sample.shape[0], 0, 0)
    per = meshes[0].shape[0]
    checked = 0
    for w in range(8):
        a = scene.placement(np.full(count, palette[w]))[:, 0].reshape(count, 3, 4)
        world = np.concatenate([meshes[mesh_of[k]].reshape(-1, 3, 3).astype(np.float64) @ a[k, :, :3].T + a[k, :, 3] for k in range(count)])
        tris = torch.from_numpy(world).cuda()
        p0, e1, e2 = tris[:, 0], tris[:, 1] - tris[:, 0], tris[:, 2] - tris[:, 0]
        rows = np.nonzero(which == w)[0]
        for s in range(0, rows.shape[0], 50):
            chunk = rows[s:s + 50]
            r = torch.from_numpy(rays[sample[chunk]].astype(np.float64)).cuda()
            o, d = r[:, None, 0:3], r[:, None, 3:6]
            pv = torch.cross(d.expand(-1, p0.shape[0], -1), e2[None].expand(d.shape[0], -1, -1), dim=-1)
            det = (e1[None] * pv).sum(-1)
            tv = o - p0[None]
            u = (tv * pv).sum(-1) / det
            qv = torch.cross(tv, e1[None].expand_as(tv), dim=-1)
            v = (d * qv).sum(-1) / det
            tt = (e2[None] * qv).sum(-1) / det
            edge = torch.minimum(torch.minimum(u, v), 1 - u - v)
            ok = (edge >= 0) & (tt >= 0)
            near = (edge.abs() < 1e-4) & (tt >= 0)
            tm = torch.where(ok, tt, torch.full_like(tt, np.inf))
            two = torch.topk(tm, 2, dim=1, largest=False)
            best, second, arg = two.values[:, 0], two.values[:, 1], two.indices[:, 0]
            for j, i in enumerate(chunk):
                bt, st = float(best[j]), float(second[j])
                close = np.isfinite(bt) and (st - bt) <= 1e-4 * max(abs(bt), 1.0)
                reach = bt + 1e-3 * max(abs(bt), 1.0) if np.isfinite(bt) else np.inf
                if close or bool((near[j] & (tt[j] <= reach)).any()):
                    continue
                checked += 1
                if not np.isfinite(bt):
                    assert ids[i] == -1, i
                else:
                    k = int(arg[j])
                    assert (int(inst[i]), int(ids[i])) == (k // per, k % per), (i, bt, float(t[i]))
                    assert abs(float(t[i]) - bt) <= 1e-4 * max(abs(bt), 1.0)
    assert checked > 3000
    assert (ids != -1).mean() > 0.1
    scene.destroy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
def test_prepare_motion_instances(dmi, gpu_lib, dtype):
    """instance_at is each key at 0 and 1, bit for bit; every box holds every vertex moved in float64 by the rounded
    placement at 65 times; a key with a NaN gives the empty box and no hits."""
    count = 12
    keys0, keys1 = moving_keys(count, seed=4, singular=(5,))
    keys1[9, 2] = np.nan
    meshes = [scenes.make_mesh("soup", 4_000, dtype=dtype), scenes.make_mesh("grid", 4_000, dtype=dtype)]
    mesh_of = np.arange(count) % 2
    scene = MotionScene(dmi, gpu_lib, meshes, mesh_of, keys0, keys1, dtype)
    boxes = host(scene.boxes).astype(np.float64)
    k0, k1 = keys0.astype(dtype).astype(np.float64), keys1.astype(dtype).astype(np.float64)
    at0, at1 = scene.placement(np.zeros(count))[:, 0], scene.placement(np.ones(count))[:, 0]
    assert (at0 == k0).all() and np.array_equal(at1, k1, equal_nan=True)
    assert (boxes[9, :3] == np.inf).all() and (boxes[9, 3:] == -np.inf).all()
    for tau in np.arange(65) / 64:
        a = scene.placement(np.full(count, tau))[:, 0].reshape(count, 3, 4)
        for k in range(count):
            if k == 9:
                continue
            v = meshes[mesh_of[k]].reshape(-1, 3).astype(np.float64) @ a[k, :, :3].T + a[k, :, 3]
            assert (boxes[k, :3] <= v.min(axis=0)).all() and (boxes[k, 3:] >= v.max(axis=0)).all(), (k, tau)
    rays = scene_rays(keys0[:9], keys1[:9], 200, 200, dtype)
    got = scene.run(cuda(rays), cuda(random_times(rays.shape[0], dtype=dtype)), rays.shape[0], 0, 0)
    assert (got[0] != -1).sum() > 0 and not (got[4] == 9).any()
    scene.destroy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
@pytest.mark.parametrize("flags", PATH_FLAGS, ids=PATH_IDS)
def test_one_launch_equals_wavefront_loop(dmi, gpu_lib, dtype, flags):
    """60 moving copies, one mirrored over the shutter: a path tracer with shadow segments and one random time per path
    gives the same radiance bits, segment counts and segment hashes in one trace_instance_paths call as in a wavefront
    loop of motion trace_instances launches."""
    scene, keys0, keys1 = moving_scene(dmi, gpu_lib, dtype)
    primary = scene_rays(keys0, keys1, 300, 300, dtype)
    centre = keys0.reshape(-1, 3, 4)[:, :, 3].mean(axis=0)
    tracer = Tracer(scene, primary, random_times(primary.shape[0], 8, dtype), centre + np.array([0.3, -0.2, -4.0]), 4)
    got = tracer(0, flags)
    assert_fields(got, tracer(1, flags), TRACER_NAMES, "one launch vs wavefront")
    rad, segs, _ = got
    assert (segs >= 1).all() and segs.max() >= 4 and (segs > 1).mean() > 0.1
    assert np.isfinite(rad).all()
    scene.destroy()


def test_every_ray_and_path_once(dmi, gpu_lib):
    """finish is called once per ray and once per path at batch sizes around the scheduler's edges and at 1M; nothing
    past n is written; n = 0 launches nothing."""
    import torch
    scene, keys0, keys1 = moving_scene(dmi, gpu_lib, np.float32, count=16, singular=())
    props = torch.cuda.get_device_properties(0)
    wave = props.multi_processor_count * 9 * 4 * 32
    big = 1_000_007
    rays = np.resize(scene_rays(keys0, keys1, 1001, 1001, np.float32), (max(wave + 1, big), 8))
    d_rays, d_times = cuda(rays), cuda(random_times(rays.shape[0]))
    centre = keys0.reshape(-1, 3, 4)[:, :, 3].mean(axis=0)
    tracer = Tracer(scene, rays, random_times(rays.shape[0], 9), centre + np.array([0.3, -0.2, -4.0]), 1)
    guard = 1000
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 4097, wave - 1, wave, wave + 1, big):
        for what in ("rays", "paths"):
            counts = torch.zeros(n + guard, dtype=torch.int32, device="cuda")
            if what == "rays":
                scene.run(d_rays, d_times, n, 0, 0, counts=counts)
            else:
                tracer(0, 0, counts=counts, n=n)
            got = host(counts)
            assert (got[:n] == 1).all(), (what, n, np.nonzero(got[:n] != 1)[0][:8])
            assert (got[n:] == 0).all(), (what, n)
    scene.destroy()


def test_errors_leave_trees_usable(dmi, gpu_lib):
    """A record count other than the top tree's raises invalid_argument, a short workspace and a bottom depth that
    overflows the 200 KB stack raise length_error, each naming the motion call; none launches anything, and the trees
    trace as before afterwards."""
    import torch
    scene, keys0, keys1 = moving_scene(dmi, gpu_lib, np.float32, count=20, singular=())
    rays = scene_rays(keys0, keys1, 300, 300, np.float32)
    d_rays, n = cuda(rays), rays.shape[0]
    d_times = cuda(random_times(n))
    first = scene.run(d_rays, d_times, n, 0, 0)
    counts = torch.zeros(n, dtype=torch.int32, device="cuda")
    with pytest.raises(TypeError, match=r"trace_instances \(motion\): 19 instance records for a top tree of 20"):
        scene.run(d_rays, d_times, n, 0, 0, counts=counts, count=19)
    with pytest.raises(ValueError, match=r"trace_instances \(motion\): a workspace of 7 bytes is too small"):
        scene.run(d_rays, d_times, n, 0, 0, counts=counts, ws_bytes=7)
    with pytest.raises(ValueError, match="shared-memory stack"):
        scene.run(d_rays, d_times, n, 0, 0, counts=counts, max_depth=400)
    centre = keys0.reshape(-1, 3, 4)[:, :, 3].mean(axis=0)
    tracer = Tracer(scene, rays, random_times(n, 3), centre + np.array([0.3, -0.2, -4.0]), 2)
    paths = tracer(0, 0)
    with pytest.raises(TypeError, match=r"trace_instance_paths \(motion\): 19 instance records"):
        tracer(0, 0, counts=counts, count=19)
    with pytest.raises(ValueError, match=r"trace_instance_paths \(motion\): a workspace of 7 bytes"):
        tracer(0, 0, counts=counts, ws_bytes=7)
    with pytest.raises(ValueError, match="shared-memory stack"):
        tracer(0, 0, counts=counts, max_depth=400)
    torch.cuda.synchronize()
    assert (host(counts) == 0).all()
    assert_same(scene.run(d_rays, d_times, n, 0, 0), first, "after the errors")
    assert_fields(tracer(0, 0), paths, TRACER_NAMES, "paths after the errors")
    scene.destroy()


def test_motion_animation_on_one_stream(dmi, gpu_lib):
    """Four frames on one torch stream, with no synchronisation between the steps: both keys rewritten on the device,
    prepare_motion_instances, refit_boxes of the top tree, the motion trace_instances.  Each frame equals the per-thread
    reference run on that frame's records afterwards, and the motion changes the hits."""
    import torch
    api = gpu_lib
    count = 30
    meshes = [scenes.make_mesh("soup", 20_000), scenes.make_mesh("grid", 20_000)]
    mesh_of = np.arange(count) % 2
    frames = [moving_keys(count, seed=20 + f, singular=()) for f in range(5)]
    rays = scene_rays(*frames[0], 400, 400, np.float32)
    d_rays, n = cuda(rays), rays.shape[0]
    d_times = cuda(random_times(n))
    scene = MotionScene(dmi, api, meshes, mesh_of, frames[0][0], frames[0][1], np.float32)
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
            # frame f moves from frame f's first key to frame f + 1's first key
            d_keys = [(cuda(frames[f][0].astype(np.float32)), cuda(frames[f + 1][0].astype(np.float32))) for f in range(4)]
            for f in range(4):
                check(dmi, dmi.dmi_set_keys3f(ptr(scene.records), ptr(d_keys[f][0]), ptr(d_keys[f][1]), count, s))
                scene.prepare(s)
                top.refit_boxes(scene.boxes.data_ptr(), api.DEVICE_POINTERS)
                out = scene.run(d_rays, d_times, n, 0, 0, stream=s, sync=False)
                got.append(tuple(x.clone() for x in out))
        stream.synchronize()
        got = [tuple(host(x) for x in f) for f in got]
        for f in range(4):
            check(dmi, dmi.dmi_set_keys3f(ptr(scene.records), ptr(d_keys[f][0]), ptr(d_keys[f][1]), count, s))
            scene.prepare(s)
            top.refit_boxes(scene.boxes.data_ptr(), api.DEVICE_POINTERS)
            stream.synchronize()
            want = scene.run(d_rays, d_times, n, 0, 0, per_thread=True, stream=s)
            assert_same(got[f], want, f"frame {f}")
    finally:
        api.set_stream(None)
    assert all((got[f][0] != -1).sum() > n // 10 for f in range(4))
    assert (got[0][1] != got[1][1]).any()
    scene.destroy()
