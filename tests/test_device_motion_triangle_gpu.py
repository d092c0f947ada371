"""The motion forms of DeviceView::trace_triangles and trace_paths, prepare_motion_triangles and triangle_at on the GPU
(test shaders in tests/device_motion_triangle_kernels.cu): with equal keys the static calls bit for bit at random times;
at one time the static trace_triangles after set_triangles with the vertices at that time, on the same tree; at random
times one thread per ray nesting DeviceView::intersect with a triangle_at leaf; closest hits against a float64 brute
force over the blended vertices; one path-tracing launch against its wavefront loop; every ray and path finished once;
the errors; and four animation frames on one torch stream against a fresh build per frame."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes
from tests.test_device_triangle_trace_gpu import special_rays

pytestmark = pytest.mark.gpu

P, SZ, U, U32 = C.c_void_p, C.c_size_t, C.c_uint, C.c_uint32
ANY, ROBUST, LAST = 1, 2, 4
MODES = [m | t for t in (0, LAST) for m in (0, ROBUST, ANY, ANY | ROBUST)]
MODE_IDS = [f"{m}-{t}" for t in ("lowest", "last") for m in ("closest", "robust", "any", "any-robust")]
PATH_FLAGS = [0, ROBUST, LAST, ROBUST | LAST]
PATH_IDS = ["fast-lowest", "robust-lowest", "fast-last", "robust-last"]
MOTION, STATIC, PER_THREAD = 0, 1, 2
TRACER_NAMES = ("radiance", "segments", "hashes")
RUN_NAMES = ("ids", "t", "u", "v", "calls", "hashes")


@pytest.fixture(scope="module")
def dmt(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_motion_triangle_tests())
    for s in ("3f", "3d"):
        real = C.c_float if s == "3f" else C.c_double
        getattr(L, f"dmt_prepare{s}").argtypes = [P, P, SZ, P, P, P]
        getattr(L, f"dmt_triangle_at{s}").argtypes = [P, P, SZ, real, P, P]
        getattr(L, f"dmt_run{s}").argtypes = [P, P, P, SZ, C.c_int, C.c_int, U, P, P, SZ] + [P] * 7 + [P, SZ, P]
        getattr(L, f"dmt_tracer{s}").argtypes = [P, P, P, SZ, C.c_int, U, SZ, P, P, P, U32, P, P, P, P, P, P, SZ, P]
        getattr(L, f"dmt_wavefront_bytes{s}").argtypes = [SZ]
        getattr(L, f"dmt_wavefront_bytes{s}").restype = SZ
    L.dmt_plain3f.argtypes = [P, P, P, SZ, C.c_int, P, P, SZ, P, P, SZ, P]
    L.dmt_steps3f.argtypes = [P, P, P, SZ, C.c_int, P, P, SZ, P, P, P]
    L.dmt_last_error.restype = C.c_char_p
    return L


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def check(lib, rc):
    if rc:
        msg = lib.dmt_last_error().decode()
        raise {-2: ValueError, -3: TypeError}.get(rc, RuntimeError)(msg)


def assert_fields(got, want, names, what=""):
    for name, a, b in zip(names, got, want):
        same = a.view(np.uint32 if a.dtype.itemsize == 4 else np.uint64) == b.view(np.uint32 if b.dtype.itemsize == 4 else np.uint64)
        assert same.all(), f"{what} {name} differs at {np.nonzero(~same)[0][:8]}"


def deform(tris, phase, amp):
    """The mesh's vertices moved by a smooth field of amplitude `amp` (shared vertices move together)"""
    p = tris.reshape(-1, 3).astype(np.float64)
    d = amp * np.sin(7.0 * p[:, [1, 2, 0]] + phase + np.array([0.0, 1.3, 2.6]))
    return np.ascontiguousarray((p + d).reshape(tris.shape).astype(tris.dtype))


def tri_size(tris):
    """The median of the triangles' longest edges"""
    v = tris.reshape(-1, 3, 3).astype(np.float64)
    edges = np.stack([np.linalg.norm(v[:, a] - v[:, b], axis=1) for a, b in ((0, 1), (1, 2), (2, 0))], axis=1)
    return float(np.median(edges.max(axis=1)))


def moving_keys(tris, seed=0):
    return tris, deform(tris, seed, tri_size(tris))


def blend(k0, k1, tau, dtype):
    """triangle_at in numpy: the time clamped to [0, 1] (NaN as 0), then the same four rounded steps in `dtype`, exact at
    the keys and where they agree"""
    k0, k1 = k0.astype(dtype), k1.astype(dtype)
    tau = dtype(tau)
    if not tau > 0:                                             # (NaN too)
        return k0.copy()
    if tau >= 1:
        return k1.copy()
    rest = dtype(1) - tau
    mixed = (rest * k0).astype(dtype) + (tau * k1).astype(dtype)
    return np.where(k0 == k1, k0, mixed.astype(dtype))


def random_times(n, seed=5, dtype=np.float32):
    return np.random.default_rng(seed).uniform(0.0, 1.0, size=n).astype(dtype)


def rounding_times(n, seed, dtype):
    """Random times whose mantissa is full, so that 1 - tau rounds (in double too, unlike k / 2^53): the times at which
    the blend's rounding can leave the interval between its keys"""
    return (np.random.default_rng(seed).uniform(0.0, 1.0, size=n) / 1.0009765625).astype(dtype)


def ulps_keys(tris, seed):
    """Both keys at 1e4 from the mesh, each coordinate of key 1 one to three ulps from key 0's, either way"""
    rng = np.random.default_rng(seed)
    k0 = (tris.astype(np.float64) + 1e4).astype(tris.dtype)
    k1 = k0.copy()
    up = np.where(rng.random(k0.shape) < 0.5, np.inf, -np.inf).astype(tris.dtype)
    steps = rng.integers(1, 4, size=k0.shape)
    for q in range(3):
        k1 = np.where(steps > q, np.nextafter(k1, up), k1)
    return k0, k1


class Scene:
    """Two device keys, prepare_motion_triangles' boxes and a tree built from them (no triangles attached unless
    attach() is called).  `same` passes key 0's pointer twice."""

    def __init__(self, dmt, api, key0, key1, same=False, stream=None):
        import torch
        self.dmt, self.api = dmt, api
        self.dtype = key0.dtype
        self.s = "3f" if self.dtype == np.float32 else "3d"
        self.tdtype = torch.float32 if self.s == "3f" else torch.float64
        self.count = key0.shape[0]
        self.k0 = cuda(key0.reshape(-1))
        self.k1 = self.k0 if same else cuda(key1.reshape(-1))
        self.boxes = torch.empty((self.count, 6), dtype=self.tdtype, device="cuda")
        self.centres = torch.empty((self.count, 3), dtype=self.tdtype, device="cuda")
        self.prepare(stream)
        torch.cuda.synchronize()
        self.bvh = api.Bvh.build_boxes(self.boxes.data_ptr(), self.centres.data_ptr(), count=self.count, dtype=self.dtype,
                                       flags=api.DEVICE_POINTERS)
        self.ws = torch.empty(64, dtype=torch.uint8, device="cuda")

    def prepare(self, stream=None):
        check(self.dmt, getattr(self.dmt, f"dmt_prepare{self.s}")(ptr(self.k0), ptr(self.k1), self.count, ptr(self.boxes),
                                                                  ptr(self.centres), stream))

    def attach(self, vertices):
        """set_triangles: the static calls' triangles (host array or device tensor, original order)"""
        import torch
        if isinstance(vertices, np.ndarray):
            self.bvh.set_triangles(np.ascontiguousarray(vertices, self.dtype))
        else:
            torch.cuda.synchronize()
            self.bvh.set_triangles(vertices.data_ptr(), self.api.DEVICE_POINTERS)

    def triangle_at(self, tau):
        import torch
        out = torch.empty(self.count * 9, dtype=self.tdtype, device="cuda")
        check(self.dmt, getattr(self.dmt, f"dmt_triangle_at{self.s}")(ptr(self.k0), ptr(self.k1), self.count, tau, ptr(out), None))
        torch.cuda.synchronize()
        return host(out).reshape(self.count, 9)

    def run(self, mode, d_rays, d_times, n, filt, flags, counts=None, ws_bytes=None, count=None, k1=True, stream=None, sync=True):
        import torch
        ids = torch.empty(n, dtype=torch.int32, device="cuda")
        t, u, v = (torch.empty(n, dtype=self.tdtype, device="cuda") for _ in range(3))
        calls = torch.empty(n, dtype=torch.int32, device="cuda")
        hashes = torch.empty(n, dtype=torch.int64, device="cuda")
        check(self.dmt, getattr(self.dmt, f"dmt_run{self.s}")(
            C.c_void_p(self.bvh.handle), ptr(self.k0), ptr(self.k1) if k1 else None, self.count if count is None else count, mode,
            filt, flags, ptr(d_rays), ptr(d_times), n, ptr(ids), ptr(t), ptr(u), ptr(v), ptr(calls), ptr(hashes), ptr(counts),
            ptr(self.ws), self.ws.numel() if ws_bytes is None else ws_bytes, stream))
        out = (ids, t, u, v, calls, hashes)
        if not sync:
            return out
        torch.cuda.synchronize()
        return tuple(host(x) for x in out)

    def destroy(self):
        self.bvh.destroy()


class Tracer:
    """The path tracer over a scene: one motion trace_paths call (mode 0), the wavefront loop (1), static trace_paths (2)"""

    def __init__(self, scene, primary, times, light, bounces):
        import torch
        self.scene, self.bounces = scene, bounces
        self.primary, self.times = cuda(primary), cuda(np.asarray(times, scene.dtype))
        self.n = primary.shape[0]
        self.light = np.asarray(light, scene.dtype)
        self.scratch = torch.empty(getattr(scene.dmt, f"dmt_wavefront_bytes{scene.s}")(self.n), dtype=torch.uint8, device="cuda")
        self.ws = torch.empty(8, dtype=torch.uint8, device="cuda")

    def __call__(self, mode, flags, counts=None, n=None, ws_bytes=8, count=None):
        import torch
        sc = self.scene
        out = (torch.full((self.n,), float("nan"), dtype=sc.tdtype, device="cuda"),
               torch.full((self.n,), -1, dtype=torch.int32, device="cuda"), torch.zeros(self.n, dtype=torch.int32, device="cuda"))
        check(sc.dmt, getattr(sc.dmt, f"dmt_tracer{sc.s}")(
            C.c_void_p(sc.bvh.handle), ptr(sc.k0), ptr(sc.k1), sc.count if count is None else count, mode, flags,
            self.n if n is None else n, ptr(self.primary), ptr(self.times), self.light.ctypes.data, self.bounces, *[ptr(x) for x in out],
            ptr(counts), ptr(self.scratch), ptr(self.ws), ws_bytes, None))
        torch.cuda.synchronize()
        return tuple(host(x) for x in out)


LIGHT = {"soup": (0.8, 1.6, -0.4), "grid": (0.3, 1.2, 0.6)}
EQUAL_SCENES = [("soup", 1_000_000, 1000, np.float32), ("grid", 1_000_000, 1000, np.float32), ("soup", 200_000, 500, np.float64)]


@pytest.fixture(scope="module", params=EQUAL_SCENES, ids=["c2-soup-3f", "c2-grid-3f", "soup-3d"])
def equal_scene(request, dmt, gpu_lib):
    """A c2 mesh passed as both keys (one pointer), its tree from prepare_motion_triangles' boxes with the key attached
    by set_triangles, primary rays with random times and a path tracer over it."""
    kind, n, img, dtype = request.param
    tris = scenes.make_mesh(kind, n, dtype=dtype)
    scene = Scene(dmt, gpu_lib, tris, tris, same=True)
    scene.attach(scene.k0)
    rays = np.concatenate([scenes.make_primary(kind, img, img, dtype=dtype), special_rays(tris, dtype)])
    times = random_times(rays.shape[0], dtype=dtype)
    tracer = Tracer(scene, scenes.make_primary(kind, img // 2, img // 2, dtype=dtype), random_times((img // 2) ** 2, 6, dtype),
                    LIGHT[kind], 4)
    yield scene, rays, cuda(rays), cuda(times), tracer
    scene.destroy()


@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
def test_equal_keys_equal_trace_triangles(equal_scene, flags):
    """Equal keys: at random per-ray times, records, accept-call counts and accept-sequence hashes equal trace_triangles
    on the same handle after set_triangles(key 0), bit for bit."""
    scene, rays, d_rays, d_times, _ = equal_scene
    n = rays.shape[0]
    for filt in (0, 1):
        got = scene.run(MOTION, d_rays, d_times, n, filt, flags)
        assert_fields(got, scene.run(STATIC, d_rays, d_times, n, filt, flags), RUN_NAMES, f"equal keys, filter {filt}")
        assert (got[0] != -1).sum() > n // 20


@pytest.mark.parametrize("flags", PATH_FLAGS, ids=PATH_IDS)
def test_equal_keys_equal_trace_paths(equal_scene, flags):
    """Equal keys: a path tracer with shadow segments, one random time per path, equals trace_paths bit for bit."""
    scene, _, _, _, tracer = equal_scene
    got = tracer(0, flags)
    assert_fields(got, tracer(2, flags), TRACER_NAMES, "equal keys paths")
    rad, segs, _ = got
    assert (segs >= 1).all() and segs.max() >= 4 and np.isfinite(rad).all()


@pytest.mark.parametrize("kind,dtype", [("soup", np.float32), ("grid", np.float32), ("soup", np.float64)],
                         ids=["soup-3f", "grid-3f", "soup-3d"])
def test_one_time_equals_static_triangles(dmt, gpu_lib, kind, dtype):
    """Moving keys, every ray at one time tau: triangle_at equals the numpy blend bit for bit, and the motion call equals
    trace_triangles after set_triangles with the vertices at tau, on the same tree, bit for bit (accept sequences
    included), under every flag."""
    tris = scenes.make_mesh(kind, 200_000, dtype=dtype)
    k0, k1 = moving_keys(tris, seed=1)
    scene = Scene(dmt, gpu_lib, k0, k1)
    rays = np.concatenate([scenes.make_primary(kind, 500, 500, dtype=dtype), special_rays(tris, dtype)])
    d_rays, n = cuda(rays), rays.shape[0]
    first = {}
    ui = np.uint32 if dtype == np.float32 else np.uint64
    for x in (-1.0, 2.0, float("nan"), -0.0, 1e-30, *rounding_times(6, 9, np.float64)):         # the clamp, NaN, random times
        assert (blend(k0, k1, x, np.dtype(dtype).type).view(ui) == scene.triangle_at(x).view(ui)).all(), x
    for tau in (0.0, 0.37, 0.5, 1.0):
        at = blend(k0, k1, tau, np.dtype(dtype).type)
        assert (at.view(ui) == scene.triangle_at(tau).view(ui)).all(), tau
        scene.attach(at)
        d_times = cuda(np.full(n, tau, dtype))
        for flags in MODES:
            for filt in (0, 1) if flags in (0, ANY) else (0,):
                got = scene.run(MOTION, d_rays, d_times, n, filt, flags)
                assert_fields(got, scene.run(STATIC, d_rays, d_times, n, filt, flags), RUN_NAMES, f"tau {tau} flags {flags} filter {filt}")
                if flags == 0 and filt == 0:
                    first[tau] = got
        assert (first[tau][0] != -1).sum() > n // 10
    assert (first[0.0][1] != first[1.0][1]).any()
    scene.destroy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
def test_random_times_equal_nested_triangle_at(dmt, gpu_lib, dtype, flags):
    """Moving keys, random per-ray times (with NaN, -1, 2, 0 and 1 among them): per ray the record, accept-call count and
    accept-sequence hash equal one thread per ray nesting DeviceView::intersect with a precompute_tri(triangle_at(...))
    leaf, with every candidate accepted and with odd ids rejected."""
    for kind in ("soup", "grid"):
        tris = scenes.make_mesh(kind, 100_000, dtype=dtype)
        k0, k1 = moving_keys(tris, seed=2)
        scene = Scene(dmt, gpu_lib, k0, k1)
        rays = np.concatenate([scenes.make_primary(kind, 400, 400, dtype=dtype), special_rays(tris, dtype)])
        d_rays, n = cuda(rays), rays.shape[0]
        times = random_times(n, dtype=dtype)
        times[::97] = np.array([np.nan, -1.0, 2.0, 0.0, 1.0], dtype)[np.arange(times[::97].shape[0]) % 5]
        d_times = cuda(times)
        for filt in (0, 1):
            got = scene.run(MOTION, d_rays, d_times, n, filt, flags)
            assert_fields(got, scene.run(PER_THREAD, d_rays, d_times, n, filt, flags), RUN_NAMES, f"{kind} filter {filt}")
            assert (got[0] != -1).sum() > n // 10
            if filt == 1:
                assert ((got[0][got[0] != -1] & 1) == 0).all()
        scene.destroy()


def test_closest_equals_float64_brute_force(dmt, gpu_lib):
    """Closest ids of 4000 sampled rays at eight times equal a float64 brute force over the blended vertices (triangle_at),
    except rays whose two best float64 distances differ by less than 1e-4 relative or whose hit lies within 1e-4 of a
    triangle's edge (where float32 rounding may decide)."""
    import torch
    tris = scenes.make_mesh("soup", 20_000)
    k0, k1 = moving_keys(tris, seed=3)
    scene = Scene(dmt, gpu_lib, k0, k1)
    rays = scenes.make_primary("soup", 300, 300)
    rng = np.random.default_rng(2)
    sample = rng.permutation(rays.shape[0])[:4000]
    palette = rng.uniform(0, 1, size=8).astype(np.float32)
    which = np.arange(sample.shape[0]) % 8
    ids, t, _, _, _, _ = scene.run(MOTION, cuda(rays[sample]), cuda(palette[which]), sample.shape[0], 0, 0)
    checked = 0
    for w in range(8):
        world = torch.from_numpy(scene.triangle_at(float(palette[w])).astype(np.float64).reshape(-1, 3, 3)).cuda()
        p0, e1, e2 = world[:, 0], world[:, 1] - world[:, 0], world[:, 2] - world[:, 0]
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
                    assert int(ids[i]) == int(arg[j]), (i, bt, float(t[i]))
                    assert abs(float(t[i]) - bt) <= 1e-4 * max(abs(bt), 1.0)
    assert checked > 3000
    assert (ids != -1).mean() > 0.1
    scene.destroy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
def test_prepare_motion_triangles(dmt, gpu_lib, dtype):
    """Every box holds its triangle at 65 uniform and 48 random times (triangle_at dumps), for a mesh moving by a
    triangle's size and for one at 1e4 whose keys are a few ulps apart; at those times the latter's triangles leave the
    plain union of the key boxes, so the check sees a missing or short widening.  With equal keys boxes and centres are
    the static ones bit for bit; a key with a NaN gives the empty box and no hits."""
    tris = scenes.make_mesh("soup", 50_000, dtype=dtype)
    k0, k1 = moving_keys(tris, seed=4)
    k1[9, 4] = np.nan
    scene = Scene(dmt, gpu_lib, k0, k1)
    boxes = host(scene.boxes)
    assert (boxes[9, :3] == np.inf).all() and (boxes[9, 3:] == -np.inf).all()
    keep = np.arange(tris.shape[0]) != 9
    times = [*(np.arange(65) / 64), *rounding_times(48, 10, dtype)]
    for tau in times:
        v = scene.triangle_at(tau).reshape(-1, 3, 3)[keep]
        assert (boxes[keep, :3] <= v.min(axis=1)).all() and (boxes[keep, 3:] >= v.max(axis=1)).all(), tau
    u0, u1 = ulps_keys(tris, 11)
    near = Scene(dmt, gpu_lib, u0, u1)
    nb = host(near.boxes)
    w0, w1 = u0.reshape(-1, 3, 3), u1.reshape(-1, 3, 3)
    lo, hi = np.minimum(w0.min(axis=1), w1.min(axis=1)), np.maximum(w0.max(axis=1), w1.max(axis=1))
    outside = 0
    for tau in times:
        v = near.triangle_at(tau).reshape(-1, 3, 3)
        assert (nb[:, :3] <= v.min(axis=1)).all() and (nb[:, 3:] >= v.max(axis=1)).all(), ("ulps", tau)
        outside += int((v.min(axis=1) < lo).sum() + (v.max(axis=1) > hi).sum())
    assert outside > 0
    near.destroy()
    rays = scenes.make_primary("soup", 300, 300, dtype=dtype)
    got = scene.run(MOTION, cuda(rays), cuda(random_times(rays.shape[0], dtype=dtype)), rays.shape[0], 0, 0)
    assert (got[0] != -1).sum() > 0 and not (got[0] == 9).any()
    scene.destroy()
    same = Scene(dmt, gpu_lib, tris, tris, same=True)
    v = tris.reshape(-1, 3, 3)
    want = np.concatenate([v.min(axis=1), v.max(axis=1)], axis=1)
    centre = ((v[:, 0] + v[:, 1]) + v[:, 2]) * np.dtype(dtype).type(1.0 / 3.0)
    assert (host(same.boxes) == want).all() and (host(same.centres) == centre.astype(dtype)).all()
    same.destroy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
@pytest.mark.parametrize("flags", PATH_FLAGS, ids=PATH_IDS)
def test_one_launch_equals_wavefront_loop(dmt, gpu_lib, dtype, flags):
    """Moving keys: a path tracer with shadow segments and one random time per path gives the same radiance bits, segment
    counts and segment hashes in one motion trace_paths call as in a wavefront loop of motion trace_triangles launches."""
    for kind in ("soup", "grid"):
        tris = scenes.make_mesh(kind, 200_000, dtype=dtype)
        k0, k1 = moving_keys(tris, seed=5)
        scene = Scene(dmt, gpu_lib, k0, k1)
        primary = scenes.make_primary(kind, 300, 300, dtype=dtype)
        tracer = Tracer(scene, primary, random_times(primary.shape[0], 8, dtype), LIGHT[kind], 4)
        got = tracer(0, flags)
        assert_fields(got, tracer(1, flags), TRACER_NAMES, f"{kind} one launch vs wavefront")
        rad, segs, _ = got
        assert (segs >= 1).all() and segs.max() >= 4 and (segs > 1).mean() > 0.1
        assert np.isfinite(rad).all()
        scene.destroy()


def test_every_ray_and_path_once(dmt, gpu_lib):
    """finish is called once per ray and once per path at batch sizes around the scheduler's edges and at 1M; nothing
    past n is written; n = 0 launches nothing."""
    import torch
    tris = scenes.make_mesh("soup", 100_000)
    k0, k1 = moving_keys(tris, seed=6)
    scene = Scene(dmt, gpu_lib, k0, k1)
    props = torch.cuda.get_device_properties(0)
    wave = props.multi_processor_count * 9 * 4 * 32
    big = 1_000_007
    rays = np.resize(scenes.make_primary("soup", 1001, 1001), (max(wave + 1, big), 8))
    d_rays, d_times = cuda(rays), cuda(random_times(rays.shape[0]))
    tracer = Tracer(scene, rays, random_times(rays.shape[0], 9), LIGHT["soup"], 1)
    guard = 1000
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 4097, wave - 1, wave, wave + 1, big):
        for what in ("rays", "paths"):
            counts = torch.zeros(n + guard, dtype=torch.int32, device="cuda")
            if what == "rays":
                scene.run(MOTION, d_rays, d_times, n, 0, 0, counts=counts)
            else:
                tracer(0, 0, counts=counts, n=n)
            got = host(counts)
            assert (got[:n] == 1).all(), (what, n, np.nonzero(got[:n] != 1)[0][:8])
            assert (got[n:] == 0).all(), (what, n)
    scene.destroy()


def test_errors_leave_tree_usable(dmt, gpu_lib):
    """A triangle count other than the tree's and a null key raise invalid_argument, a short workspace length_error, each
    naming the motion call; none launches anything, and the tree traces as before afterwards.  The tree needs no
    attached triangles: the static call on it raises, the motion call does not."""
    import torch
    tris = scenes.make_mesh("soup", 50_000)
    k0, k1 = moving_keys(tris, seed=7)
    scene = Scene(dmt, gpu_lib, k0, k1)
    rays = scenes.make_primary("soup", 300, 300)
    d_rays, n = cuda(rays), rays.shape[0]
    d_times = cuda(random_times(n))
    first = scene.run(MOTION, d_rays, d_times, n, 0, 0)
    counts = torch.zeros(n, dtype=torch.int32, device="cuda")
    with pytest.raises(TypeError, match=r"trace_triangles \(motion\): 49999 triangles for a tree of 50000 primitives"):
        scene.run(MOTION, d_rays, d_times, n, 0, 0, counts=counts, count=49_999)
    with pytest.raises(TypeError, match=r"trace_triangles \(motion\): a null key pointer"):
        scene.run(MOTION, d_rays, d_times, n, 0, 0, counts=counts, k1=False)
    with pytest.raises(ValueError, match=r"trace_triangles \(motion\): a workspace of 7 bytes is too small"):
        scene.run(MOTION, d_rays, d_times, n, 0, 0, counts=counts, ws_bytes=7)
    with pytest.raises(TypeError, match=r"trace_triangles: the tree has no triangles"):
        scene.run(STATIC, d_rays, d_times, n, 0, 0, counts=counts)
    tracer = Tracer(scene, rays, random_times(n, 3), LIGHT["soup"], 2)
    paths = tracer(0, 0)
    with pytest.raises(TypeError, match=r"trace_paths \(motion\): 49999 triangles"):
        tracer(0, 0, counts=counts, count=49_999)
    with pytest.raises(ValueError, match=r"trace_paths \(motion\): a workspace of 7 bytes"):
        tracer(0, 0, counts=counts, ws_bytes=7)
    torch.cuda.synchronize()
    assert (host(counts) == 0).all()
    assert_fields(scene.run(MOTION, d_rays, d_times, n, 0, 0), first, RUN_NAMES, "after the errors")
    assert_fields(tracer(0, 0), paths, TRACER_NAMES, "paths after the errors")
    scene.destroy()


def test_animation_on_one_stream(dmt, gpu_lib):
    """Four frames on one torch stream, with no synchronisation between the steps: both keys rewritten on the device,
    prepare_motion_triangles, refit_boxes, the motion trace_triangles.  Each frame's records equal the motion call on a
    tree freshly built from that frame's boxes (closest hit, canonical tie rule: the record does not depend on the
    tree), and the motion changes the hits."""
    import torch
    api = gpu_lib
    tris = scenes.make_mesh("grid", 200_000)
    amp = 4 * tri_size(tris)
    frames = [deform(tris, 0.7 * f, amp) for f in range(5)]
    rays = scenes.make_primary("grid", 500, 500)
    d_rays, n = cuda(rays), rays.shape[0]
    d_times = cuda(random_times(n))
    d_keys = [cuda(f.reshape(-1)) for f in frames]
    stream = torch.cuda.Stream()
    api.set_stream(stream.cuda_stream)
    got = []
    try:
        scene = Scene(dmt, api, frames[0], frames[1])
        s = C.c_void_p(stream.cuda_stream)
        with torch.cuda.stream(stream):
            for f in range(4):
                scene.k0.copy_(d_keys[f])
                scene.k1.copy_(d_keys[f + 1])
                scene.prepare(s)
                scene.bvh.refit_boxes(scene.boxes.data_ptr(), api.DEVICE_POINTERS)
                out = scene.run(MOTION, d_rays, d_times, n, 0, 0, stream=s, sync=False)
                got.append(tuple(x.clone() for x in out))
        stream.synchronize()
        got = [tuple(host(x) for x in f) for f in got]
        scene.destroy()
    finally:
        api.set_stream(None)
    for f in range(4):
        fresh = Scene(dmt, api, frames[f], frames[f + 1])
        want = fresh.run(MOTION, d_rays, d_times, n, 0, 0)
        assert_fields(got[f][:4], want[:4], RUN_NAMES[:4], f"frame {f}")
        fresh.destroy()
    assert all((got[f][0] != -1).sum() > n // 10 for f in range(4))
    assert (got[0][1] != got[1][1]).any()
