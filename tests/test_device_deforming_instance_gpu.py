"""The deforming forms of DeviceView::trace_instances and trace_instance_paths, make_deforming_instance and
prepare_deforming_instances on the GPU (test shaders in tests/device_deforming_instance_kernels.cu).

Scenes mix three bottom kinds: a static soup, a deforming soup on shutter boxes (its tree built over
prepare_motion_triangles' boxes) and the same deforming soup with motion nodes (prepare_motion_nodes).  Checked, in
float and double and for every flag and tie rule: the three reductions (static bottoms only: the motion
trace_instances; one identity record: the motion or motion-node trace_triangles on its mesh; equal vertex keys: the
static bottom on the same tree) bit for bit; a mixed scene of 60 copies with moving placements against one thread per
ray nesting the traversal by hand and against a float64 brute force; shutter-box and motion-node bottoms giving the same
robust canonical closest hits; scripted paths against the same segments through trace_instances; every ray and path
finished once; the errors; and four animated frames on one torch stream."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes
from tests.test_device_instance_trace_gpu import placements, world_rays
from tests.test_device_motion_instance_gpu import moving_keys

pytestmark = pytest.mark.gpu

P, SZ, U = C.c_void_p, C.c_size_t, C.c_uint
ANY, ROBUST, LAST = 1, 2, 4
MODES = [m | t for t in (0, LAST) for m in (0, ROBUST, ANY, ANY | ROBUST)]
MODE_IDS = [f"{m}-{t}" for t in ("lowest", "last") for m in ("closest", "robust", "any", "any-robust")]
DTYPES = [np.float32, np.float64]
NAMES = ("ids", "t", "u", "v", "inst", "calls", "hashes")


@pytest.fixture(scope="module")
def ddi(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_deforming_instance_tests())
    for s in ("3f", "3d"):
        getattr(L, f"ddi_records{s}").argtypes = [P, P, P, P, P, P, P, P, SZ, P, C.POINTER(SZ), P]
        getattr(L, f"ddi_set_keys{s}").argtypes = [P, P, P, SZ, P]
        getattr(L, f"ddi_prepare{s}").argtypes = [P, SZ, SZ, P, P, P]
        getattr(L, f"ddi_bottom{s}").argtypes = [P, P, P, SZ, P, P, P, P, SZ, P]
        getattr(L, f"ddi_run{s}").argtypes = [P, P, P, SZ, SZ, C.c_int, C.c_int, U, P, P, SZ] + [P] * 8 + [P, P, SZ, P]
        getattr(L, f"ddi_paths{s}").argtypes = [P, P, SZ, SZ, C.c_int, U, SZ, P, P, P, P] + [P] * 9 + [P, SZ, P]
        for f in ("record_bytes", "motion_record_bytes", "motion_node_bytes"):
            getattr(L, f"ddi_{f}{s}").restype = SZ
    L.ddi_last_error.restype = C.c_char_p
    return L


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def check(lib, rc):
    if rc:
        msg = lib.ddi_last_error().decode()
        raise {-2: ValueError, -3: TypeError}.get(rc, RuntimeError)(msg)


def bits(a):
    return a.view(np.uint32 if a.dtype.itemsize == 4 else np.uint64) if a.dtype.kind == "f" else a


def assert_same(got, want, what=""):
    for name, a, b in zip(NAMES, got, want):
        same = bits(a) == bits(b)
        assert same.all(), f"{what} {name} differs at {np.nonzero(~same)[0][:8]}"


def deforming_keys(tris, dtype, step, seed=5, equal=False):
    """vertex keys: the soup at time 0, and each vertex moved by up to `step` at time 1"""
    k0 = np.ascontiguousarray(tris, dtype)
    if equal:
        return k0, k0
    rng = np.random.default_rng(seed)
    return k0, np.ascontiguousarray(k0 + rng.uniform(-step, step, size=k0.shape), dtype)


class Bottom:
    """A mesh as a static handle (build_triangles) or a deforming one: vertex keys on the device, a tree over
    prepare_motion_triangles' boxes and its motion nodes."""

    def __init__(self, ddi, api, tris, dtype, step=0.0, equal=False, attach=False):
        import torch
        self.s = "3f" if np.dtype(dtype) == np.float32 else "3d"
        td = torch.float32 if self.s == "3f" else torch.float64
        self.ddi, self.api, self.dtype = ddi, api, np.dtype(dtype)
        self.k0, self.k1 = deforming_keys(tris, dtype, step, equal=equal)
        self.d0, self.d1 = cuda(self.k0), cuda(self.k1)
        n = self.k0.shape[0]
        self.boxes = torch.empty((n, 6), dtype=td, device="cuda")
        self.centres = torch.empty((n, 3), dtype=td, device="cuda")
        self.step(boxes_only=True)
        self.h = api.Bvh.build_boxes(self.boxes.data_ptr(), self.centres.data_ptr(), count=n, dtype=self.dtype, flags=api.DEVICE_POINTERS)
        if attach:
            self.h.set_triangles(self.k0)
        nb = getattr(ddi, f"ddi_motion_node_bytes{self.s}")()
        self.nodes = torch.zeros((self.h.node_count + 1) * nb, dtype=torch.uint8, device="cuda")
        self.ws = torch.empty(2 * (self.h.node_count + 1) * 4 + 16, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        self.step()

    def step(self, boxes_only=False, stream=None, sync=True):
        """the bottom's per-frame step: prepare_motion_triangles, the refit, prepare_motion_nodes.  sync=False: nothing
        waits, so `stream` must be the handle's (api.set_stream before the handle was built)"""
        import torch
        check(self.ddi, getattr(self.ddi, f"ddi_bottom{self.s}")(None, ptr(self.d0), ptr(self.d1), self.k0.shape[0], ptr(self.boxes),
                                                                 ptr(self.centres), None, None, 0, stream))
        if boxes_only:
            return
        if sync:
            torch.cuda.synchronize()
        self.h.refit_boxes(self.boxes.data_ptr(), flags=self.api.DEVICE_POINTERS)
        if sync:
            self.h.sync()
        check(self.ddi, getattr(self.ddi, f"ddi_bottom{self.s}")(C.c_void_p(self.h.handle), ptr(self.d0), ptr(self.d1), self.k0.shape[0],
                                                                 None, None, ptr(self.nodes), ptr(self.ws), self.ws.numel(), stream))
        if sync:
            torch.cuda.synchronize()


class Scene:
    """Records of (kind, mesh index, key0, key1) over bottoms, prepare_deforming_instances' boxes and a top tree."""

    def __init__(self, ddi, api, static, deforming, kinds, mesh_of, keys0, keys1, dtype):
        import torch
        self.ddi, self.api = ddi, api
        self.s = "3f" if np.dtype(dtype) == np.float32 else "3d"
        self.dtype = np.dtype(dtype)
        self.tdtype = torch.float32 if self.s == "3f" else torch.float64
        self.bottoms = [static, deforming]
        self.count = len(kinds)
        self.kinds = np.ascontiguousarray(kinds, np.int32)
        # mesh 0: the static handle; mesh 1: the deforming handle
        mesh_of = np.ascontiguousarray([0 if k == 0 else 1 for k in kinds] if mesh_of is None else mesh_of, np.uint32)
        handles = (C.c_void_p * 2)(static.h.handle if static else deforming.h.handle, deforming.h.handle if deforming else static.h.handle)
        dev = deforming if deforming else static
        vk0 = (C.c_void_p * 2)(dev.d0.data_ptr(), dev.d0.data_ptr())
        vk1 = (C.c_void_p * 2)(dev.d1.data_ptr(), dev.d1.data_ptr())
        mn = (C.c_void_p * 2)(dev.nodes.data_ptr(), dev.nodes.data_ptr())
        self.rec_bytes = getattr(ddi, f"ddi_record_bytes{self.s}")()
        self.records = torch.zeros(self.count * self.rec_bytes, dtype=torch.uint8, device="cuda")
        self.scratch = torch.zeros(self.count * getattr(ddi, f"ddi_motion_record_bytes{self.s}")() + 16, dtype=torch.uint8, device="cuda")
        k0, k1 = np.ascontiguousarray(keys0, dtype), np.ascontiguousarray(keys1, dtype)
        depth = SZ(0)
        torch.cuda.synchronize()
        check(ddi, getattr(ddi, f"ddi_records{self.s}")(handles, mesh_of.ctypes.data, self.kinds.ctypes.data, k0.ctypes.data, k1.ctypes.data,
                                                        vk0, vk1, mn, self.count, ptr(self.records), C.byref(depth), None))
        self.max_depth = depth.value
        self.boxes = torch.empty((self.count, 6), dtype=self.tdtype, device="cuda")
        self.centres = torch.empty((self.count, 3), dtype=self.tdtype, device="cuda")
        self.prepare()
        torch.cuda.synchronize()
        self.top = api.Bvh.build_boxes(self.boxes.data_ptr(), self.centres.data_ptr(), count=self.count, dtype=self.dtype,
                                       flags=api.DEVICE_POINTERS)
        self.ws = torch.empty(64, dtype=torch.uint8, device="cuda")

    def prepare(self, stream=None):
        check(self.ddi, getattr(self.ddi, f"ddi_prepare{self.s}")(ptr(self.records), self.count, self.max_depth, ptr(self.boxes),
                                                                  ptr(self.centres), stream))

    def run(self, d_rays, d_times, n, filt, flags, mode=0, counts=None, bottom=None, ws_bytes=None, count=None, max_depth=None,
            stream=None):
        import torch
        ids = torch.empty(n, dtype=torch.int32, device="cuda")
        t, u, v = (torch.empty(n, dtype=self.tdtype, device="cuda") for _ in range(3))
        inst, calls = (torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2))
        hashes = torch.empty(n, dtype=torch.int64, device="cuda")
        rc = getattr(self.ddi, f"ddi_run{self.s}")(
            C.c_void_p(self.top.handle), C.c_void_p(bottom.h.handle) if bottom else None, ptr(self.records),
            self.count if count is None else count, self.max_depth if max_depth is None else max_depth, mode, filt, flags, ptr(d_rays),
            ptr(d_times), n, ptr(ids), ptr(t), ptr(u), ptr(v), ptr(inst), ptr(calls), ptr(hashes), ptr(counts), ptr(self.scratch), ptr(self.ws),
            self.ws.numel() if ws_bytes is None else ws_bytes, stream)
        check(self.ddi, rc)
        torch.cuda.synchronize()
        out = [x.cpu().numpy() for x in (ids, t, u, v, inst, calls, hashes)]
        out[0], out[4], out[5] = (x.view(np.uint32) for x in (out[0], out[4], out[5]))
        return out


def ray_times(n, seed=11):
    rng = np.random.default_rng(seed)
    t = rng.uniform(0.0, 1.0, size=n)
    t[::7] = 0.0
    t[1::7] = 1.0
    t[2::7] = 0.5
    t[3::11] = -1.0
    t[4::11] = 2.0
    t[5::13] = np.nan
    return t


def mixed_scene(ddi, api, dtype, count=60, kinds=None, equal_vertices=False, move=True):
    tris = scenes.soup(4000)
    static = Bottom(ddi, api, tris, dtype, attach=True, equal=True)
    deforming = Bottom(ddi, api, tris, dtype, step=0.01, equal=equal_vertices)
    if kinds is None:
        kinds = [k % 3 for k in range(count)]
    keys0, keys1 = moving_keys(count, singular=(7,)) if move else (placements(count),) * 2
    return Scene(ddi, api, static, deforming, kinds, None, keys0, keys1, dtype), tris


def rays_for(scene_keys, dtype, w=96, h=96):
    rays = world_rays(scene_keys, w, h, dtype)
    times = ray_times(rays.shape[0]).astype(dtype)
    return rays, times


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
def test_mixed_scene_equals_hand_nested(ddi, gpu_lib, dtype, flags):
    api = gpu_lib
    scene, _ = mixed_scene(ddi, api, dtype)
    keys0, _ = moving_keys(60, singular=(7,))
    rays, times = rays_for(keys0, dtype)
    d_rays, d_times = cuda(rays), cuda(times)
    for filt in (0, 1):
        got = scene.run(d_rays, d_times, rays.shape[0], filt, flags, mode=0)
        want = scene.run(d_rays, d_times, rays.shape[0], filt, flags, mode=1)
        assert_same(got, want, f"filter {filt}")
        if filt == 0 and not flags & ANY:
            assert (got[4] != 0xFFFFFFFF).sum() > rays.shape[0] // 10
            kinds = np.array([k % 3 for k in range(60)])
            hit_kinds = set(kinds[got[4][got[4] != 0xFFFFFFFF]].tolist())
            assert hit_kinds == {0, 1, 2}, hit_kinds


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
def test_static_bottoms_equal_motion_instances(ddi, gpu_lib, dtype, flags):
    api = gpu_lib
    scene, _ = mixed_scene(ddi, api, dtype, kinds=[0] * 60)
    keys0, _ = moving_keys(60, singular=(7,))
    rays, times = rays_for(keys0, dtype)
    d_rays, d_times = cuda(rays), cuda(times)
    for filt in (0, 1):
        assert_same(scene.run(d_rays, d_times, rays.shape[0], filt, flags, mode=0),
                    scene.run(d_rays, d_times, rays.shape[0], filt, flags, mode=2), f"filter {filt}")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("kind", [1, 2], ids=["shutter", "nodes"])
@pytest.mark.parametrize("name", ["soup", "grid"])
def test_identity_record_equals_trace_triangles(ddi, gpu_lib, dtype, flags, kind, name):
    api = gpu_lib
    tris = scenes.soup(20000) if name == "soup" else scenes.grid(20000)
    b = Bottom(ddi, api, tris, dtype, step=0.002)
    ident = np.array([[1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]], np.float64)
    scene = Scene(ddi, api, None, b, [kind], [0], ident, ident, dtype)
    rays = scenes.make_primary(name, 128, 128).astype(dtype)
    times = ray_times(rays.shape[0]).astype(dtype)
    d_rays, d_times = cuda(rays), cuda(times)
    got = scene.run(d_rays, d_times, rays.shape[0], 0, flags, mode=0)
    want = scene.run(d_rays, d_times, rays.shape[0], 0, flags, mode=3, bottom=b)
    assert_same(got, want)
    assert (got[4] != 0xFFFFFFFF).sum() > 0


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
def test_equal_vertex_keys_equal_static_bottom(ddi, gpu_lib, dtype, flags):
    """With equal vertex keys, shutter-box and motion-node bottoms are the static bottom on the same tree."""
    api = gpu_lib
    tris = scenes.soup(4000)
    b = Bottom(ddi, api, tris, dtype, equal=True, attach=True)
    keys0, keys1 = moving_keys(24)
    rays, times = rays_for(keys0, dtype, 64, 64)
    d_rays, d_times = cuda(rays), cuda(times)
    runs, boxes = [], []
    for kind in (0, 1, 2):
        scene = Scene(ddi, api, None, b, [kind] * 24, [0] * 24, keys0, keys1, dtype)
        runs.append(scene.run(d_rays, d_times, rays.shape[0], 0, flags))
        boxes.append(scene.boxes.cpu().numpy())
    assert np.array_equal(bits(boxes[1]), bits(boxes[0])) and np.array_equal(bits(boxes[2]), bits(boxes[0]))
    assert_same(runs[1], runs[0], "shutter boxes")
    assert_same(runs[2], runs[0], "motion nodes")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_shutter_and_nodes_same_closest_hits(ddi, gpu_lib, dtype):
    api = gpu_lib
    tris = scenes.soup(4000)
    static = Bottom(ddi, api, tris, dtype, attach=True, equal=True)
    deforming = Bottom(ddi, api, tris, dtype, step=0.01)
    keys0, keys1 = moving_keys(40)
    rays, times = rays_for(keys0, dtype)
    d_rays, d_times = cuda(rays), cuda(times)
    out = []
    for kind in (1, 2):
        scene = Scene(ddi, api, static, deforming, [kind] * 40, None, keys0, keys1, dtype)
        out.append(scene.run(d_rays, d_times, rays.shape[0], 0, ROBUST))
    for k in (0, 1, 2, 3, 4):
        assert np.array_equal(bits(out[0][k]), bits(out[1][k])), NAMES[k]


def blend(k0, k1, tau):
    """detail::blend_key in numpy, at the keys' precision"""
    tau = np.where(np.isnan(tau), 0, np.clip(tau, 0, 1)).astype(k0.dtype)
    rest = (np.ones_like(tau) - tau).astype(k0.dtype)
    out = (rest * k0 + tau * k1).astype(k0.dtype)
    out = np.where(k0 == k1, k0, out)
    out = np.where(tau == 0, k0, out)
    return np.where(tau == 1, k1, out)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_mixed_scene_brute_force(ddi, gpu_lib, dtype):
    """Closest hits against a float64 brute force over the blended, placed vertices of every record."""
    api = gpu_lib
    scene, tris = mixed_scene(ddi, api, dtype, count=12, move=True)
    keys0, keys1 = moving_keys(12, singular=(7,))
    rays, times = rays_for(keys0, dtype, 24, 24)
    got = scene.run(cuda(rays), cuda(times), rays.shape[0], 0, 0)
    dev = scene.bottoms[1]
    kinds = [k % 3 for k in range(12)]
    checked = 0
    for i in range(rays.shape[0]):
        tau = times[i:i + 1]
        o = rays[i, :3].astype(np.float64)
        d = rays[i, 3:6].astype(np.float64)
        best, best_k, second = np.inf, -1, np.inf
        for k in range(12):
            m = blend(np.asarray(keys0[k], dtype), np.asarray(keys1[k], dtype), tau).astype(np.float64).reshape(3, 4)
            if abs(np.linalg.det(m[:, :3])) < 1e-12:
                continue
            v = (blend(dev.k0, dev.k1, tau) if kinds[k] else dev.k0).astype(np.float64).reshape(-1, 3, 3)
            w = v @ m[:, :3].T + m[:, 3]
            e1, e2 = w[:, 1] - w[:, 0], w[:, 2] - w[:, 0]
            p = np.cross(d, e2)
            det = (e1 * p).sum(1)
            s = o - w[:, 0]
            with np.errstate(divide="ignore", invalid="ignore"):
                uu = (s * p).sum(1) / det
                q = np.cross(s, e1)
                vv = (q @ d) / det
                tt = (e2 * q).sum(1) / det
            ok = (uu >= 0) & (vv >= 0) & (uu + vv <= 1) & (tt >= 0) & np.isfinite(tt)
            for t_ in np.sort(tt[ok])[:2]:
                if t_ < best:
                    best, second, best_k = t_, best, k
                elif t_ < second:
                    second = t_
        if best_k < 0:
            continue
        if second - best > 1e-4 * max(1.0, best):
            assert got[4][i] == best_k, (i, got[4][i], best_k)
            assert abs(float(got[1][i]) - best) < 1e-3 * max(1.0, best), (i, got[1][i], best)
            checked += 1
    assert checked > 50


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
@pytest.mark.parametrize("flags", [0, ROBUST, LAST, ROBUST | LAST], ids=["fast-lowest", "robust-lowest", "fast-last", "robust-last"])
def test_paths_equal_segments(ddi, gpu_lib, dtype, flags):
    api = gpu_lib
    import torch
    scene, _ = mixed_scene(ddi, api, dtype)
    keys0, _ = moving_keys(60, singular=(7,))
    rays, _ = rays_for(keys0, dtype, 48, 48)
    n_paths = 700
    rng = np.random.default_rng(4)
    lengths = rng.integers(0, 9, size=n_paths)
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.uint64)
    segs = int(offsets[-1])
    pick = rng.integers(0, rays.shape[0], size=segs)
    seg_rays = np.ascontiguousarray(rays[pick])
    seg_any = (rng.uniform(size=segs) < 0.4).astype(np.uint8)
    times = ray_times(n_paths).astype(dtype)
    seg_times = np.repeat(times, lengths).astype(dtype)
    outs = [torch.empty(segs, dtype=x, device="cuda") for x in (torch.int32, scene.tdtype, scene.tdtype, scene.tdtype, torch.int32,
                                                                  torch.int32, torch.int64)]
    counts = torch.zeros(n_paths, dtype=torch.int32, device="cuda")
    ray_ok = torch.zeros(segs, dtype=torch.int32, device="cuda")
    # (each device array held in a name for the whole call: a temporary would be freed, and its block reused, before it)
    d_seg, d_any, d_off, d_pt = cuda(seg_rays), cuda(seg_any), cuda(offsets), cuda(times)
    check(ddi, getattr(ddi, f"ddi_paths{scene.s}")(C.c_void_p(scene.top.handle), ptr(scene.records), scene.count, scene.max_depth, 0, flags,
                                                   n_paths, ptr(d_seg), ptr(d_any), ptr(d_off), ptr(d_pt),
                                                   *[ptr(o) for o in outs], ptr(counts), ptr(ray_ok), ptr(scene.ws), scene.ws.numel(), None))
    torch.cuda.synchronize()
    got = [o.cpu().numpy() for o in outs]
    got[0], got[4], got[5] = (x.view(np.uint32) for x in (got[0], got[4], got[5]))
    assert (counts.cpu().numpy() == 1).all()
    assert (ray_ok.cpu().numpy() == 1).all()
    for any_hit in (0, 1):
        sel = np.nonzero(seg_any == any_hit)[0]
        want = scene.run(cuda(seg_rays[sel]), cuda(seg_times[sel]), sel.size, 0, flags | (ANY if any_hit else 0))
        assert_same([g[sel] for g in got], want, f"any {any_hit}")


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 255, 256, 257, 4095, 4096, 4097, 1_000_000])
def test_every_ray_and_path_finishes_once(ddi, gpu_lib, n):
    api = gpu_lib
    import torch
    scene, _ = mixed_scene(ddi, api, np.float32)
    keys0, _ = moving_keys(60, singular=(7,))
    side = max(1, int(np.ceil(np.sqrt(max(n, 1)))))
    rays, _ = rays_for(keys0, np.float32, side, side)
    rays = np.ascontiguousarray(rays[:n])
    times = ray_times(n).astype(np.float32)
    counts = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
    scene.run(cuda(rays), cuda(times), n, 0, 0, counts=counts)
    assert (counts.cpu().numpy()[:n] == 1).all()
    if n <= 4097:
        counts.zero_()
        lengths = np.full(n, 2)
        offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.uint64)
        seg_rays = np.ascontiguousarray(np.repeat(rays, 2, axis=0)) if n else np.zeros((1, 8), np.float32)
        seg_any = np.tile([0, 1], max(n, 1)).astype(np.uint8)
        segs = max(2 * n, 1)
        outs = [torch.empty(segs, dtype=torch.int32, device="cuda") for _ in range(7)]
        ray_ok = torch.zeros(segs, dtype=torch.int32, device="cuda")
        d_seg, d_any, d_off = cuda(seg_rays), cuda(seg_any), cuda(offsets)
        d_pt = cuda(times if n else np.zeros(1, np.float32))
        check(ddi, ddi.ddi_paths3f(C.c_void_p(scene.top.handle), ptr(scene.records), scene.count, scene.max_depth, 0, 0, n, ptr(d_seg),
                                   ptr(d_any), ptr(d_off), ptr(d_pt),
                                   ptr(outs[0]), None, None, None, ptr(outs[4]), None, None, ptr(counts), ptr(ray_ok), ptr(scene.ws),
                                   scene.ws.numel(), None))
        torch.cuda.synchronize()
        assert (counts.cpu().numpy()[:n] == 1).all()


def test_errors_leave_trees_usable(ddi, gpu_lib):
    api = gpu_lib
    scene, _ = mixed_scene(ddi, api, np.float32)
    keys0, _ = moving_keys(60, singular=(7,))
    rays, times = rays_for(keys0, np.float32, 32, 32)
    d_rays, d_times = cuda(rays), cuda(times)
    before = scene.run(d_rays, d_times, rays.shape[0], 0, 0)
    with pytest.raises(TypeError, match=r"trace_instances \(deforming\)"):
        scene.run(d_rays, d_times, rays.shape[0], 0, 0, count=scene.count - 1)
    with pytest.raises(ValueError, match=r"trace_instances \(deforming\)"):
        scene.run(d_rays, d_times, rays.shape[0], 0, 0, ws_bytes=4)
    with pytest.raises(ValueError, match=r"trace_instances \(deforming\)"):
        scene.run(d_rays, d_times, rays.shape[0], 0, 0, max_depth=60000)
    assert_same(scene.run(d_rays, d_times, rays.shape[0], 0, 0), before, "after errors")


def test_animation_frames_on_one_stream(ddi, gpu_lib):
    """Four frames, each with no wait between its steps: new vertex keys and placement keys (device copies), the
    deforming bottom's step (prepare_motion_triangles, its refit, prepare_motion_nodes), prepare_deforming_instances,
    the top refit and the trace, all on one torch stream that every handle uses.  The boxes equal a fresh preparation
    per frame and the trace the hand-nested reference."""
    api = gpu_lib
    import torch
    stream = torch.cuda.Stream()
    sp = C.c_void_p(stream.cuda_stream)
    api.set_stream(stream.cuda_stream)
    try:
        with torch.cuda.stream(stream):
            scene, tris = mixed_scene(ddi, api, np.float32)
            dev = scene.bottoms[1]
            rng = np.random.default_rng(8)
            frames = []
            for frame in range(4):
                keys0, keys1 = moving_keys(60, seed=20 + frame, singular=(7,))
                v1 = (dev.k0 + rng.uniform(-0.01, 0.01, size=dev.k0.shape)).astype(np.float32)
                rays, times = rays_for(keys0, np.float32, 48, 48)
                frames.append((keys0, keys1, v1, cuda(v1), cuda(np.asarray(keys0, np.float32)), cuda(np.asarray(keys1, np.float32)),
                               cuda(rays), cuda(times), rays.shape[0]))
            torch.cuda.synchronize()
            for frame, (keys0, keys1, v1, d_v1, d_k0, d_k1, d_rays, d_times, n) in enumerate(frames):
                dev.d1.copy_(d_v1, non_blocking=True)                               # the frame's vertex keys
                dev.step(stream=sp, sync=False)
                check(ddi, ddi.ddi_set_keys3f(ptr(scene.records), ptr(d_k0), ptr(d_k1), 60, sp))
                scene.prepare(sp)
                scene.top.refit_boxes(scene.boxes.data_ptr(), flags=api.DEVICE_POINTERS)
                got = scene.run(d_rays, d_times, n, 0, 0, stream=sp)               # (synchronises after the trace)
                dev.k1 = v1
                # the boxes equal a fresh preparation bit for bit; the refitted top tree keeps its first topology, so
                # the trace is compared with the hand-nested reference on that tree (the accept order depends on it)
                fresh = Scene(ddi, api, scene.bottoms[0], dev, [k % 3 for k in range(60)], None, keys0, keys1, np.float32)
                assert np.array_equal(bits(fresh.boxes.cpu().numpy()), bits(scene.boxes.cpu().numpy()))
                want = scene.run(d_rays, d_times, n, 0, 0, mode=1, stream=sp)
                assert_same(got, want, f"frame {frame}")
    finally:
        torch.cuda.synchronize()
        api.set_stream(None)
