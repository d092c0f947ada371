"""prepare_motion_nodes, node_at and the motion-node forms of DeviceView::trace_triangles and trace_paths on the GPU
(test shaders in tests/device_motion_nodes_kernels.cu; scenes and helpers from tests/test_device_motion_triangle_gpu.py).
With equal keys the records are the refitted bounds bit for bit and the calls equal the motion calls on the shutter-box
tree bit for bit; with moving keys (all of the mesh, or half of it beside a static half), robust closest-hit records with
canonical ties equal the motion call on every ray, robust any-hit agrees on hit or miss, and fast closest hits match a
float64 brute force; a recording shader equals one thread per ray through a node_at node test; node_at boxes hold their
subtrees at uniform and full-mantissa random times, a half-static grid among the meshes;
a view with NaN node bounds gives the same results; a motion of four triangle sizes needs less than half the triangle
tests; one path-tracing launch equals its wavefront loop and, with robust traversal, the motion call's radiance; every
ray and path is finished once; the errors leave the tree usable; four animation frames on one stream equal a fresh
prepare_motion_nodes per frame."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes
from tests.test_device_motion_triangle_gpu import (ANY, LAST, LIGHT, MODE_IDS, MODES, PATH_FLAGS, PATH_IDS, ROBUST, RUN_NAMES,
                                                   TRACER_NAMES, P, SZ, U, U32, Scene, Tracer, assert_fields, cuda, deform, dmt,
                                                   host, moving_keys, ptr, random_times, rounding_times, tri_size, ulps_keys)
from tests.test_device_triangle_trace_gpu import special_rays

pytestmark = pytest.mark.gpu
__all__ = ["dmt"]                       # (the deforming-mesh fixture, used by Scene)

NODES, SHUTTER, PER_THREAD, NAN_VIEW = 0, 1, 2, 3


@pytest.fixture(scope="module")
def dmn(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_motion_nodes_tests())
    for s in ("3f", "3d"):
        real = C.c_float if s == "3f" else C.c_double
        getattr(L, f"dmn_prepare{s}").argtypes = [P, P, P, SZ, P, P, SZ, P]
        getattr(L, f"dmn_node_at{s}").argtypes = [P, SZ, real, P, P]
        getattr(L, f"dmn_extent{s}").argtypes = [P, P, P, SZ, real, P, P, SZ, P]
        getattr(L, f"dmn_run{s}").argtypes = [P, P, P, SZ, P, SZ, C.c_int, C.c_int, U, P, P, SZ] + [P] * 9 + [P, SZ, P]
        getattr(L, f"dmn_tracer{s}").argtypes = [P, P, P, SZ, P, SZ, C.c_int, U, SZ, P, P, P, U32, P, P, P, P, P, P, SZ, P]
        getattr(L, f"dmn_wavefront_bytes{s}").argtypes = [SZ]
        getattr(L, f"dmn_wavefront_bytes{s}").restype = SZ
    L.dmn_last_error.restype = C.c_char_p
    return L


def check(lib, rc):
    if rc:
        msg = lib.dmn_last_error().decode()
        raise {-2: ValueError, -3: TypeError}.get(rc, RuntimeError)(msg)


class NodeScene(Scene):
    """Scene (keys, prepare_motion_triangles' boxes, the shutter-box tree) with its motion nodes"""

    def __init__(self, dmn, dmt, api, key0, key1, same=False, stream=None):
        import torch
        super().__init__(dmt, api, key0, key1, same, stream)
        self.dmn = dmn
        self.node_count = self.bvh.node_count
        self.nodes = torch.zeros((self.node_count + 1) * (64 if self.s == "3f" else 128), dtype=torch.uint8, device="cuda")
        self.bu_ws = torch.empty(2 * (self.node_count + 1) * 4, dtype=torch.uint8, device="cuda")
        self.prepare_nodes(stream)
        torch.cuda.synchronize()

    def prepare_nodes(self, stream=None, count=None, ws_bytes=None, out=True):
        check(self.dmn, getattr(self.dmn, f"dmn_prepare{self.s}")(
            C.c_void_p(self.bvh.handle), ptr(self.k0), ptr(self.k1), self.count if count is None else count,
            ptr(self.nodes) if out else None, ptr(self.bu_ws), self.bu_ws.numel() if ws_bytes is None else ws_bytes, stream))

    def records(self):
        """(key 0 bounds, key 1 bounds, index) per slot, host arrays; bounds as minx, maxx, miny, maxy, minz, maxz"""
        import torch
        torch.cuda.synchronize()
        raw = host(self.nodes)
        real, ui = (np.float32, np.uint32) if self.s == "3f" else (np.float64, np.uint64)
        rec = np.dtype([("xy", real, (2, 4)), ("z", real, (2, 2)), ("index", ui), ("pad", ui, 3)])
        r = raw.view(rec)
        keys = [np.concatenate([r["xy"][:, k], r["z"][:, k]], axis=1) for k in range(2)]
        return keys[0], keys[1], r["index"]

    def node_at(self, tau):
        import torch
        out = torch.zeros((self.node_count + 1) * 6, dtype=self.tdtype, device="cuda")
        check(self.dmn, getattr(self.dmn, f"dmn_node_at{self.s}")(ptr(self.nodes), self.node_count, tau, ptr(out), None))
        torch.cuda.synchronize()
        return host(out).reshape(-1, 6)[1:]

    def extent(self, tau):
        import torch
        out = torch.zeros((self.node_count + 1) * 6, dtype=self.tdtype, device="cuda")
        check(self.dmn, getattr(self.dmn, f"dmn_extent{self.s}")(C.c_void_p(self.bvh.handle), ptr(self.k0), ptr(self.k1), self.count,
                                                                 tau, ptr(out), ptr(self.bu_ws), self.bu_ws.numel(), None))
        torch.cuda.synchronize()
        return host(out).reshape(-1, 6)[1:]

    def run_nodes(self, mode, d_rays, d_times, n, filt, flags, counts=None, ws_bytes=None, node_count=None, nodes=True, steps=False,
                  stream=None, sync=True):
        import torch
        ids = torch.empty(n, dtype=torch.int32, device="cuda")
        t, u, v = (torch.empty(n, dtype=self.tdtype, device="cuda") for _ in range(3))
        calls = torch.empty(n, dtype=torch.int32, device="cuda")
        hashes = torch.empty(n, dtype=torch.int64, device="cuda")
        inner, tests = (torch.zeros(n, dtype=torch.int32, device="cuda") for _ in range(2)) if steps else (None, None)
        check(self.dmn, getattr(self.dmn, f"dmn_run{self.s}")(
            C.c_void_p(self.bvh.handle), ptr(self.k0), ptr(self.k1), self.count, ptr(self.nodes) if nodes else None,
            self.node_count if node_count is None else node_count, mode, filt, flags, ptr(d_rays), ptr(d_times), n, ptr(ids), ptr(t),
            ptr(u), ptr(v), ptr(calls), ptr(hashes), ptr(counts), ptr(inner), ptr(tests), ptr(self.ws),
            self.ws.numel() if ws_bytes is None else ws_bytes, stream))
        out = (ids, t, u, v, calls, hashes)
        if not sync:
            return out
        torch.cuda.synchronize()
        if steps:
            return tuple(host(x) for x in out), host(inner), host(tests)
        return tuple(host(x) for x in out)


class NodeTracer(Tracer):
    """The path tracer: one motion-node trace_paths call (mode 0), its wavefront loop (1), the motion trace_paths (2)"""

    def __init__(self, scene, primary, times, light, bounces):
        import torch
        super().__init__(scene, primary, times, light, bounces)
        self.scratch = torch.empty(getattr(scene.dmn, f"dmn_wavefront_bytes{scene.s}")(self.n), dtype=torch.uint8, device="cuda")

    def __call__(self, mode, flags, counts=None, n=None, ws_bytes=8, node_count=None):
        import torch
        sc = self.scene
        out = (torch.full((self.n,), float("nan"), dtype=sc.tdtype, device="cuda"),
               torch.full((self.n,), -1, dtype=torch.int32, device="cuda"), torch.zeros(self.n, dtype=torch.int32, device="cuda"))
        check(sc.dmn, getattr(sc.dmn, f"dmn_tracer{sc.s}")(
            C.c_void_p(sc.bvh.handle), ptr(sc.k0), ptr(sc.k1), sc.count, ptr(sc.nodes), sc.node_count if node_count is None else node_count,
            mode, flags, self.n if n is None else n, ptr(self.primary), ptr(self.times), self.light.ctypes.data, self.bounces,
            *[ptr(x) for x in out], ptr(counts), ptr(self.scratch), ptr(self.ws), ws_bytes, None))
        torch.cuda.synchronize()
        return tuple(host(x) for x in out)


EQUAL_SCENES = [("soup", 1_000_000, 1000, np.float32), ("grid", 1_000_000, 1000, np.float32), ("soup", 200_000, 500, np.float64)]


@pytest.fixture(scope="module", params=EQUAL_SCENES, ids=["c2-soup-3f", "c2-grid-3f", "soup-3d"])
def equal_scene(request, dmn, dmt, gpu_lib):
    kind, n, img, dtype = request.param
    tris = scenes.make_mesh(kind, n, dtype=dtype)
    scene = NodeScene(dmn, dmt, gpu_lib, tris, tris, same=True)
    rays = np.concatenate([scenes.make_primary(kind, img, img, dtype=dtype), special_rays(tris, dtype)])
    times = random_times(rays.shape[0], dtype=dtype)
    tracer = NodeTracer(scene, scenes.make_primary(kind, img // 2, img // 2, dtype=dtype), random_times((img // 2) ** 2, 6, dtype),
                        LIGHT[kind], 4)
    yield scene, rays, cuda(rays), cuda(times), tracer
    scene.destroy()


def test_equal_keys_records_are_refit_bounds(equal_scene):
    """Equal keys: both keys of every record are the tree's bounds after refit over prepare_motion_triangles' boxes (the
    tree built from them), bit for bit, and every index is the tree's."""
    scene = equal_scene[0]
    bounds, index, _ = scene.bvh.arrays()
    k0, k1, idx = scene.records()
    ui = np.uint32 if scene.s == "3f" else np.uint64
    want = np.ascontiguousarray(bounds, scene.dtype).view(ui)
    assert (k0[1:].view(ui) == want).all() and (k1[1:].view(ui) == want).all()
    assert (idx[1:] == index.astype(idx.dtype)).all()


@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
def test_equal_keys_equal_motion_call(equal_scene, flags):
    """Equal keys: records, accept-call counts and accept-sequence hashes equal the motion call on the shutter-box tree."""
    scene, rays, d_rays, d_times, _ = equal_scene
    n = rays.shape[0]
    for filt in (0, 1):
        got = scene.run_nodes(NODES, d_rays, d_times, n, filt, flags)
        assert_fields(got, scene.run_nodes(SHUTTER, d_rays, d_times, n, filt, flags), RUN_NAMES, f"equal keys, filter {filt}")
        assert (got[0] != -1).sum() > n // 20


@pytest.mark.parametrize("flags", PATH_FLAGS, ids=PATH_IDS)
def test_equal_keys_equal_motion_paths(equal_scene, flags):
    scene, _, _, _, tracer = equal_scene
    got = tracer(0, flags)
    assert_fields(got, tracer(2, flags), TRACER_NAMES, "equal keys paths")
    assert (got[1] >= 1).all() and got[1].max() >= 4


def partial_keys(tris, seed=0):
    """Part of the mesh static: the triangles whose centre lies below the median x keep their vertices, the others move
    from the deformed mesh at time 0 to the mesh at time 1 (shared vertices of a grid then meet at key 1)"""
    cx = tris.reshape(-1, 3, 3)[:, :, 0].astype(np.float64).mean(axis=1)
    moving = (cx >= np.median(cx))[:, None]
    k0 = np.where(moving, deform(tris, seed, tri_size(tris)), tris)
    return np.ascontiguousarray(k0), tris


def moving_scene(dmn, dmt, api, kind, n, dtype, amplitude=1.0, seed=2, partial=False):
    tris = scenes.make_mesh(kind, n, dtype=dtype)
    if partial:
        k0, k1 = partial_keys(tris, seed)
    else:
        k0, k1 = tris, deform(tris, seed, amplitude * tri_size(tris))
    return tris, NodeScene(dmn, dmt, api, k0, k1)


@pytest.mark.parametrize("kind,dtype,partial", [("soup", np.float32, False), ("grid", np.float32, False), ("soup", np.float64, False),
                                               ("grid", np.float32, True), ("grid", np.float64, True)],
                         ids=["soup-3f", "grid-3f", "soup-3d", "grid-partial-3f", "grid-partial-3d"])
def test_moving_keys_against_motion_call(dmn, dmt, gpu_lib, kind, dtype, partial):
    """Moving keys, random per-ray times (NaN, -1, 2, 0 and 1 among them): robust closest-hit records with canonical
    ties equal the motion call on every ray (both trees hold the closest triangle); robust any-hit agrees on hit or miss;
    a view whose node bounds are all NaN gives the motion-node call's results bit for bit."""
    tris, scene = moving_scene(dmn, dmt, gpu_lib, kind, 200_000, dtype, partial=partial)
    rays = np.concatenate([scenes.make_primary(kind, 500, 500, dtype=dtype), special_rays(tris, dtype)])
    d_rays, n = cuda(rays), rays.shape[0]
    times = random_times(n, dtype=dtype)
    times[::97] = np.array([np.nan, -1.0, 2.0, 0.0, 1.0], dtype)[np.arange(times[::97].shape[0]) % 5]
    d_times = cuda(times)
    for filt in (0, 1):
        got = scene.run_nodes(NODES, d_rays, d_times, n, filt, ROBUST)
        assert_fields(got[:4], scene.run_nodes(SHUTTER, d_rays, d_times, n, filt, ROBUST)[:4], RUN_NAMES[:4], f"robust closest {filt}")
        assert (got[0] != -1).sum() > n // 10
        anyh = scene.run_nodes(NODES, d_rays, d_times, n, filt, ANY | ROBUST)[0]
        assert ((anyh != -1) == (scene.run_nodes(SHUTTER, d_rays, d_times, n, filt, ANY | ROBUST)[0] != -1)).all()
    for flags in MODES:
        assert_fields(scene.run_nodes(NAN_VIEW, d_rays, d_times, n, 0, flags), scene.run_nodes(NODES, d_rays, d_times, n, 0, flags),
                      RUN_NAMES, f"NaN view, flags {flags}")
    scene.destroy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
@pytest.mark.parametrize("flags", MODES, ids=MODE_IDS)
def test_random_times_equal_node_at_per_thread(dmn, dmt, gpu_lib, dtype, flags):
    """Moving keys at random per-ray times: the recording shader's records, accept-call counts and hashes equal one
    thread per ray through traverse_top_down with a three-argument node test applying node_at and the slab test, and a
    triangle_at leaf, with every candidate accepted and with odd ids rejected."""
    for kind in ("soup", "grid"):
        tris, scene = moving_scene(dmn, dmt, gpu_lib, kind, 100_000, dtype)
        rays = np.concatenate([scenes.make_primary(kind, 400, 400, dtype=dtype), special_rays(tris, dtype)])
        d_rays, n = cuda(rays), rays.shape[0]
        times = random_times(n, dtype=dtype)
        times[::97] = np.array([np.nan, -1.0, 2.0, 0.0, 1.0], dtype)[np.arange(times[::97].shape[0]) % 5]
        d_times = cuda(times)
        for filt in (0, 1):
            got = scene.run_nodes(NODES, d_rays, d_times, n, filt, flags)
            assert_fields(got, scene.run_nodes(PER_THREAD, d_rays, d_times, n, filt, flags), RUN_NAMES, f"{kind} filter {filt}")
            assert (got[0] != -1).sum() > n // 10
        scene.destroy()


def test_fast_closest_equals_float64_brute_force(dmn, dmt, gpu_lib):
    """Fast-traversal closest ids of 4000 sampled rays at eight times equal a float64 brute force over the blended
    vertices, with the deforming-mesh test's tolerance (rays whose two best distances are within 1e-4 relative, or whose
    hit is within 1e-4 of an edge, are skipped)."""
    import torch
    tris, scene = moving_scene(dmn, dmt, gpu_lib, "soup", 20_000, np.float32, seed=3)
    rays = scenes.make_primary("soup", 300, 300)
    rng = np.random.default_rng(2)
    sample = rng.permutation(rays.shape[0])[:4000]
    palette = rng.uniform(0, 1, size=8).astype(np.float32)
    which = np.arange(sample.shape[0]) % 8
    ids, t, _, _, _, _ = scene.run_nodes(NODES, cuda(rays[sample]), cuda(palette[which]), sample.shape[0], 0, 0)
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
def test_node_boxes_hold_their_subtrees(dmn, dmt, gpu_lib, dtype):
    """Every node_at box holds triangle_at of every finite triangle of its subtree at 65 uniform times and 64
    full-mantissa random times, for a moving grid, for keys a few ulps apart at 1e4 and for a grid whose one half is
    static while the other moves onto it at time 1; a node that holds nothing is
    +-max at every time; no bound is NaN."""
    tris = scenes.make_mesh("grid", 50_000, dtype=dtype)
    pairs = [moving_keys(tris, seed=4), ulps_keys(tris, seed=5), partial_keys(tris, seed=6)]
    big = np.finfo(dtype).max
    for k0, k1 in pairs:
        scene = NodeScene(dmn, dmt, gpu_lib, k0, k1)
        for tau in [*np.linspace(0.0, 1.0, 65), *rounding_times(64, 11, np.float64)]:
            box, ext = scene.node_at(tau), scene.extent(tau)
            assert not np.isnan(box).any()
            full = ext[:, 0] <= ext[:, 1]
            inside = (box[:, 0::2] <= ext[:, 0::2]) & (ext[:, 1::2] <= box[:, 1::2])
            assert inside[full].all(), (tau, np.nonzero(~inside.all(axis=1) & full)[0][:8])
            assert (box[~full][:, 0::2] == big).all() and (box[~full][:, 1::2] == -big).all()
        scene.destroy()


def test_fewer_triangle_tests(dmn, dmt, gpu_lib):
    """At a motion of four triangle sizes, one thread per ray through the node_at node test counts less than half the
    triangle tests per ray of the shutter-box tree."""
    tris, scene = moving_scene(dmn, dmt, gpu_lib, "soup", 200_000, np.float32, amplitude=4.0)
    rays = scenes.make_primary("soup", 300, 300)
    d_rays, n = cuda(rays), rays.shape[0]
    d_times = cuda(random_times(n))
    (ids, *_), _, tests = scene.run_nodes(PER_THREAD, d_rays, d_times, n, 0, 0, steps=True)
    import torch
    inner = torch.zeros(n, dtype=torch.int32, device="cuda")
    shutter_tests = torch.zeros(n, dtype=torch.int32, device="cuda")
    dmt.dmt_steps3f.argtypes = [P, P, P, SZ, C.c_int, P, P, SZ, P, P, P]
    rc = dmt.dmt_steps3f(C.c_void_p(scene.bvh.handle), ptr(scene.k0), ptr(scene.k1), scene.count, 1, ptr(d_rays), ptr(d_times), n,
                         ptr(inner), ptr(shutter_tests), None)
    assert rc == 0, dmt.dmt_last_error()
    torch.cuda.synchronize()
    assert (ids != -1).sum() > n // 10
    assert tests.mean() < 0.5 * host(shutter_tests).mean(), (tests.mean(), host(shutter_tests).mean())
    scene.destroy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
@pytest.mark.parametrize("flags", PATH_FLAGS, ids=PATH_IDS)
def test_one_launch_equals_wavefront_loop(dmn, dmt, gpu_lib, dtype, flags):
    """One motion-node trace_paths launch equals its wavefront loop of motion-node trace_triangles bit for bit; with
    robust traversal and canonical ties (the shadow step uses only hit or miss) it gives the motion call's radiance."""
    tris, scene = moving_scene(dmn, dmt, gpu_lib, "soup", 100_000, dtype, seed=5)
    primary = scenes.make_primary("soup", 200, 200, dtype=dtype)
    tracer = NodeTracer(scene, primary, random_times(primary.shape[0], 8, dtype), LIGHT["soup"], 3)
    got = tracer(0, flags)
    assert_fields(got, tracer(1, flags), TRACER_NAMES, "one launch vs wavefront")
    if flags == ROBUST:
        assert_fields(got[:1], tracer(2, flags)[:1], TRACER_NAMES[:1], "radiance vs the motion call")
    assert (got[1] >= 1).all() and got[1].max() >= 3
    scene.destroy()


def test_every_ray_and_path_once(dmn, dmt, gpu_lib):
    """finish is called once per ray and once per path at batch sizes around the scheduler's edges and at 1M; nothing
    past n is written; n = 0 launches nothing."""
    import torch
    tris, scene = moving_scene(dmn, dmt, gpu_lib, "soup", 100_000, np.float32, seed=6)
    props = torch.cuda.get_device_properties(0)
    wave = props.multi_processor_count * 9 * 4 * 32
    big = 1_000_007
    rays = np.resize(scenes.make_primary("soup", 1001, 1001), (max(wave + 1, big), 8))
    d_rays, d_times = cuda(rays), cuda(random_times(rays.shape[0]))
    tracer = NodeTracer(scene, rays, random_times(rays.shape[0], 9), LIGHT["soup"], 1)
    guard = 1000
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 4097, wave - 1, wave, wave + 1, big):
        for what in ("rays", "paths"):
            counts = torch.zeros(n + guard, dtype=torch.int32, device="cuda")
            if what == "rays":
                scene.run_nodes(NODES, d_rays, d_times, n, 0, 0, counts=counts)
            else:
                tracer(0, 0, counts=counts, n=n)
            got = host(counts)
            assert (got[:n] == 1).all(), (what, n, np.nonzero(got[:n] != 1)[0][:8])
            assert (got[n:] == 0).all(), (what, n)
    scene.destroy()


def test_errors_leave_tree_usable(dmn, dmt, gpu_lib):
    """A node count other than the tree's and a null motion-node pointer raise invalid_argument, a short workspace
    length_error, each naming the motion-node call; prepare_motion_nodes raises on a wrong triangle count, a null output
    and a short workspace, naming itself; nothing is launched and the tree traces as before."""
    import torch
    tris, scene = moving_scene(dmn, dmt, gpu_lib, "soup", 50_000, np.float32, seed=7)
    rays = scenes.make_primary("soup", 300, 300)
    d_rays, n = cuda(rays), rays.shape[0]
    d_times = cuda(random_times(n))
    first = scene.run_nodes(NODES, d_rays, d_times, n, 0, 0)
    counts = torch.zeros(n, dtype=torch.int32, device="cuda")
    nc = scene.node_count
    with pytest.raises(TypeError, match=rf"trace_triangles \(motion nodes\): motion nodes of {nc - 1} nodes for a tree of {nc} nodes"):
        scene.run_nodes(NODES, d_rays, d_times, n, 0, 0, counts=counts, node_count=nc - 1)
    with pytest.raises(TypeError, match=r"trace_triangles \(motion nodes\): a null motion-node pointer"):
        scene.run_nodes(NODES, d_rays, d_times, n, 0, 0, counts=counts, nodes=False)
    with pytest.raises(ValueError, match=r"trace_triangles \(motion nodes\): a workspace of 7 bytes is too small"):
        scene.run_nodes(NODES, d_rays, d_times, n, 0, 0, counts=counts, ws_bytes=7)
    tracer = NodeTracer(scene, rays, random_times(n, 3), LIGHT["soup"], 2)
    paths = tracer(0, 0)
    with pytest.raises(TypeError, match=r"trace_paths \(motion nodes\): motion nodes of"):
        tracer(0, 0, counts=counts, node_count=nc + 1)
    with pytest.raises(ValueError, match=r"trace_paths \(motion nodes\): a workspace of 7 bytes"):
        tracer(0, 0, counts=counts, ws_bytes=7)
    before = host(scene.nodes)
    with pytest.raises(TypeError, match=r"prepare_motion_nodes: 49999 triangles for a tree of 50000 primitives"):
        scene.prepare_nodes(count=49_999)
    with pytest.raises(TypeError, match=r"prepare_motion_nodes: null keys or motion nodes"):
        scene.prepare_nodes(out=False)
    with pytest.raises(ValueError, match=r"prepare_motion_nodes: a workspace of 7 bytes is too small"):
        scene.prepare_nodes(ws_bytes=7)
    torch.cuda.synchronize()
    assert (host(counts) == 0).all()
    assert (host(scene.nodes) == before).all()
    assert_fields(scene.run_nodes(NODES, d_rays, d_times, n, 0, 0), first, RUN_NAMES, "after the errors")
    assert_fields(tracer(0, 0), paths, TRACER_NAMES, "paths after the errors")
    scene.destroy()


def test_animation_on_one_stream(dmn, dmt, gpu_lib):
    """Four frames on one torch stream, with no synchronisation between the steps: both keys rewritten on the device,
    prepare_motion_nodes on the frame-0 topology, the motion-node trace_triangles.  Each frame equals a fresh
    prepare_motion_nodes and trace on the same topology, bit for bit, and the motion changes the hits."""
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
        scene = NodeScene(dmn, dmt, api, frames[0], frames[1])
        s = C.c_void_p(stream.cuda_stream)
        with torch.cuda.stream(stream):
            for f in range(4):
                scene.k0.copy_(d_keys[f])
                scene.k1.copy_(d_keys[f + 1])
                scene.prepare_nodes(s)
                out = scene.run_nodes(NODES, d_rays, d_times, n, 0, 0, stream=s, sync=False)
                got.append(tuple(x.clone() for x in out))
        stream.synchronize()
        got = [tuple(host(x) for x in f) for f in got]
        for f in range(4):
            scene.k0.copy_(d_keys[f])
            scene.k1.copy_(d_keys[f + 1])
            torch.cuda.synchronize()
            scene.prepare_nodes()
            torch.cuda.synchronize()
            assert_fields(got[f], scene.run_nodes(NODES, d_rays, d_times, n, 0, 0), RUN_NAMES, f"frame {f}")
        scene.destroy()
    finally:
        api.set_stream(None)
    assert all((got[f][0] != -1).sum() > n // 10 for f in range(4))
    assert (got[0][1] != got[1][1]).any()
