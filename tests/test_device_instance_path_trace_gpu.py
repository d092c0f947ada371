"""DeviceView::trace_instance_paths on the GPU (test shaders in tests/device_instance_path_trace_kernels.cu; instance
records from tests/device_instance_trace_kernels.cu): a path tracer with next-event shadow segments under one identity
instance bit for bit equal to trace_paths on the mesh, over 60 placed copies equal to the same shader as a wavefront
loop of trace_instances launches, scripted segments equal to one thread per segment nesting DeviceView::intersect by
hand, every path started and finished once, the errors, and a rigid animation on one torch stream."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes
from tests.test_device_instance_trace_gpu import Scene, dit, many_scene, placements, special_rays, world_rays  # noqa: F401
from tests.test_device_path_trace_gpu import scripted

pytestmark = pytest.mark.gpu

P, SZ, U, U32 = C.c_void_p, C.c_size_t, C.c_uint, C.c_uint32
ROBUST, LAST = 2, 4
FLAGS = [0, ROBUST, LAST, ROBUST | LAST]
FLAG_IDS = ["fast-lowest", "robust-lowest", "fast-last", "robust-last"]
ONE_LAUNCH, WAVEFRONT, MESH = 0, 1, 2
IDENTITY = np.array([[1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]], np.float64)


@pytest.fixture(scope="module")
def dipt(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_instance_path_trace_tests())
    for s in ("3f", "3d"):
        getattr(L, f"dipt_tracer{s}").argtypes = [P, P, SZ, SZ, C.c_int, U, SZ, P, P, P, U32, P, P, P, P, P, SZ, P]
        getattr(L, f"dipt_wavefront_bytes{s}").argtypes = [SZ]
        getattr(L, f"dipt_wavefront_bytes{s}").restype = SZ
        getattr(L, f"dipt_record{s}").argtypes = [P, P, SZ, SZ, C.c_int, C.c_int, U, SZ, P, P, P, P, P, SZ] + [P] * 11 + [P, SZ, P]
    L.dipt_last_error.restype = C.c_char_p
    return L


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def bits(a):
    return a.view(np.uint32 if a.dtype.itemsize == 4 else np.uint64)


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def check(lib, rc):
    if rc:
        msg = lib.dipt_last_error().decode()
        raise {-2: ValueError, -3: TypeError}.get(rc, RuntimeError)(msg)


def assert_same(got, want, names, what=""):
    for name, a, b in zip(names, got, want):
        same = bits(a) == bits(b) if a.dtype.kind == "f" else a == b
        assert same.all(), f"{what} {name} differs at {np.nonzero(~same)[0][:8]}"


class Tracer:
    """dipt_tracer over a Scene: primary rays, a point light, and each instance's mesh vertices."""

    def __init__(self, dipt, scene, primary, light, mesh_tris, bounces):
        import torch
        self.dipt, self.scene, self.bounces = dipt, scene, bounces
        self.primary = cuda(primary)
        self.n = primary.shape[0]
        self.light = np.asarray(light, scene.dtype)
        self.d_verts = [cuda(np.ascontiguousarray(t, scene.dtype).reshape(-1)) for t in mesh_tris]
        self.verts = torch.tensor([self.d_verts[k].data_ptr() for k in scene.mesh_of], dtype=torch.int64, device="cuda")
        self.scratch = torch.empty(getattr(dipt, f"dipt_wavefront_bytes{scene.s}")(self.n), dtype=torch.uint8, device="cuda")
        self.ws = torch.empty(8, dtype=torch.uint8, device="cuda")

    def __call__(self, mode, flags, handle=None, stream=None, sync=True):
        import torch
        sc = self.scene
        rad = torch.full((self.n,), float("nan"), dtype=sc.tdtype, device="cuda")
        segs = torch.full((self.n,), -1, dtype=torch.int32, device="cuda")
        hashes = torch.zeros(self.n, dtype=torch.int32, device="cuda")
        check(self.dipt, getattr(self.dipt, f"dipt_tracer{sc.s}")(
            C.c_void_p(handle if handle is not None else sc.top.handle), ptr(sc.records), sc.count, sc.max_depth, mode, flags, self.n,
            ptr(self.primary), self.light.ctypes.data, ptr(self.verts), self.bounces, ptr(rad), ptr(segs), ptr(hashes),
            ptr(self.scratch), ptr(self.ws), 8, stream))
        out = (rad, segs, hashes)
        if not sync:
            return out
        torch.cuda.synchronize()
        return tuple(host(x) for x in out)


TRACER_NAMES = ("radiance", "segments", "hashes")


def placed_scene(dit, api, meshes, mesh_of, mats, dtype):
    scene = Scene(dit, api, meshes, mesh_of, mats, dtype)
    scene.mesh_of = list(mesh_of)
    return scene


SCENES = [("soup", 1_000_000, 700, np.float32), ("grid", 1_000_000, 700, np.float32), ("soup", 200_000, 400, np.float64)]


@pytest.fixture(scope="module", params=SCENES, ids=["c2-soup-3f", "c2-grid-3f", "soup-3d"])
def identity_scene(request, dipt, dit, gpu_lib):
    kind, n, img, dtype = request.param
    tris = scenes.make_mesh(kind, n, dtype=dtype)
    scene = placed_scene(dit, gpu_lib, [tris], [0], IDENTITY, dtype)
    light = np.asarray(scenes.CAMERAS[kind]["eye"], np.float64) + np.array([0.25, 0.15, 0.0])
    tracer = Tracer(dipt, scene, scenes.make_primary(kind, img, img, dtype=dtype), light, [tris], 4)
    yield scene, tracer
    scene.destroy()


@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
def test_identity_instance_equals_trace_paths(dipt, identity_scene, flags):
    """One identity instance under a top tree of one leaf: per path the radiance bits, segment count and hash of the
    segment records and instances equal trace_paths on the mesh, bit for bit."""
    scene, tracer = identity_scene
    got = tracer(ONE_LAUNCH, flags)
    want = tracer(MESH, flags, handle=scene.meshes[0].handle)
    assert_same(got, want, TRACER_NAMES, "identity")
    rad, segs, _ = got
    assert (segs >= 1).all() and segs.max() >= 6
    assert (segs % 2 == 0).any() and (segs % 2 == 1).any()
    assert np.isfinite(rad).all() and (rad > 0).mean() > 0.2


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
def test_one_launch_equals_wavefront_loop(dipt, dit, gpu_lib, dtype, flags):
    """60 rotated and scaled copies of two meshes, one of them singular: one trace_instance_paths call equals the same
    shader run as a wavefront loop of trace_instances launches, bit for bit."""
    scene, meshes, mesh_of, mats = many_scene(dit, gpu_lib, dtype, count=60, singular=(7,))
    scene.mesh_of = list(mesh_of)
    primary = world_rays(mats, 300, 300, dtype)
    centre = mats.reshape(-1, 3, 4)[:, :, 3].mean(axis=0)
    tracer = Tracer(dipt, scene, primary, centre + np.array([0.3, -0.2, -4.0]), meshes, 4)
    got = tracer(ONE_LAUNCH, flags)
    want = tracer(WAVEFRONT, flags)
    assert_same(got, want, TRACER_NAMES, "one launch vs wavefront")
    rad, segs, _ = got
    assert (segs >= 1).all() and segs.max() >= 4 and (segs > 1).mean() > 0.1
    assert np.isfinite(rad).all()
    scene.destroy()


class Record:
    """dipt_record over a Scene and a pool of device-resident rays."""

    def __init__(self, dipt, scene):
        import torch
        self.dipt, self.scene = dipt, scene
        self.ws = torch.empty(64, dtype=torch.uint8, device="cuda")

    def __call__(self, d_rays, script, flags, filt=0, per_thread=False, outputs=True, counts=False, ws_bytes=8, count=None,
                 max_depth=None, stream=None, sync=True, into=None):
        """into: (out, per_path) tensors of an earlier call's shape to write to, instead of new ones"""
        import torch
        sc = self.scene
        lengths, offsets, seg_ray, seg_kind, total = script
        n = lengths.shape[0]
        d = [cuda(x) for x in (offsets, lengths, seg_ray, seg_kind)]
        m = max(total, 1)
        out = (torch.full((m,), -2, dtype=torch.int32, device="cuda"),) + tuple(
            torch.empty(m, dtype=sc.tdtype, device="cuda") for _ in range(3)) + tuple(
            torch.full((m,), -2, dtype=torch.int32, device="cuda") for _ in range(2)) + (torch.empty(m, dtype=torch.int64, device="cuda"),)
        if not outputs:
            out = (None,) * 7
        per_path = (torch.zeros(n + 1, dtype=torch.int32, device="cuda"), torch.zeros(n + 1, dtype=torch.int32, device="cuda"),
                    torch.full((n + 1,), -1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda"))
        if not counts:
            per_path = (None,) * 4
        if into is not None:
            out, per_path = into
        check(self.dipt, getattr(self.dipt, f"dipt_record{sc.s}")(
            C.c_void_p(sc.top.handle), ptr(sc.records), sc.count if count is None else count,
            sc.max_depth if max_depth is None else max_depth, int(per_thread), filt, flags, n, ptr(d_rays), *[ptr(x) for x in d], total,
            *[ptr(x) for x in out], *[ptr(x) for x in per_path], ptr(self.ws), ws_bytes, stream))
        if not sync:
            return out, per_path
        torch.cuda.synchronize()
        return tuple(None if x is None else host(x) for x in out), tuple(None if x is None else host(x) for x in per_path)


RECORD_NAMES = ("ids", "t", "u", "v", "inst", "calls", "hashes")


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
def test_segments_equal_per_thread(dipt, dit, gpu_lib, dtype, flags):
    """Scripted paths of 0 to 64 segments, Closest and Occlusion mixed within every warp, over world, scattered, NaN-interval
    and axis-parallel rays through 60 placed copies (two singular): per segment the record, instance, accept-call count and
    accept-sequence hash equal one thread per segment nesting DeviceView::intersect by hand, with every candidate accepted
    and with odd instances rejected; next always receives the scripted world ray."""
    scene, meshes, _, mats = many_scene(dit, gpu_lib, dtype, count=60, singular=(5, 40))
    rng = np.random.default_rng(17)
    primary = world_rays(mats, 200, 200, dtype)
    scattered = primary[rng.permutation(primary.shape[0])[:10_000]].copy()
    scattered[:, 3:6] = rng.normal(size=(scattered.shape[0], 3))
    scattered[:, 2] = rng.uniform(-1.0, 1.0, scattered.shape[0])
    rays = np.concatenate([primary, scattered, special_rays(meshes[0], dtype)]).astype(dtype)
    d_rays = cuda(rays)
    run = Record(dipt, scene)
    script = scripted(6000, rays.shape[0], rng)
    for filt in (0, 1):
        got, (starts, finishes, done, bad) = run(d_rays, script, flags, filt=filt, counts=True)
        want, _ = run(d_rays, script, flags, filt=filt, per_thread=True)
        assert_same(got, want, RECORD_NAMES, f"filter {filt}")
        lengths = script[0]
        n = lengths.shape[0]
        assert (starts[:n] == 1).all() and (finishes[:n] == 1).all() and (done[:n] == lengths.astype(np.int32)).all()
        assert bad[0] == 0
        hit = got[0] != -1
        assert hit.mean() > 0.1 and (got[5] > 0).mean() > 0.1
        assert not np.isin(got[4][hit], (5, 40)).any()
        if filt == 1:
            assert ((got[4][hit] & 1) == 0).all()
        else:
            assert len(np.unique(got[4][hit])) > 30
    scene.destroy()


def test_every_path_once(dipt, dit, gpu_lib):
    """start and finish once per path, with the scripted segment count, at batch sizes around the scheduler's edges and
    at 1M paths; nothing past n is touched; n = 0 launches nothing."""
    import torch
    scene, _, _, mats = many_scene(dit, gpu_lib, np.float32, count=16)
    rays = world_rays(mats, 300, 300, np.float32)
    run, d_rays = Record(dipt, scene), cuda(rays)
    rng = np.random.default_rng(3)
    props = torch.cuda.get_device_properties(0)
    wave = props.multi_processor_count * 9 * 4 * 32           # one resident wave of warps (9 blocks of 4 warps per SM), in paths
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 4097, wave - 1, wave, wave + 1, 1_000_003):
        lengths = rng.integers(0, 5, n).astype(np.uint32)
        _, (starts, finishes, done, bad) = run(d_rays, scripted(n, rays.shape[0], rng, lengths=lengths), 0, outputs=False,
                                               counts=True)
        assert (starts[:n] == 1).all() and (finishes[:n] == 1).all(), n
        assert (done[:n] == lengths.astype(np.int32)).all(), n
        assert starts[n] == 0 and finishes[n] == 0 and done[n] == -1 and bad[0] == 0, n
    scene.destroy()


def test_errors_leave_trees_usable(dipt, dit, gpu_lib):
    """A record count other than the top tree's raises invalid_argument; a short workspace and a bottom depth that
    overflows the 200 KB stack raise length_error; none launches anything, and both trees trace as before afterwards."""
    import torch
    scene, _, _, mats = many_scene(dit, gpu_lib, np.float32, count=20)
    rays = world_rays(mats, 200, 200, np.float32)
    run, d_rays = Record(dipt, scene), cuda(rays)
    script = scripted(3000, rays.shape[0], np.random.default_rng(8), max_len=8)
    first, _ = run(d_rays, script, 0)
    n = script[0].shape[0]
    # the failing calls write into these: records at their fill value (-2), counters at 0, done at -1
    into = run(d_rays, script, 0, counts=True, sync=False)
    torch.cuda.synchronize()
    for x in into[0] + into[1]:
        x.fill_(-2 if x is into[0][0] else -1 if x is into[1][2] else 0)
    for kwargs, exc, match in (({"count": 19}, TypeError, "19 instance records for a top tree of 20"),
                               ({"ws_bytes": 7}, ValueError, "workspace of 7 bytes is too small"),
                               ({"max_depth": 400}, ValueError, "shared-memory stack")):
        with pytest.raises(exc, match=match):
            run(d_rays, script, 0, counts=True, into=into, **kwargs)
    torch.cuda.synchronize()
    out, (starts, finishes, done, bad) = (tuple(host(x) for x in into[0]), tuple(host(x) for x in into[1]))
    assert (out[0] == -2).all() and (starts == 0).all() and (finishes == 0).all() and (done == -1).all() and bad[0] == 0
    second, (starts, finishes, done, _) = run(d_rays, script, 0, counts=True)
    assert_same(second, first, RECORD_NAMES, "after the errors")
    assert (starts[:n] == 1).all() and (finishes[:n] == 1).all()
    want, _ = run(d_rays, script, 0, per_thread=True)
    assert_same(second, want, RECORD_NAMES, "per-thread after the errors")
    scene.destroy()


def test_rigid_animation_on_one_stream(dipt, dit, gpu_lib):
    """Four frames on one torch stream, with no synchronisation between the steps: new matrices written on the device,
    prepare_instances, refit_boxes of the top tree, trace_instance_paths.  Each frame equals the same frame run with the
    host synchronised between the steps, and the motion changes the records."""
    import torch
    api = gpu_lib
    count = 30
    meshes = [scenes.make_mesh("soup", 20_000), scenes.make_mesh("grid", 20_000)]
    mesh_of = np.arange(count) % 2
    frames = [placements(count, seed=20 + f) for f in range(4)]
    rays = world_rays(frames[0], 300, 300, np.float32)
    d_rays = cuda(rays)
    scene = Scene(dit, api, meshes, mesh_of, frames[0], np.float32)
    script = scripted(20_000, rays.shape[0], np.random.default_rng(5), max_len=6)
    run = Record(dipt, scene)
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
                check_dit(dit, dit.dit_set_matrices3f(ptr(scene.records), ptr(d_frames[f]), count, s))
                scene.prepare(s)
                top.refit_boxes(scene.boxes.data_ptr(), api.DEVICE_POINTERS)
                out, _ = run(d_rays, script, 0, stream=s, sync=False)
                got.append(tuple(x.clone() for x in out))
        stream.synchronize()
        got = [tuple(host(x) for x in f) for f in got]
        for f in range(4):
            check_dit(dit, dit.dit_set_matrices3f(ptr(scene.records), ptr(d_frames[f]), count, s))
            stream.synchronize()
            scene.prepare(s)
            stream.synchronize()
            top.refit_boxes(scene.boxes.data_ptr(), api.DEVICE_POINTERS)
            stream.synchronize()
            want, _ = run(d_rays, script, 0, stream=s)
            assert_same(got[f], want, RECORD_NAMES, f"frame {f}")
    finally:
        api.set_stream(None)
    assert all((got[f][0] != -1).mean() > 0.1 for f in range(4))
    assert (got[0][1] != got[1][1]).any()
    scene.destroy()


def check_dit(dit, rc):
    if rc:
        raise RuntimeError(dit.dit_last_error().decode())
