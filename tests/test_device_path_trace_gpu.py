"""DeviceView::trace_paths on the GPU (test shaders in tests/device_path_trace_kernels.cu): a path tracer with next-event
shadow segments bit for bit equal to the same shader as a wavefront loop of trace_triangles launches, scripted segments
equal to one thread per segment through DeviceView::intersect, every path started and finished once with its segments,
the errors, and a one-stream torch pipeline."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes

pytestmark = pytest.mark.gpu

P, SZ, U, U32 = C.c_void_p, C.c_size_t, C.c_uint, C.c_uint32
ROBUST, LAST = 2, 4
CLOSEST, OCCLUSION = 1, 2
FLAGS = [0, ROBUST, LAST, ROBUST | LAST]
FLAG_IDS = ["fast-lowest", "robust-lowest", "fast-last", "robust-last"]


@pytest.fixture(scope="module")
def dpt(gpu_lib):
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_path_trace_tests())
    for s in ("3f", "3d"):
        getattr(L, f"dpt_tracer{s}").argtypes = [P, C.c_int, U, SZ, P, P, P, U32, P, P, P, P, P, SZ, P]
        getattr(L, f"dpt_wavefront_bytes{s}").argtypes = [SZ]
        getattr(L, f"dpt_wavefront_bytes{s}").restype = SZ
        getattr(L, f"dpt_record{s}").argtypes = [P, C.c_int, U, SZ, P, P, P, P, P, SZ] + [P] * 10 + [SZ, P, SZ, P]
    L.dpt_last_error.restype = C.c_char_p
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


def check(dpt, rc):
    if rc:
        msg = dpt.dpt_last_error().decode()
        raise {-2: ValueError, -3: TypeError}.get(rc, RuntimeError)(msg)


def sfx(dtype):
    return "3f" if np.dtype(dtype) == np.float32 else "3d"


class Tracer:
    """dpt_tracer over one mesh: the mesh's primary rays (bvh_b200.scenes cameras), a point light beside the camera."""

    def __init__(self, dpt, bvh, tris, kind, size, bounces):
        import torch
        self.dpt, self.bvh, self.bounces = dpt, bvh, bounces
        self.s = sfx(tris.dtype)
        self.primary = cuda(scenes.make_primary(kind, size, size, dtype=tris.dtype))
        self.light = np.asarray(scenes.CAMERAS[kind]["eye"], np.float64).astype(tris.dtype) + np.array([0.25, 0.15, 0.0], tris.dtype)
        self.verts = cuda(tris.reshape(-1))
        self.n = size * size
        self.tdtype = torch.float32 if self.s == "3f" else torch.float64
        self.scratch = torch.empty(getattr(dpt, f"dpt_wavefront_bytes{self.s}")(self.n), dtype=torch.uint8, device="cuda")
        self.ws = torch.empty(8, dtype=torch.uint8, device="cuda")

    def __call__(self, wavefront, flags, stream=None, sync=True):
        import torch
        rad = torch.full((self.n,), float("nan"), dtype=self.tdtype, device="cuda")
        segs = torch.full((self.n,), -1, dtype=torch.int32, device="cuda")
        hashes = torch.zeros(self.n, dtype=torch.int32, device="cuda")
        check(self.dpt, getattr(self.dpt, f"dpt_tracer{self.s}")(
            C.c_void_p(self.bvh.handle), int(wavefront), flags, self.n, ptr(self.primary), self.light.ctypes.data,
            ptr(self.verts), self.bounces, ptr(rad), ptr(segs), ptr(hashes), ptr(self.scratch), ptr(self.ws), 8, stream))
        out = (rad, segs, hashes)
        if not sync:
            return out
        torch.cuda.synchronize()
        return tuple(host(x) for x in out)


SCENES = [("soup", 1_000_000, np.float32), ("grid", 1_000_000, np.float32), ("soup", 1_000_000, np.float64),
          ("grid", 1_000_000, np.float64)]


@pytest.fixture(scope="module", params=SCENES, ids=["c2-soup-3f", "c2-grid-3f", "c2-soup-3d", "c2-grid-3d"])
def mesh(request, gpu_lib):
    kind, n, dtype = request.param
    tris = scenes.make_mesh(kind, n, dtype=dtype)
    bvh = gpu_lib.Bvh.build_triangles(tris)
    yield kind, tris, bvh
    bvh.destroy()


@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
def test_path_tracer_equals_wavefront_loop(dpt, mesh, flags):
    """A diffuse path tracer with next-event shadow segments and 4 bounces: per path the radiance bits, the segment count
    and the hash of the segment records of one trace_paths call equal those of the same shader run as a wavefront loop
    of trace_triangles launches with its state in arrays."""
    kind, tris, bvh = mesh
    tracer = Tracer(dpt, bvh, tris, kind, 700 if tris.dtype == np.float32 else 400, 4)
    got = tracer(False, flags)
    want = tracer(True, flags)
    for name, a, b in zip(("radiance", "segments", "hashes"), got, want):
        same = bits(a) == bits(b)
        assert same.all(), f"{name} differs at {np.nonzero(~same)[0][:8]}"
    rad, segs, _ = got
    assert (segs >= 1).all() and segs.max() >= 6            # every path traced; some bounced more than twice
    assert (segs % 2 == 0).any() and (segs % 2 == 1).any()
    assert np.isfinite(rad).all() and (rad > 0).mean() > 0.2


def scripted(n, ray_count, rng, max_len=64, lengths=None):
    """Scripted paths: lengths, offsets, per segment the ray index and the kind (mixed in every warp)."""
    if lengths is None:
        lengths = rng.integers(0, max_len + 1, n).astype(np.uint32)
    offsets = np.zeros(n, np.uint64)
    offsets[1:] = np.cumsum(lengths.astype(np.uint64))[:-1]
    total = int(lengths.astype(np.int64).sum())
    seg_ray = rng.integers(0, ray_count, total).astype(np.uint32)
    seg_kind = rng.choice(np.array([CLOSEST, OCCLUSION], np.uint8), total)
    return lengths, offsets, seg_ray, seg_kind, total


class Record:
    """dpt_record over one tree and a pool of device-resident rays."""

    def __init__(self, dpt, bvh, dtype):
        import torch
        self.dpt, self.bvh, self.s = dpt, bvh, sfx(dtype)
        self.tdtype = torch.float32 if self.s == "3f" else torch.float64
        self.ws = torch.empty(64, dtype=torch.uint8, device="cuda")

    def __call__(self, d_rays, script, flags, per_thread=False, outputs=True, counts=False, ws_bytes=8, depth=0, stream=None,
                 sync=True):
        import torch
        lengths, offsets, seg_ray, seg_kind, total = script
        n = lengths.shape[0]
        d = [cuda(x) for x in (offsets, lengths, seg_ray, seg_kind)]
        m = max(total, 1)
        out = (torch.full((m,), -2, dtype=torch.int32, device="cuda"),) + tuple(
            torch.empty(m, dtype=self.tdtype, device="cuda") for _ in range(3)) + (
            torch.empty(m, dtype=torch.int32, device="cuda"), torch.empty(m, dtype=torch.int64, device="cuda"))
        if not outputs:
            out = (None,) * 6
        per_path = (torch.zeros(n + 1, dtype=torch.int32, device="cuda"), torch.zeros(n + 1, dtype=torch.int32, device="cuda"),
                    torch.full((n + 1,), -1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda"))
        if not counts:
            per_path = (None,) * 4
        check(self.dpt, getattr(self.dpt, f"dpt_record{self.s}")(
            C.c_void_p(self.bvh.handle), int(per_thread), flags, n, ptr(d_rays), *[ptr(x) for x in d], total,
            *[ptr(x) for x in out], *[ptr(x) for x in per_path], depth, ptr(self.ws), ws_bytes, stream))
        if not sync:
            return out, per_path
        torch.cuda.synchronize()
        return tuple(None if x is None else host(x) for x in out), tuple(None if x is None else host(x) for x in per_path)


def special_rays(tris, dtype):
    from tests.test_device_api_host import extra_rays
    return extra_rays(tris, dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
def test_segments_equal_per_thread(dpt, gpu_lib, dtype, flags):
    """Scripted paths of 0 to 64 segments in one batch, Closest and Occlusion mixed within every warp, over primary,
    scattered, NaN-interval and axis-parallel rays: per segment the record, the accept-call count and the hash of the
    accept sequence equal one thread per segment through DeviceView::intersect; next always receives the scripted ray."""
    tris = scenes.make_mesh("soup", 200_000, dtype=dtype)
    rng = np.random.default_rng(11)
    primary = scenes.make_primary("soup", 300, 300, dtype=dtype)
    scattered = primary[rng.permutation(primary.shape[0])[:20_000]].copy()
    scattered[:, 3:6] = rng.normal(size=(scattered.shape[0], 3))
    scattered[:, 0:3] = rng.random((scattered.shape[0], 3))
    rays = np.concatenate([primary, scattered, special_rays(tris, dtype)]).astype(dtype)
    bvh = gpu_lib.Bvh.build_triangles(tris)
    run, d_rays = Record(dpt, bvh, dtype), cuda(rays)
    script = scripted(6000, rays.shape[0], rng)
    got, (starts, finishes, done, bad) = run(d_rays, script, flags, counts=True)
    want, _ = run(d_rays, script, flags, per_thread=True)
    for name, a, b in zip(("ids", "t", "u", "v", "calls", "hashes"), got, want):
        same = bits(a) == bits(b) if a.dtype.kind == "f" else a == b
        assert same.all(), f"{name} differs at {np.nonzero(~same)[0][:8]}"
    lengths = script[0]
    n = lengths.shape[0]
    assert (starts[:n] == 1).all() and (finishes[:n] == 1).all() and (done[:n] == lengths.astype(np.int32)).all()
    assert bad[0] == 0
    assert (lengths == 0).any() and (lengths == 64).any()
    hit = got[0] != -1
    assert hit.mean() > 0.1 and (got[4] > 0).mean() > 0.1
    bvh.destroy()


def test_every_path_once(dpt, gpu_lib):
    """start and finish once per path, with the scripted segment count, for batch sizes around the scheduler's edges and
    a batch of 1M paths; nothing past n is touched; n = 0 launches nothing."""
    import torch
    tris = scenes.make_mesh("soup", 100_000)
    rays = scenes.make_primary("soup", 300, 300)
    bvh = gpu_lib.Bvh.build_triangles(tris)
    run, d_rays = Record(dpt, bvh, np.float32), cuda(rays)
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
    bvh.destroy()


def test_errors_leave_tree_usable(dpt, gpu_lib):
    """A short workspace and a tree too deep for the shared-memory stack raise length_error, a view without triangles
    invalid_argument; afterwards the tree traces as before."""
    import torch
    api = gpu_lib
    tris = scenes.make_mesh("soup", 100_000)
    rays = scenes.make_primary("soup", 200, 200)
    bvh = api.Bvh.build_triangles(tris)
    run, d_rays = Record(dpt, bvh, np.float32), cuda(rays)
    script = scripted(2000, rays.shape[0], np.random.default_rng(8), max_len=8)
    first, _ = run(d_rays, script, 0)
    with pytest.raises(ValueError, match="workspace of 7 bytes is too small"):
        run(d_rays, script, 0, ws_bytes=7)
    with pytest.raises(ValueError, match="tree of depth 400"):
        run(d_rays, script, 0, depth=400)
    centres = tris.reshape(-1, 3, 3).mean(axis=1).astype(np.float32)
    boxes = np.concatenate([tris.reshape(-1, 3, 3).min(axis=1), tris.reshape(-1, 3, 3).max(axis=1)], axis=1).astype(np.float32)
    d_boxes, d_centres = cuda(boxes), cuda(centres)
    torch.cuda.synchronize()
    box_bvh = api.Bvh.build_boxes(d_boxes.data_ptr(), d_centres.data_ptr(), count=centres.shape[0], dtype=np.float32,
                                  flags=api.DEVICE_POINTERS)
    with pytest.raises(TypeError, match="no triangles"):
        Record(dpt, box_bvh, np.float32)(d_rays, script, 0)
    box_bvh.destroy()
    second, (starts, finishes, done, _) = run(d_rays, script, 0, counts=True)
    for a, b in zip(first, second):
        assert (bits(a) == bits(b)).all() if a.dtype.kind == "f" else (a == b).all()
    assert (starts[:-1] == 1).all() and (finishes[:-1] == 1).all()
    bvh.destroy()


def test_build_trace_refit_trace_on_one_stream(dpt, gpu_lib):
    """build_triangles, trace_paths, refit_triangles with moved vertices, trace_paths again: one torch stream, no
    synchronisation between the steps.  Both results equal the same steps run synchronously."""
    import torch
    api = gpu_lib
    tris = scenes.make_mesh("soup", 200_000)
    moved = (tris + 0.01 * (np.random.default_rng(4).random(tris.shape) - 0.5)).astype(np.float32)
    torch.cuda.synchronize()

    def frames(sync):
        stream = torch.cuda.Stream()
        api.set_stream(stream.cuda_stream)
        out = []
        try:
            with torch.cuda.stream(stream):
                d_tris, d_moved = cuda(tris), cuda(moved)
                bvh = api.Bvh.build_triangles(d_tris.data_ptr(), count=tris.shape[0], dtype=np.float32, flags=api.DEVICE_POINTERS)
                tracer = Tracer(dpt, bvh, tris, "soup", 400, 3)
                for frame in range(2):
                    if frame:
                        bvh.refit_triangles(d_moved.data_ptr(), api.DEVICE_POINTERS)
                        tracer.verts = d_moved
                        if sync:
                            stream.synchronize()
                    res = tracer(False, 0, stream=C.c_void_p(stream.cuda_stream), sync=False)
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
            assert (bits(x) == bits(y)).all()
    assert (fast[0][2] != fast[1][2]).any(), "moving the triangles changed no segment record"
