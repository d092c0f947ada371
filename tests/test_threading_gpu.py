"""The library from several host threads at once (INTEGRATION.md §2 "Threading"): one handle per thread, deep trees whose
traversal stacks need different amounts of shared memory traced at once (bvhNN_intersect_rays and DeviceView::trace), many
threads on one handle, the per-thread error, device and stream, and bvh_cuda_trim during work.

Every scenario first runs its calls serially on the main thread; the threads must then give the same bytes.  ctypes
releases the GIL around foreign calls, so the library's calls really overlap.  Every loop has a fixed count."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

from bvh_b200 import scenes
from tests.test_device_trace_gpu import LEAF_TRI, Run, cuda, dtr, sfx  # noqa: F401 (dtr: a fixture)

pytestmark = pytest.mark.gpu

TIMEOUT = 300.0                     # seconds for all threads of one run_threads call


def run_threads(fns, timeout=TIMEOUT):
    """Calls fns[k]() on thread k, all released at once by a barrier, and returns their results in order.  A thread that
    raised fails the test with every thread's error; a thread still running after `timeout` seconds fails it too."""
    barrier = threading.Barrier(len(fns))
    results, errors = [None] * len(fns), [None] * len(fns)

    def body(k):
        try:
            barrier.wait(timeout)
            results[k] = fns[k]()
        except BaseException as e:          # (reported below, on the main thread)
            errors[k] = e

    threads = [threading.Thread(target=body, args=(k,), daemon=True) for k in range(len(fns))]
    for t in threads:
        t.start()
    deadline = time.monotonic() + timeout
    for t in threads:
        t.join(max(0.0, deadline - time.monotonic()))
    hung = [k for k, t in enumerate(threads) if t.is_alive()]
    if hung:
        pytest.fail(f"threads {hung} of {len(fns)} still running after {timeout:.0f} s")
    failed = [f"thread {k}: {type(e).__name__}: {e}" for k, e in enumerate(errors) if e is not None]
    if failed:
        raise AssertionError(f"{len(failed)} of {len(fns)} threads failed:\n" + "\n".join(failed))
    return results


def assert_same(got, want, what):
    """Bit for bit: the bytes of every array (structured hit records included), recursively through lists and tuples."""
    if isinstance(want, (list, tuple)):
        assert isinstance(got, (list, tuple)) and len(got) == len(want), what
        for k, (g, w) in enumerate(zip(got, want)):
            assert_same(g, w, f"{what}[{k}]")
        return
    g, w = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert g.dtype == w.dtype and g.shape == w.shape, f"{what}: {g.dtype}{g.shape} vs {w.dtype}{w.shape}"
    same = g.reshape(-1).view(np.uint8) == w.reshape(-1).view(np.uint8)
    assert same.all(), f"{what}: {int((~same).sum())} bytes differ"


# ---- a. one handle per thread, private streams --------------------------------------------------------------------
MESHES = [("soup", 20_000, np.float32, "low"), ("grid", 300_000, np.float32, "high"), ("soup", 150_000, np.float64, "high"),
          ("grid", 50_000, np.float64, "low"), ("soup", 300_000, np.float32, "low"), ("grid", 100_000, np.float32, "high"),
          ("soup", 60_000, np.float64, "low")]


def mesh_sequence(api, kind, n, dtype, quality):
    """Build, download the tree, trace closest-hit, any-hit and robust rays from host arrays, move the vertices, refit,
    trace again and download the refitted tree."""
    tris = scenes.make_mesh(kind, n, dtype=dtype)
    rays = scenes.make_primary(kind, 192, 192, dtype=dtype)
    moved = (tris * dtype(1.01) + dtype(0.003)).astype(dtype)
    bvh = api.Bvh.build_triangles(tris, quality=quality)
    try:
        out = [bvh.arrays()]
        out += [bvh.intersect_rays(rays, flags=f) for f in (0, api.ANY_HIT, api.ROBUST)]
        bvh.refit_triangles(moved)
        out += [bvh.intersect_rays(rays), bvh.arrays()]
    finally:
        bvh.destroy()
    return out


def test_one_handle_per_thread(gpu_lib):
    """Seven threads, each with its own mesh (soup and grid, float and double, 20k to 300k triangles, low and high
    quality) on a handle of its own: every hit array and every downloaded tree equals the serial run."""
    api = gpu_lib
    want = [mesh_sequence(api, *m) for m in MESHES]
    got = run_threads([lambda m=m: mesh_sequence(api, *m) for m in MESHES])
    for m, g, w in zip(MESHES, got, want):
        assert_same(g, w, f"{m[0]} {m[1]} {np.dtype(m[2]).name} {m[3]}")
    assert (want[0][1]["prim_id"] != api.INVALID_ID).any()


# ---- b. traversal stacks of different sizes above 48 KB, traced at once ------------------------------------------------
# Chains of one-primitive leaves under unit-cube boxes: every ray that enters the cube tests every triangle.  Stack per
# block: (depth + 2) * 128 entries of 4 (float) or 8 (double) bytes, 61 to 152 KB here.
CHAINS = [(120, np.float32), (200, np.float32), (300, np.float32), (60, np.float64), (150, np.float64)]
POOL = 1024                          # rays per chain; each call traces a slice of them
CALLS = 200


def chain_formats(dtype):
    """The struct formats of the reference's serialized tree for `dtype`: the header (node and primitive counts), one node
    (six bounds and the index first_id << 4 | count) and one primitive id.  Float trees store u32 counts, indices and ids;
    double trees u64 ones."""
    return ("<II", "<6fI", "I") if np.dtype(dtype) == np.float32 else ("<QQ", "<6dQ", "Q")


def save_chain(path, inner, dtype):
    """A chain of `inner` inner nodes under unit-cube boxes in the serialized format of chain_formats: inner node k is node
    2k, its left child 2k + 1 is a one-primitive leaf and its right child 2k + 2 is the next inner node (the last one a
    leaf).  (tests/test_device_trace_gpu.py writes the float form of the same chain.)"""
    import struct
    head, node, prim_id = chain_formats(dtype)
    nodes, prim = [], 0
    for k in range(inner):
        nodes.append(((2 * k + 1) << 4) | 0)
        nodes.append((prim << 4) | 1)
        prim += 1
    nodes.append((prim << 4) | 1)
    prim += 1
    with open(path, "wb") as f:
        f.write(struct.pack(head, len(nodes), prim))
        for index in nodes:
            f.write(struct.pack(node, 0, 1, 0, 1, 0, 1, index))
        f.write(struct.pack(f"<{prim}{prim_id}", *range(prim)))


def load_chain(api, tmp_path, depth, dtype):
    """A loaded chain tree whose reported depth is `depth`."""
    path = tmp_path / f"chain{depth}{sfx(dtype)}.bvh"
    save_chain(path, depth, dtype)
    bvh = api.Bvh.load(str(path), dtype=dtype)
    if bvh.depth != depth:                              # (whether the root counts)
        inner = 2 * depth - bvh.depth
        bvh.destroy()
        save_chain(path, inner, dtype)
        bvh = api.Bvh.load(str(path), dtype=dtype)
    assert bvh.depth == depth
    return bvh


@pytest.fixture(scope="module")
def chains(gpu_lib, oracle, tmp_path_factory):
    """Per chain: the loaded handle with one triangle per leaf inside the unit cube, a pool of rays and their brute-force
    closest hits."""
    tmp = tmp_path_factory.mktemp("chains")
    out = []
    for k, (depth, dtype) in enumerate(CHAINS):
        bvh = load_chain(gpu_lib, tmp, depth, dtype)
        tris = (0.15 + 0.7 * scenes.soup(bvh.prim_count, seed=100 + k, dtype=np.float64)).astype(dtype)
        assert (tris > 0).all() and (tris < 1).all()
        bvh.set_triangles(tris)
        rng = np.random.default_rng(200 + k)
        org = np.concatenate([rng.random((POOL, 2)), np.full((POOL, 1), -0.5)], axis=1)
        rays = np.zeros((POOL, 8), dtype)
        rays[:, :3], rays[:, 3:6], rays[:, 6], rays[:, 7] = org, rng.random((POOL, 3)) - org, 0, np.inf
        bf = oracle.brute_force(tris, rays)
        assert (bf[0] != gpu_lib.INVALID_ID).sum() > POOL // 10
        out.append((bvh, tris, rays, bf))
    yield out
    for bvh, *_ in out:
        bvh.destroy()


def chain_calls(api, k):
    """The fixed calls of chain k: (first ray, ray count, flags, stats), cycling through the default kernel, the simple
    kernel, the TMA kernel and the stats kernel."""
    rng = np.random.default_rng(300 + k)
    modes = [(0, False), (api.KERNEL_SIMPLE, False), (api.KERNEL_TMA, False), (0, True)]
    calls = []
    for c in range(CALLS):
        n = int(rng.integers(64, POOL + 1))
        calls.append((int(rng.integers(0, POOL - n + 1)), n) + modes[c % len(modes)])
    return calls


def trace_chain(api, chain, calls):
    bvh, _, rays, _ = chain
    out = []
    for first, n, flags, stats in calls:
        res = bvh.intersect_rays(rays[first:first + n], flags=flags, stats=stats)
        out.append(list(res) if stats else [res])
    return out


def test_deep_stacks_batched(gpu_lib, chains):
    """Five chain trees (float depth 120, 200, 300; double depth 60, 150), one thread each, 200 host-array calls of 64 to
    1024 rays through four kernels: every call succeeds, equals brute force and equals the serial run, stats included."""
    api = gpu_lib
    calls = [chain_calls(api, k) for k in range(len(chains))]
    want = [trace_chain(api, ch, cs) for ch, cs in zip(chains, calls)]
    for (depth, dtype), ch, cs, w in zip(CHAINS, chains, calls, want):
        bf = ch[3]
        for (first, n, flags, stats), res in zip(cs, w):
            hits = res[0]
            assert_same([hits["prim_id"].astype(np.uint32), hits["t"], hits["u"], hits["v"]],
                        [x[first:first + n] for x in bf], f"chain {depth} {np.dtype(dtype).name} flags {flags} stats {stats}")
    got = run_threads([lambda ch=ch, cs=cs: trace_chain(api, ch, cs) for ch, cs in zip(chains, calls)])
    for (depth, dtype), g, w in zip(CHAINS, got, want):
        assert_same(g, w, f"chain {depth} {np.dtype(dtype).name}")




@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["3f", "3d"])
def test_chain_format_is_saved_format(gpu_lib, tmp_path, dtype):
    """The chain trees above are written in chain_formats: Bvh.save of a built tree is exactly that layout."""
    import struct
    tris = scenes.soup(300, dtype=dtype)
    bvh = gpu_lib.Bvh.build_triangles(tris)
    bounds, index_values, prim_ids = bvh.arrays()
    path = str(tmp_path / "tree.bvh")
    bvh.save(path)
    bvh.destroy()
    data = open(path, "rb").read()
    head, node, prim_id = chain_formats(dtype)
    n, p = struct.unpack_from(head, data)
    assert (n, p) == (bounds.shape[0], prim_ids.shape[0])
    at = struct.calcsize(head)
    for k in range(n):
        *b, index = struct.unpack_from(node, data, at)
        assert_same(np.array(b, dtype), bounds[k], f"node {k} bounds")
        assert index == index_values[k], f"node {k} index"
        at += struct.calcsize(node)
    assert_same(np.array(struct.unpack_from(f"<{p}{prim_id}", data, at), np.uint64), prim_ids, "primitive ids")
    assert at + struct.calcsize(f"<{p}{prim_id}") == len(data)


def test_deep_stacks_device_view(gpu_lib, dtr, chains):
    """DeviceView::trace with the triangle leaf on the three float chains, one thread each with its own workspace and torch
    stream, 100 calls of 64 to 1024 device rays: every call equals brute force and the serial run."""
    import torch
    floats = [k for k, (_, dtype) in enumerate(CHAINS) if dtype == np.float32]

    def trace(k):
        bvh, _, rays, _ = chains[k]
        stream = torch.cuda.Stream()
        out = []
        with torch.cuda.stream(stream):
            run, d_rays = Run(dtr, bvh, np.float32), cuda(rays)
            for first, n, _, _ in chain_calls(gpu_lib, k)[:100]:
                res = run(d_rays[first:], n, LEAF_TRI, 0, stream=C.c_void_p(stream.cuda_stream), sync=False)
                out.append([x.clone() for x in res[:4]])
        stream.synchronize()
        return [[x.cpu().numpy() for x in res] for res in out]

    want = [trace(k) for k in floats]
    for k, w in zip(floats, want):
        bf = chains[k][3]
        for (first, n, _, _), res in zip(chain_calls(gpu_lib, k)[:100], w):
            assert_same([res[0].view(np.uint32)] + res[1:], [x[first:first + n] for x in bf], f"chain {CHAINS[k][0]}")
    got = run_threads([lambda k=k: trace(k) for k in floats])
    for k, g, w in zip(floats, got, want):
        assert_same(g, w, f"chain {CHAINS[k][0]}")


# ---- c. many threads on one handle ------------------------------------------------------------------------------------
SHARED_CALLS = [(1_000, 0, False), (2_560_000, 0, False), (100_000, 0, True), (1_000, 1, False), (100_000, 0, False),
                (2_560_000, 0, True)]           # (rays, ANY_HIT or not, stats); the 2.56M batches run in two 1M-ray chunks
PER_RAY = 300


def per_ray_leaves(api, bvh, rays):
    """bvh3f_intersect_ray with a C callback that records every leaf call (begin, end) and reports no hit."""
    CB = C.CFUNCTYPE(C.c_bool, C.c_void_p, C.POINTER(C.c_float), C.c_size_t, C.c_size_t)

    class Callback(C.Structure):
        _fields_ = [("user_data", C.c_void_p), ("user_fn", CB)]

    calls = []

    def leaf(_, tmax, begin, end):
        calls.append((begin, end))
        return False

    cb = Callback(None, CB(leaf))
    fn = api.lib().bvh3f_intersect_ray
    out = []
    for i in range(rays.shape[0]):
        calls.clear()
        fn(bvh.handle, C.c_void_p(rays[i].ctypes.data), C.byref(cb))
        out.append(np.array(calls, np.uint64).reshape(-1, 2))
    return out


def test_many_threads_one_handle(gpu_lib):
    """Four threads issue batched calls of 1k, 100k and 2.56M rays (stats calls included, so the staging buffers grow
    between calls) on one freshly built handle while two threads trace rays one at a time through bvh3f_intersect_ray,
    whose first call downloads the tree: every answer and the tree equal the serial run on an identical handle."""
    api = gpu_lib
    tris = scenes.make_mesh("soup", 300_000)
    rays = scenes.make_primary("soup", 1600, 1600)
    per_ray = [rays[k * 7919 % 1_000_000::4099][:PER_RAY] for k in range(2)]

    def batched(bvh, calls):
        out = []
        for n, any_hit, stats in calls:
            res = bvh.intersect_rays(rays[:n], flags=api.ANY_HIT if any_hit else 0, stats=stats)
            out.append(list(res) if stats else [res])
        return out

    serial = api.Bvh.build_triangles(tris)
    want_batched = batched(serial, SHARED_CALLS)
    want_rays = [per_ray_leaves(api, serial, r) for r in per_ray]
    want_tree = serial.arrays()
    serial.destroy()
    assert sum(x.shape[0] for x in want_rays[0]) > PER_RAY

    bvh = api.Bvh.build_triangles(tris)
    orders = [SHARED_CALLS[k:] + SHARED_CALLS[:k] for k in range(4)]      # the threads start on different sizes
    got = run_threads([lambda o=o: batched(bvh, o) for o in orders] + [lambda r=r: per_ray_leaves(api, bvh, r) for r in per_ray])
    for k, (o, g) in enumerate(zip(orders, got)):
        for call, res in zip(o, g):
            assert_same(res, want_batched[SHARED_CALLS.index(call)], f"thread {k} call {call}")
    for k in range(2):
        assert_same(got[len(orders) + k], want_rays[k], f"per-ray thread {k}")
    assert_same(bvh.arrays(), want_tree, "tree")
    bvh.destroy()


# ---- d. per-thread state ---------------------------------------------------------------------------------------------
def test_last_error_is_per_thread(gpu_lib):
    """One thread makes calls that fail in their argument checks (a null stats pointer, a wrong primitive count to
    refit_boxes) and sees each one's message; another makes only successful calls on the same handle and never sees a
    message, and its hits equal the serial ones."""
    api = gpu_lib
    tris = scenes.make_mesh("soup", 50_000)
    rays = scenes.make_primary("soup", 64, 64)
    bvh = api.Bvh.build_triangles(tris)
    want = bvh.intersect_rays(rays)
    fn = api.lib().bvh3f_intersect_rays_stats
    hits = np.empty(rays.shape[0], api.HIT3F)
    boxes = np.zeros((bvh.prim_count - 1, 6), np.float32)

    def failing():
        seen = []
        for k in range(200):
            if k % 2:
                with pytest.raises(api.BvhError):
                    bvh.refit_boxes(boxes)
                seen.append(api.last_error() == "refit_boxes: prim_count mismatch")
            else:
                assert fn(bvh.handle, C.c_void_p(rays.ctypes.data), rays.shape[0], C.c_void_p(hits.ctypes.data), None, 0) == -1
                seen.append(api.last_error() == "stats pointer is null")
        return seen

    def succeeding():
        errors, out = [], []
        for _ in range(200):
            out.append(bvh.intersect_rays(rays))
            errors.append(api.last_error())
        return errors, out

    seen, (errors, out) = run_threads([failing, succeeding])
    assert all(seen), f"{seen.count(False)} of {len(seen)} failed calls left another message"
    assert set(errors) == {""}, f"the succeeding thread saw {set(errors) - {''}}"
    assert_same(out, [want] * len(out), "hits")
    bvh.destroy()


def test_stream_is_per_thread(gpu_lib):
    """A handle created on a thread that set a torch stream reports that stream; one built at the same time on another
    thread reports a private stream.  The device-pointer trace on the torch stream equals the serial run."""
    import torch
    api = gpu_lib
    tris = scenes.make_mesh("soup", 200_000)
    rays = scenes.make_primary("soup", 512, 512)

    def on_torch_stream():
        stream = torch.cuda.Stream()
        api.set_stream(stream.cuda_stream)
        try:
            with torch.cuda.stream(stream):
                verts, d_rays = cuda(tris), cuda(rays)
                hits = torch.empty((rays.shape[0], 4), dtype=torch.int32, device="cuda")
                bvh = api.Bvh.build_triangles(verts.data_ptr(), count=tris.shape[0], dtype=np.float32, flags=api.DEVICE_POINTERS)
                bvh.intersect_rays(d_rays.data_ptr(), count=rays.shape[0], hits=hits.data_ptr(), flags=api.DEVICE_POINTERS)
                reported = bvh.get_property("stream")
            stream.synchronize()
            bvh.destroy()
        finally:
            api.set_stream(None)
        return reported, stream.cuda_stream, hits.cpu().numpy().view(api.HIT3F).reshape(-1)

    def private():
        bvh = api.Bvh.build_triangles(tris)
        reported = bvh.get_property("stream")
        hits = bvh.intersect_rays(rays)
        bvh.destroy()
        return reported, hits

    _, _, want = on_torch_stream()
    (reported, stream, hits), (other, private_hits) = run_threads([on_torch_stream, private])
    assert reported == stream
    assert other not in (0, stream)
    assert_same(hits, want, "torch-stream hits")
    assert_same(private_hits, want, "private-stream hits")


def device_sequence(api, device, tris, rays):
    """On `device` through bvh_cuda_set_device while torch's current device is the other one, which every call leaves as
    it found it: build, trace, refit, trace."""
    import torch
    other = 1 - device
    torch.cuda.set_device(other)
    api.set_device(device)
    current = []
    bvh = api.Bvh.build_triangles(tris)
    current.append(torch.cuda.current_device())
    out = [bvh.intersect_rays(rays)]
    current.append(torch.cuda.current_device())
    bvh.refit_triangles(tris * np.float32(1.01))
    current.append(torch.cuda.current_device())
    out.append(bvh.intersect_rays(rays))
    current.append(torch.cuda.current_device())
    assert bvh.device_view()["device"] == device
    bvh.destroy()
    api.set_device(0)
    assert current == [other] * len(current), current
    return out


def test_device_is_per_thread(gpu_lib):
    """Threads on devices 0 and 1 at once: each one's handle is on its own device, torch's current device is unchanged
    after every call, and the hits equal the serial run."""
    import torch
    api = gpu_lib
    if api.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    tris = scenes.make_mesh("soup", 200_000)
    rays = scenes.make_primary("soup", 256, 256)
    previous = torch.cuda.current_device()
    try:
        want = [device_sequence(api, d, tris, rays) for d in (0, 1)]
    finally:
        torch.cuda.set_device(previous)
    got = run_threads([lambda d=d: device_sequence(api, d, tris, rays) for d in (0, 1)])
    assert_same(got, want, "hits")
    assert_same(want[1], want[0], "device 1 against device 0")


# ---- e. trim during work ---------------------------------------------------------------------------------------------
def test_trim_during_work(gpu_lib):
    """bvh_cuda_trim(0) 200 times on one thread while four others build, trace, refit and download their trees: every
    answer equals the serial run."""
    api = gpu_lib
    meshes = MESHES[:4]
    want = [mesh_sequence(api, *m) for m in meshes]

    def trim():
        for _ in range(200):
            api.trim(0)
            time.sleep(0.001)

    got = run_threads([lambda m=m: mesh_sequence(api, *m) for m in meshes] + [trim])
    for m, g, w in zip(meshes, got, want):
        assert_same(g, w, f"{m[0]} {m[1]} {np.dtype(m[2]).name} {m[3]}")
