"""Times the device traversal API's triangle kernel against the library's own traversal kernels.

    python scripts/device_api_bench.py [--steps 20] [--warmup 3] [--mesh soup grid]

For each scene (bench.py's c2: 1M triangles, 3163 x 3163 primary rays) it prints the median of `steps` CUDA-event timed
launches, rays on the device, of
  device_api   tests/device_api_kernels.cu trace_kernel: DeviceView::intersect with the triangle leaf, one thread per
               ray, shared-memory stack (what a user kernel built on include/bvh/v2/cuda/intersect.cuh looks like)
  simple       bvh3f_intersect_rays with BVH_KERNEL_SIMPLE (the library's one-thread-per-ray kernel)
  persistent   bvh3f_intersect_rays with the default (persistent) kernel
  device_trace tests/device_trace_kernels.cu: DeviceView::trace with the same triangle leaf (the library's persistent
               scheduler over a user's tracer); its hit records are checked bit for bit against `persistent` first
all with BVH_TIE_LAST_VISITED (the device API kernel's tie rule), plus the card's name and power limit.  A sphere scene
(1M spheres built from device boxes, 10M primary rays) times the same sphere tracer one thread per ray (`per_thread`)
and through DeviceView::trace (`device_trace`).  --ptxas prints the registers, shared memory and spills of the test
tracers' instantiations (a compile, no GPU needed).  Nothing is
written to the tree except the test kernels' build under tests/_build when it is stale.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mesh", nargs="+", default=["soup", "grid"])
    ap.add_argument("--no-spheres", action="store_true")
    ap.add_argument("--ptxas", action="store_true")
    args = ap.parse_args()
    if args.ptxas:
        return ptxas_report()

    import torch
    import bvh_b200.api as api
    from bvh_b200 import build_ext, scenes
    dapi = C.CDLL(build_ext.build_device_api_tests())
    dapi.dapi_bench3f.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint, C.c_void_p, C.c_int, C.POINTER(C.c_float)]
    dapi.dapi_last_error.restype = C.c_char_p
    dtr = C.CDLL(build_ext.build_device_trace_tests())
    dtr.dtr_run3f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint] + [C.c_void_p, C.c_size_t] + [C.c_void_p] * 9 + [C.c_size_t, C.c_void_p]
    dtr.dtr_last_error.restype = C.c_char_p
    api.set_device(0)
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream()
    api.set_stream(stream.cuda_stream)                    # the handles' work and the timing events on one stream
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    results = []
    for mesh in args.mesh:
        tris = scenes.make_mesh(mesh, 1_000_000)
        rays = scenes.make_primary(mesh, 3163, 3163)
        n = rays.shape[0]
        bvh = api.Bvh.build_triangles(tris)
        d_rays = torch.from_numpy(rays).cuda()
        d_hits = torch.empty((n, 4), dtype=torch.float32, device="cuda")
        scratch = torch.empty(n * 8 + 3 * n * 4, dtype=torch.uint8, device="cuda")

        def timed(fn):
            for _ in range(args.warmup):
                fn()
            ms = []
            for _ in range(args.steps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                fn()
                b.record(stream)
                b.synchronize()
                ms.append(a.elapsed_time(b))
            return float(np.median(ms))

        def lib_call(flags):
            return lambda: bvh.intersect_rays(d_rays.data_ptr(), n, hits=d_hits.data_ptr(),
                                              flags=api.DEVICE_POINTERS | api.TIE_LAST_VISITED | flags)

        ms = (C.c_float * (args.steps + args.warmup))()
        rc = dapi.dapi_bench3f(C.c_void_p(bvh.handle), C.c_void_p(d_rays.data_ptr()), n, 0, C.c_void_p(scratch.data_ptr()),
                               args.steps + args.warmup, ms)
        if rc:
            raise RuntimeError(dapi.dapi_last_error().decode())
        trace = tracer_call(dtr, bvh, d_rays, n, 1, stream)
        lib_call(0)()
        trace()
        torch.cuda.synchronize()
        want = d_hits.cpu().numpy()
        ids, t, u, v = (x.cpu().numpy() for x in trace.outputs[:4])
        same = ((ids.view(np.uint32) == want[:, 0].view(np.uint32)) & (t.view(np.uint32) == want[:, 1].view(np.uint32)) &
                (u.view(np.uint32) == want[:, 2].view(np.uint32)) & (v.view(np.uint32) == want[:, 3].view(np.uint32)))
        if not same.all():
            raise RuntimeError(f"{mesh}: device_trace records differ from persistent at {np.nonzero(~same)[0][:8]}")
        row = {"mesh": mesh, "rays": n,
               "device_api_ms": float(np.median(list(ms)[args.warmup:])),
               "simple_ms": timed(lib_call(api.KERNEL_SIMPLE)),
               "persistent_ms": timed(lib_call(0)),
               "device_trace_ms": timed(trace),
               "device_trace_records_equal_persistent": True}
        for k in ("device_api", "simple", "persistent", "device_trace"):
            row[k + "_mrays_s"] = n / row[k + "_ms"] / 1e3
        print(json.dumps(row), flush=True)
        results.append(row)
        bvh.destroy()
    if not args.no_spheres:
        results.append(sphere_scene(api, dtr, stream, timed_on(stream, args)))
        print(json.dumps(results[-1]), flush=True)
    api.set_stream(None)
    return results


def timed_on(stream, args):
    import torch

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        ms = []
        for _ in range(args.steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fn()
            b.record(stream)
            b.synchronize()
            ms.append(a.elapsed_time(b))
        return float(np.median(ms))
    return timed


class tracer_call:
    """One dtr_run3f launch (tests/device_trace_kernels.cu) on `stream`, no synchronisation; leaf 1 triangles, 2 spheres."""

    def __init__(self, dtr, bvh, d_rays, n, leaf, stream, per_thread=False, spheres=None):
        import torch
        self.dtr, self.bvh, self.d_rays, self.n, self.leaf, self.per_thread = dtr, bvh, d_rays, n, leaf, per_thread
        self.spheres, self.stream = spheres, stream
        self.outputs = [torch.empty(n, dtype=torch.int32, device="cuda")] + [torch.empty(n, dtype=torch.float32, device="cuda") for _ in range(3)]
        self.ws = torch.empty(8, dtype=torch.uint8, device="cuda")

    def __call__(self):
        p = [C.c_void_p(x.data_ptr()) for x in self.outputs]
        rc = self.dtr.dtr_run3f(C.c_void_p(self.bvh.handle), int(self.per_thread), self.leaf, 0, C.c_void_p(self.d_rays.data_ptr()),
                                self.n, C.c_void_p(self.spheres.data_ptr()) if self.spheres is not None else None, *p,
                                None, None, None, C.c_void_p(self.ws.data_ptr()), 8, C.c_void_p(self.stream.cuda_stream))
        if rc:
            raise RuntimeError(self.dtr.dtr_last_error().decode())


def sphere_scene(api, dtr, stream, timed, n=1_000_000, w=3163):
    """1M spheres in the unit cube (as scripts/device_query_bench.py makes them), built from device boxes, and w x w primary
    rays from a pinhole camera in front of the cube."""
    import torch
    rng = np.random.default_rng(1)
    centers = rng.random((n, 3), dtype=np.float32)
    radii = (0.002 + 0.004 * rng.random(n)).astype(np.float32)
    c, r = torch.from_numpy(centers).cuda(), torch.from_numpy(radii).cuda()[:, None]
    boxes = torch.cat([c - r, c + r], dim=1).contiguous()
    spheres = torch.cat([c, r], dim=1).contiguous()
    torch.cuda.synchronize()
    bvh = api.Bvh.build_boxes(boxes.data_ptr(), c.data_ptr(), count=n, dtype=np.float32, flags=api.DEVICE_POINTERS)
    ys, xs = np.meshgrid((np.arange(w) + 0.5) / w, (np.arange(w) + 0.5) / w, indexing="ij")
    rays = np.zeros((w * w, 8), np.float32)
    rays[:, 0], rays[:, 1], rays[:, 2] = 0.5, 0.5, -1.0
    rays[:, 3], rays[:, 4], rays[:, 5] = xs.ravel() - 0.5, ys.ravel() - 0.5, 1.0
    rays[:, 7] = np.inf
    d_rays = torch.from_numpy(rays).cuda()
    m = rays.shape[0]
    per_thread = tracer_call(dtr, bvh, d_rays, m, 2, stream, per_thread=True, spheres=spheres)
    trace = tracer_call(dtr, bvh, d_rays, m, 2, stream, spheres=spheres)
    per_thread(); trace()
    torch.cuda.synchronize()
    same = all((a.cpu().numpy().view(np.uint32) == b.cpu().numpy().view(np.uint32)).all()
               for a, b in zip(per_thread.outputs, trace.outputs))
    if not same:
        raise RuntimeError("spheres: device_trace records differ from per_thread")
    row = {"scene": "spheres-1M", "rays": m, "hits": int((trace.outputs[0] != -1).sum().item()),
           "per_thread_ms": timed(per_thread), "device_trace_ms": timed(trace), "device_trace_records_equal_per_thread": True}
    for k in ("per_thread", "device_trace"):
        row[k + "_mrays_s"] = m / row[k + "_ms"] / 1e3
    bvh.destroy()
    return row


def ptxas_report():
    """Registers, shared memory and spills of every kernel of tests/device_trace_kernels.cu, from ptxas -v."""
    from bvh_b200 import build_ext
    import re
    import tempfile
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = ["-std=c++20" if f == "-std=c++17" else f for f in build_ext.NVCC_FLAGS]
    with tempfile.TemporaryDirectory() as d:
        res = subprocess.run([nvcc, *flags, "-Xptxas=-v", "-c", build_ext.TRACE_KERNELS_SRC, "-o", os.path.join(d, "k.o")],
                             capture_output=True, text=True)
    if res.returncode:
        raise RuntimeError(res.stderr)
    lines = res.stderr.split("\n")
    names = []
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if not m:
            continue
        dem = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        spill = next((l for l in lines[i:i + 4] if "spill" in l), "").strip()
        used = next((l for l in lines[i:i + 5] if "Used" in l), "").strip()
        names.append((dem, used, spill))
    for dem, used, spill in names:
        short = dem.replace("(anonymous namespace)::", "").replace("bvh::v2::cuda::", "")
        short = re.sub(r"\(.*", "", short)
        print(json.dumps({"kernel": short, "resources": used, "spills": spill}))
    return names


if __name__ == "__main__":
    main()
