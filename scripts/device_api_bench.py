"""Times the device traversal API's triangle kernel against the library's own traversal kernels.

    python scripts/device_api_bench.py [--steps 20] [--warmup 3] [--mesh soup grid]

For each scene (bench.py's c2: 1M triangles, 3163 x 3163 primary rays) it prints the median of `steps` CUDA-event timed
launches, rays on the device, of
  device_api   tests/device_api_kernels.cu trace_kernel: DeviceView::intersect with the triangle leaf, one thread per
               ray, shared-memory stack (what a user kernel built on include/bvh/v2/cuda/intersect.cuh looks like)
  simple       bvh3f_intersect_rays with BVH_KERNEL_SIMPLE (the library's one-thread-per-ray kernel)
  persistent   bvh3f_intersect_rays with the default (persistent) kernel
all with BVH_TIE_LAST_VISITED (the device API kernel's tie rule), plus the card's name and power limit.  Nothing is
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
    args = ap.parse_args()

    import torch
    import bvh_b200.api as api
    from bvh_b200 import build_ext, scenes
    dapi = C.CDLL(build_ext.build_device_api_tests())
    dapi.dapi_bench3f.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint, C.c_void_p, C.c_int, C.POINTER(C.c_float)]
    dapi.dapi_last_error.restype = C.c_char_p
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
        row = {"mesh": mesh, "rays": n,
               "device_api_ms": float(np.median(list(ms)[args.warmup:])),
               "simple_ms": timed(lib_call(api.KERNEL_SIMPLE)),
               "persistent_ms": timed(lib_call(0))}
        for k in ("device_api", "simple", "persistent"):
            row[k + "_mrays_s"] = n / row[k + "_ms"] / 1e3
        print(json.dumps(row), flush=True)
        results.append(row)
        bvh.destroy()
    api.set_stream(None)
    return results


if __name__ == "__main__":
    main()
