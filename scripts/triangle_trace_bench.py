"""Times DeviceView::trace_triangles against the library's own triangle kernel and against DeviceView::trace with a
triangle leaf written by the caller.

    python scripts/triangle_trace_bench.py [--steps 20] [--warmup 3] [--mesh soup grid]
    python scripts/triangle_trace_bench.py --ptxas

For each scene (bench.py's c2: 1M triangles, 3163 x 3163 = 10 004 569 primary rays, float, rays resident in HBM) it prints
the median of `steps` CUDA-event timed calls, after `warmup` calls, of
  persistent      bvh3f_intersect_rays, default persistent kernel, device pointers, canonical tie rule
  trace_triangles tests/device_triangle_trace_kernels.cu dtt_plain3f: every hit accepted, rays from an array, 16-byte
                  records to an array
  trace           tests/device_trace_kernels.cu: DeviceView::trace with the test tracer's triangle leaf (intersect_tri per
                  triangle), last-visited tie rule
  camera          dtt_camera3f: a pinhole camera computes each ray from its index inside the shader; only t is written
and the card's name and power limit.  Before any timing every arm's output is checked against the library kernel's:
trace_triangles records bit for bit against `persistent`, trace's against bvh3f_intersect_rays with BVH_TIE_LAST_VISITED,
the camera's depths against bvh3f_intersect_rays on the same camera's rays written to an array.  --ptxas prints the
registers, stack frame and spills of every device_view_triangle_kernel instantiation of the test file (a compile, no GPU
needed).  Nothing is written to the tree except the test kernels' build under tests/_build when it is stale.
"""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import tempfile

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
    ap.add_argument("--ptxas", action="store_true")
    args = ap.parse_args()
    if args.ptxas:
        return ptxas_report()

    import torch
    import bvh_b200.api as api
    from bvh_b200 import build_ext, scenes
    dtt = C.CDLL(build_ext.build_device_triangle_trace_tests())
    dtt.dtt_plain3f.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    dtt.dtt_camera3f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    dtt.dtt_camera_rays3f.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    dtt.dtt_last_error.restype = C.c_char_p
    dtr = C.CDLL(build_ext.build_device_trace_tests())
    dtr.dtr_run3f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint, C.c_void_p, C.c_size_t] + [C.c_void_p] * 9 + [C.c_size_t, C.c_void_p]
    dtr.dtr_last_error.restype = C.c_char_p
    api.set_device(0)
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream()
    api.set_stream(stream.cuda_stream)                    # the handles' work and the timing events on one stream
    sp = C.c_void_p(stream.cuda_stream)
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)

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

    def ok(rc, lib):
        if rc:
            raise RuntimeError(lib.dtt_last_error().decode() if lib is dtt else lib.dtr_last_error().decode())

    results = []
    for mesh in args.mesh:
        tris = scenes.make_mesh(mesh, 1_000_000)
        rays = scenes.make_primary(mesh, 3163, 3163)
        n = rays.shape[0]
        bvh = api.Bvh.build_triangles(tris)
        h = C.c_void_p(bvh.handle)
        d_rays = torch.from_numpy(rays).cuda()
        lib_hits = torch.empty((n, 4), dtype=torch.float32, device="cuda")
        tt_hits = torch.empty((n, 4), dtype=torch.float32, device="cuda")
        tr_out = [torch.empty(n, dtype=torch.int32, device="cuda")] + [torch.empty(n, dtype=torch.float32, device="cuda") for _ in range(3)]
        ws = torch.empty(8, dtype=torch.uint8, device="cuda")
        lo, hi = tris.reshape(-1, 3).min(axis=0), tris.reshape(-1, 3).max(axis=0)
        cam = np.array([(lo[0] + hi[0]) / 2, (lo[1] + hi[1]) / 2, lo[2] - 1.0, lo[0], hi[0], lo[1], hi[1]], np.float32)
        depth = torch.empty(n, dtype=torch.float32, device="cuda")

        def persistent(flags=0):
            return lambda: bvh.intersect_rays(d_rays.data_ptr(), n, hits=lib_hits.data_ptr(), flags=api.DEVICE_POINTERS | flags)

        def trace_triangles():
            ok(dtt.dtt_plain3f(h, C.c_void_p(d_rays.data_ptr()), n, C.c_void_p(tt_hits.data_ptr()), C.c_void_p(ws.data_ptr()), 8, sp), dtt)

        def trace():
            p = [C.c_void_p(x.data_ptr()) for x in tr_out]
            ok(dtr.dtr_run3f(h, 0, 1, 0, C.c_void_p(d_rays.data_ptr()), n, None, *p, None, None, None, C.c_void_p(ws.data_ptr()), 8, sp), dtr)

        def camera():
            ok(dtt.dtt_camera3f(h, cam.ctypes.data, 3163, 3163, C.c_void_p(depth.data_ptr()), C.c_void_p(ws.data_ptr()), 8, sp), dtt)

        # outputs first: every arm against the library's kernel
        def u32(t):
            return t.cpu().numpy().view(np.uint32)
        persistent(api.TIE_LAST_VISITED)()
        trace()
        torch.cuda.synchronize()
        last = u32(lib_hits)
        if not all((u32(tr_out[k]) == last[:, k]).all() for k in range(4)):
            raise RuntimeError(f"{mesh}: trace records differ from bvh3f_intersect_rays(TIE_LAST_VISITED)")
        persistent()()
        trace_triangles()
        torch.cuda.synchronize()
        if not (u32(tt_hits) == u32(lib_hits)).all():
            raise RuntimeError(f"{mesh}: trace_triangles records differ from bvh3f_intersect_rays")
        cam_rays = torch.empty((n, 8), dtype=torch.float32, device="cuda")
        ok(dtt.dtt_camera_rays3f(cam.ctypes.data, 3163, 3163, C.c_void_p(cam_rays.data_ptr()), sp), dtt)
        camera()
        bvh.intersect_rays(cam_rays.data_ptr(), n, hits=lib_hits.data_ptr(), flags=api.DEVICE_POINTERS)
        torch.cuda.synchronize()
        if not (u32(depth) == u32(lib_hits)[:, 1]).all():
            raise RuntimeError(f"{mesh}: camera depths differ from bvh3f_intersect_rays on the same rays")
        cam_hits = int((u32(lib_hits)[:, 0] != 0xFFFFFFFF).sum())

        row = {"mesh": mesh, "rays": n, "camera_hits": cam_hits,
               "persistent_ms": timed(persistent()),
               "trace_triangles_ms": timed(trace_triangles),
               "trace_ms": timed(trace),
               "camera_ms": timed(camera),
               "outputs_checked": True}
        for k in ("persistent", "trace_triangles", "trace", "camera"):
            row[k + "_mrays_s"] = n / row[k + "_ms"] / 1e3
        print(json.dumps(row), flush=True)
        results.append(row)
        bvh.destroy()
    api.set_stream(None)
    return results


def ptxas_report():
    """Registers, stack frame and spills of every device_view_triangle_kernel instantiation of
    tests/device_triangle_trace_kernels.cu, from ptxas -v."""
    from bvh_b200 import build_ext
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = ["-std=c++20" if f == "-std=c++17" else f for f in build_ext.NVCC_FLAGS]
    with tempfile.TemporaryDirectory() as d:
        res = subprocess.run([nvcc, *flags, "-Xptxas=-v", "-c", build_ext.TRIANGLE_TRACE_KERNELS_SRC, "-o", os.path.join(d, "k.o")],
                             capture_output=True, text=True)
    if res.returncode:
        raise RuntimeError(res.stderr)
    lines = res.stderr.split("\n")
    out = []
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if not m:
            continue
        dem = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        if "device_view_triangle_kernel" not in dem:
            continue
        spill = next((l for l in lines[i:i + 4] if "spill" in l), "").strip()
        used = next((l for l in lines[i:i + 5] if "Used" in l), "").strip()
        short = re.sub(r"\(.*", "", dem.replace("(anonymous namespace)::", "").replace("bvh::v2::cuda::", ""))
        out.append({"kernel": short, "resources": used, "spills": spill})
        print(json.dumps(out[-1]))
    return out


if __name__ == "__main__":
    main()
