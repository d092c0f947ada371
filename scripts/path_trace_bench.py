"""Times DeviceView::trace_paths against the same path tracer run as a wavefront loop of trace_triangles launches.

    python scripts/path_trace_bench.py [--steps 20] [--warmup 3] [--mesh soup grid] [--size 2048] [--bounces 4]
    python scripts/path_trace_bench.py --ptxas

The workload is tests/device_path_trace_kernels.cu's PathTracer (float): a grey diffuse path tracer with a point light,
one next-event shadow segment per closest hit with the light above the surface, and `bounces` diffuse bounces, over
bench.py's 1M-triangle meshes, one path per primary ray of bench.py's size x size camera (2048 x 2048 = 4 194 304 paths).
  trace_paths  dpt_tracer3f(wavefront = 0): one DeviceView::trace_paths launch, the payload in registers
  wavefront    dpt_tracer3f(wavefront = 1): a start kernel, then per bounce one closest-hit and one occlusion
               trace_triangles launch over all paths, the path state (ray, payload, next step) in arrays; no host
               synchronisation between the launches
Before any timing both arms' outputs are compared per path: the radiance bits, the segment count and the hash of the
segment records.  Each arm is timed as the median of `steps` CUDA-event timed batches after `warmup` batches; the
card's name and power limit are read in the same run.  Segments per second counts every segment of every path, the
same number in both arms.  --ptxas prints the registers, stack frame and spills of every device_view_path_kernel and
device_view_triangle_kernel instantiation of the test file (a compile, no GPU needed).  Nothing is written to the tree
except the test kernels' build under tests/_build when it is stale.
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


def light_for(mesh, dtype):
    """The path tracer's point light: beside the mesh's camera (bvh_b200.scenes.CAMERAS), offset in x and y."""
    from bvh_b200 import scenes
    return np.asarray(scenes.CAMERAS[mesh]["eye"], np.float64).astype(dtype) + np.array([0.25, 0.15, 0.0], dtype)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mesh", nargs="+", default=["soup", "grid"])
    ap.add_argument("--size", type=int, default=2048)
    ap.add_argument("--bounces", type=int, default=4)
    ap.add_argument("--ptxas", action="store_true")
    args = ap.parse_args()
    if args.ptxas:
        return ptxas_report()

    import torch
    import bvh_b200.api as api
    from bvh_b200 import build_ext, scenes
    L = C.CDLL(build_ext.build_device_path_trace_tests())
    L.dpt_tracer3f.argtypes = [C.c_void_p, C.c_int, C.c_uint, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_uint32] + [C.c_void_p] * 5 + [C.c_size_t, C.c_void_p]
    L.dpt_wavefront_bytes3f.argtypes = [C.c_size_t]
    L.dpt_wavefront_bytes3f.restype = C.c_size_t
    L.dpt_last_error.restype = C.c_char_p
    api.set_device(0)
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream()
    api.set_stream(stream.cuda_stream)
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

    results = []
    w = h = args.size
    n = w * h
    for mesh in args.mesh:
        tris = scenes.make_mesh(mesh, 1_000_000)
        bvh = api.Bvh.build_triangles(tris)
        d_primary = torch.from_numpy(scenes.make_primary(mesh, w, h)).cuda()
        light = light_for(mesh, np.float32)
        d_verts = torch.from_numpy(tris.reshape(-1)).cuda()
        ws = torch.empty(8, dtype=torch.uint8, device="cuda")
        scratch = torch.empty(L.dpt_wavefront_bytes3f(n), dtype=torch.uint8, device="cuda")
        outs = {arm: (torch.empty(n, dtype=torch.float32, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda"),
                      torch.empty(n, dtype=torch.int32, device="cuda")) for arm in (0, 1)}

        def run(arm):
            rad, segs, hashes = outs[arm]
            rc = L.dpt_tracer3f(C.c_void_p(bvh.handle), arm, 0, n, C.c_void_p(d_primary.data_ptr()), light.ctypes.data,
                                C.c_void_p(d_verts.data_ptr()), args.bounces, C.c_void_p(rad.data_ptr()),
                                C.c_void_p(segs.data_ptr()), C.c_void_p(hashes.data_ptr()), C.c_void_p(scratch.data_ptr()),
                                C.c_void_p(ws.data_ptr()), 8, sp)
            if rc:
                raise RuntimeError(L.dpt_last_error().decode())

        for arm in (0, 1):
            for t in outs[arm]:
                t.fill_(-1)
            run(arm)
        torch.cuda.synchronize()
        got = [tuple(t.cpu().numpy().view(np.uint32) for t in outs[arm]) for arm in (0, 1)]
        same = all((a == b).all() for a, b in zip(*got))
        if not same:
            raise RuntimeError(f"{mesh}: trace_paths and the wavefront loop differ")
        segments = int(got[0][1].astype(np.int64).sum())
        row = {"mesh": mesh, "paths": n, "bounces": args.bounces, "segments": segments,
               "lit_paths": int((got[0][0] != 0).sum()), "outputs_equal": True,
               "trace_paths_ms": timed(lambda: run(0)), "wavefront_ms": timed(lambda: run(1))}
        for k in ("trace_paths", "wavefront"):
            row[k + "_msegments_s"] = segments / row[k + "_ms"] / 1e3
        row["speedup"] = row["wavefront_ms"] / row["trace_paths_ms"]
        print(json.dumps(row), flush=True)
        results.append(row)
        bvh.destroy()
    api.set_stream(None)
    return results


def ptxas_report():
    """Registers, stack frame and spills of every device_view_path_kernel and device_view_triangle_kernel instantiation
    of tests/device_path_trace_kernels.cu, from ptxas -v."""
    from bvh_b200 import build_ext
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = ["-std=c++20" if f == "-std=c++17" else f for f in build_ext.NVCC_FLAGS]
    with tempfile.TemporaryDirectory() as d:
        res = subprocess.run([nvcc, *flags, "-Xptxas=-v", "-c", build_ext.PATH_TRACE_KERNELS_SRC, "-o", os.path.join(d, "k.o")],
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
        if "device_view_path_kernel" not in dem and "device_view_triangle_kernel" not in dem:
            continue
        spill = next((l for l in lines[i:i + 4] if "spill" in l), "").strip()
        used = next((l for l in lines[i:i + 5] if "Used" in l), "").strip()
        short = re.sub(r"\(.*", "", dem.replace("(anonymous namespace)::", "").replace("bvh::v2::cuda::", ""))
        short = short.replace("void ", "")
        out.append({"kernel": short, "resources": used.split(":", 1)[-1].strip(), "spills": spill.split(":", 1)[-1].strip()})
    for row in sorted(out, key=lambda r: r["kernel"]):
        print(json.dumps(row))
    return out


if __name__ == "__main__":
    main()
