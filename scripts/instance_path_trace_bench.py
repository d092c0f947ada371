"""Times DeviceView::trace_instance_paths against the same path tracer run as a wavefront loop of trace_instances
launches, with trace_paths over the flattened scene for context.

    python scripts/instance_path_trace_bench.py [--instances 256] [--width 2048 --height 2048] [--bounces 4] [--steps 10] [--warmup 2]
    python scripts/instance_path_trace_bench.py --ptxas      # registers and spills of the kernel (no GPU needed)

The scene is scripts/instance_trace_bench.py's: `--instances` copies, alternately of soup-64k and grid-64k, each rotated
and scaled on a grid of cells, and one path per primary ray from below, in pixel order.  The workload is
tests/device_instance_path_trace_kernels.cu's InstancePathTracer (float): a grey diffuse path tracer with a point light,
one next-event shadow segment per closest hit with the light above the surface, and `bounces` diffuse bounces.
  one_launch  dipt_tracer3f(mode 0): one DeviceView::trace_instance_paths launch, the payload in registers
  wavefront   dipt_tracer3f(mode 1): a start kernel, then per bounce one closest-hit and one occlusion trace_instances
              launch over all paths, the path state (ray, payload, next step) in arrays; no host synchronisation inside
              the batch
  flattened   dipt_tracer3f(mode 2): trace_paths over one tree built from all placed triangles in world space.  Those
              triangles are rounded in world space, so some paths differ; their count is printed
Before any timing the first two arms are compared per path: the radiance bits, the segment count and the hash of the
segment records.  Each arm is timed with CUDA events as the median of `steps` batches after `warmup` batches; the card's
name and power limit are read in the same run.  Nothing is written to the tree except the test kernels' build under
tests/_build when it is stale.
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


def ptxas_table():
    """Compiles tests/device_instance_path_trace_kernels.cu with the library's flags and -Xptxas=-v into a temporary
    directory and prints registers, stack frame and spills of every device_view_instance_path_kernel."""
    from bvh_b200 import build_ext
    flags = ["-std=c++20" if f == "-std=c++17" else f for f in build_ext.NVCC_FLAGS]
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, *flags, "-Xcompiler", "-march=x86-64-v3", "-Xptxas=-v", "-c", build_ext.INSTANCE_PATH_TRACE_KERNELS_SRC,
                              "-o", os.path.join(tmp, "k.o")], capture_output=True, text=True)
    if res.returncode:
        sys.exit(res.stderr)
    lines = res.stderr.splitlines()
    rows, name = [], None
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        m = re.search(r"Used (\d+) registers", line)
        if m and name and "instance_path_kernel" in name:
            prev = " ".join(lines[i - 2:i])
            s = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", prev)
            kind = re.match(r"void bvh::v2::cuda::(\w+)<(\w+), (\w+), (\w+), \(anonymous namespace\)::(\w+)", name)
            rows.append((kind.groups() if kind else (name,), int(m.group(1))) + (s.groups() if s else ("0", "0", "0")))
    print("| kernel | T | robust | last | shader | registers | stack frame | spill stores | spill loads |")
    print("|---|---|---|---|---|---|---|---|---|")
    for g, regs, frame, st, ld in sorted(rows, key=lambda r: r[0]):
        print("| " + " | ".join(g) + f" | {regs} | {frame} | {st} | {ld} |")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=256)
    ap.add_argument("--tris", type=int, default=65536)
    ap.add_argument("--width", type=int, default=2048)
    ap.add_argument("--height", type=int, default=2048)
    ap.add_argument("--bounces", type=int, default=4)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ptxas", action="store_true")
    a = ap.parse_args()
    if a.ptxas:
        ptxas_table()
        return
    import torch
    import bvh_b200.api as api
    from bvh_b200 import build_ext, scenes
    from tests.test_device_instance_trace_gpu import Scene, cuda, host, placements, ptr, world_rays, world_triangles

    api.lib()
    assert api.device_count() > 0, "needs a CUDA device"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True).stdout.strip()
    P, SZ, U, U32 = C.c_void_p, C.c_size_t, C.c_uint, C.c_uint32
    dit = C.CDLL(build_ext.build_device_instance_trace_tests())
    dit.dit_records3f.argtypes = [P, P, P, SZ, P, C.POINTER(SZ), P]
    dit.dit_prepare3f.argtypes = [P, SZ, SZ, P, P, P]
    dit.dit_record_bytes3f.restype = SZ
    dit.dit_last_error.restype = C.c_char_p
    L = C.CDLL(build_ext.build_device_instance_path_trace_tests())
    L.dipt_tracer3f.argtypes = [P, P, SZ, SZ, C.c_int, U, SZ, P, P, P, U32, P, P, P, P, P, SZ, P]
    L.dipt_wavefront_bytes3f.argtypes = [SZ]
    L.dipt_wavefront_bytes3f.restype = SZ
    L.dipt_last_error.restype = C.c_char_p

    # every handle, call and event on one stream, so that the events time the work
    stream = torch.cuda.Stream()
    api.set_stream(stream.cuda_stream)
    torch.cuda.set_stream(stream)
    sp = C.c_void_p(stream.cuda_stream)
    meshes = [scenes.make_mesh("soup", a.tris), scenes.make_mesh("grid", a.tris)]
    mats = placements(a.instances, seed=1)
    mesh_of = np.arange(a.instances) % 2
    scene = Scene(dit, api, meshes, mesh_of, mats, np.float32)
    flat_tris = world_triangles(meshes, mesh_of, mats).reshape(-1, 9).astype(np.float32)
    flat = api.Bvh.build_triangles(flat_tris)
    primary = cuda(world_rays(mats, a.width, a.height, np.float32))
    n = a.width * a.height
    light = (mats.reshape(-1, 3, 4)[:, :, 3].mean(axis=0) + np.array([0.3, -0.2, -4.0])).astype(np.float32)
    d_meshes = [cuda(m.reshape(-1)) for m in meshes]
    d_flat = cuda(flat_tris.reshape(-1))
    verts = torch.tensor([d_meshes[k].data_ptr() for k in mesh_of], dtype=torch.int64, device="cuda")
    flat_verts = torch.tensor([d_flat.data_ptr()], dtype=torch.int64, device="cuda")
    scratch = torch.empty(L.dipt_wavefront_bytes3f(n), dtype=torch.uint8, device="cuda")
    ws = torch.empty(8, dtype=torch.uint8, device="cuda")
    outs = [(torch.empty(n, dtype=torch.float32, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda"),
             torch.empty(n, dtype=torch.int32, device="cuda")) for _ in range(3)]

    def arm(mode):
        handle = flat.handle if mode == 2 else scene.top.handle
        rad, segs, hashes = outs[mode]

        def run():
            rc = L.dipt_tracer3f(C.c_void_p(handle), ptr(scene.records), scene.count, scene.max_depth, mode, 0, n, ptr(primary),
                                 light.ctypes.data, ptr(flat_verts if mode == 2 else verts), a.bounces, ptr(rad), ptr(segs),
                                 ptr(hashes), ptr(scratch), ptr(ws), 8, sp)
            if rc:
                raise RuntimeError(L.dipt_last_error().decode())
        return run

    runs = {"one_launch": arm(0), "wavefront": arm(1), "flattened": arm(2)}
    for f in runs.values():
        f()
    torch.cuda.synchronize()
    got = [tuple(host(x) for x in o) for o in outs]
    for name, x, y in zip(("radiance", "segments", "hashes"), got[0], got[1]):
        same = x.view(np.uint32) == y.view(np.uint32)
        assert same.all(), f"one launch and wavefront loop differ in {name} at {np.nonzero(~same)[0][:8]}"
    differ = int(((got[0][0].view(np.uint32) != got[2][0].view(np.uint32)) | (got[0][1] != got[2][1])).sum())
    segments = int(got[0][1].astype(np.int64).sum())

    def timed(f):
        for _ in range(a.warmup):
            f()
        torch.cuda.synchronize()
        times = []
        for _ in range(a.steps):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(stream)
            f()
            t1.record(stream)
            t1.synchronize()
            times.append(t0.elapsed_time(t1))
        return float(np.median(times)), float(np.min(times)), float(np.max(times))

    t = {k: timed(f) for k, f in runs.items()}
    print(f"# {gpu}")
    print(f"# {a.instances} instances, {flat_tris.shape[0]} placed triangles, {n} paths, {a.bounces} bounces, {segments} segments")
    for k, (med, lo, hi) in t.items():
        print(f"{k:10s} {med:8.3f} ms (min {lo:.3f}, max {hi:.3f})  {segments / med / 1e3:8.1f} Msegments/s")
    print(f"one_launch / wavefront speed-up {t['wavefront'][0] / t['one_launch'][0]:.3f}x; flattened paths differing: {differ}")
    out = {"gpu": gpu, "instances": a.instances, "placed_triangles": int(flat_tris.shape[0]), "paths": n, "bounces": a.bounces,
           "segments": segments, "flat_differ": differ, "ms": {k: round(v[0], 3) for k, v in t.items()},
           "msegments_per_s": {k: round(segments / v[0] / 1e3, 1) for k, v in t.items()},
           "speedup_vs_wavefront": round(t["wavefront"][0] / t["one_launch"][0], 3)}
    print(json.dumps(out))
    flat.destroy()
    scene.destroy()
    api.set_stream(None)


if __name__ == "__main__":
    main()
