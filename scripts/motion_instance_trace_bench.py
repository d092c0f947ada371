"""The motion form of DeviceView::trace_instances against the static call on the same scene.

The scene: instance_trace_bench.py's `--instances` copies (alternately of soup-64k and grid-64k, each randomly rotated
and scaled on a grid of cells; 256 copies give about 16.8M placed triangles), each with a second key moved by up to
one cell width and turned by up to 30 degrees (tests/test_device_motion_instance_gpu.py moving_keys), and `--width` x
`--height` primary rays from below, in pixel order, each at a random time in [0, 1].  Timed with CUDA events, float,
closest-hit, every hit accepted, median of `--reps` after a warm-up:
  static   trace_instances over static records at tau = 0.5, on their own top tree (tests/device_instance_trace_kernels.cu
           dit_plain3f)
  equal    the motion call with both keys at tau = 0.5's placement, on its own top tree (dmi_plain3f): the cost of
           building the placement on every instance entry
  motion   the motion call with moving keys at the rays' times, on the top tree of the union boxes: adds the looser boxes
  frame    one frame of the top level: prepare_motion_instances + bvh3f_refit_boxes, stream-ordered
Before timing, `equal` is checked against `static`: records and instances bit for bit, on all but at most one ray in
10 000 (their top trees differ by the blend's widening of the boxes, which can change which of two exactly tied hits
is visited first); the count that differs is printed.  Prints the card's name and power limit with the numbers, and one JSON line.

    python scripts/motion_instance_trace_bench.py [--instances 256] [--width 2048 --height 2048] [--reps 10]
    python scripts/motion_instance_trace_bench.py --ptxas    # registers and spills of the motion kernels (no GPU needed)
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
    """Compiles tests/device_motion_instance_kernels.cu with the library's flags and -Xptxas=-v into a temporary
    directory and prints registers and spills of both motion kernels (device_view_instance_kernel and
    device_view_instance_path_kernel under a MotionShader)."""
    from bvh_b200 import build_ext
    flags = ["-std=c++20" if f == "-std=c++17" else f for f in build_ext.NVCC_FLAGS]
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, *flags, "-Xcompiler", "-march=x86-64-v3", "-Xptxas=-v", "-c", build_ext.MOTION_INSTANCE_KERNELS_SRC,
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
        if m and name and "MotionShader" in name and ("instance_kernel" in name or "instance_path_kernel" in name):
            spill = next((x for x in lines[i - 2:i] if "spill" in x), "")
            s = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", spill)
            kernel = re.match(r"void bvh::v2::cuda::(\w+)<(.*?), bvh::v2::cuda::detail::MotionShader<\w+, \(anonymous namespace\)::(\w+)", name)
            g = (kernel.group(1), kernel.group(2), kernel.group(3)) if kernel else (name, "", "")
            rows.append((g, int(m.group(1)), s.group(1) if s else "0", s.group(2) if s else "0"))
    print("| kernel | T, flags | shader | registers | spill stores | spill loads |")
    print("|---|---|---|---|---|---|")
    for g, regs, st, ld in sorted(rows, key=lambda r: r[0]):
        print("| " + " | ".join(g) + f" | {regs} | {st} | {ld} |")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=256)
    ap.add_argument("--tris", type=int, default=65536)
    ap.add_argument("--width", type=int, default=2048)
    ap.add_argument("--height", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--ptxas", action="store_true")
    a = ap.parse_args()
    if a.ptxas:
        ptxas_table()
        return
    import torch
    import bvh_b200.api as api
    from bvh_b200 import build_ext, scenes
    from tests.test_device_instance_trace_gpu import Scene, check, cuda, host, ptr, world_rays
    from tests.test_device_motion_instance_gpu import MotionScene, moving_keys

    api.lib()
    assert api.device_count() > 0, "needs a CUDA device"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True).stdout.strip()
    P, SZ = C.c_void_p, C.c_size_t
    S = C.CDLL(build_ext.build_device_instance_trace_tests())
    S.dit_records3f.argtypes = [P, P, P, SZ, P, C.POINTER(SZ), P]
    S.dit_prepare3f.argtypes = [P, SZ, SZ, P, P, P]
    S.dit_record_bytes3f.restype = SZ
    S.dit_plain3f.argtypes = [P, P, SZ, SZ, P, SZ, P, P, P, SZ, P]
    S.dit_last_error.restype = C.c_char_p
    M = C.CDLL(build_ext.build_device_motion_instance_tests())
    M.dmi_records3f.argtypes = [P, P, P, P, SZ, P, C.POINTER(SZ), P]
    M.dmi_prepare3f.argtypes = [P, SZ, SZ, P, P, P]
    M.dmi_placement3f.argtypes = [P, P, SZ, P, P]
    M.dmi_record_bytes3f.restype = SZ
    M.dmi_plain3f.argtypes = [P, P, SZ, SZ, P, P, SZ, P, P, P, SZ, P]
    M.dmi_last_error.restype = C.c_char_p

    def mcheck(rc):
        if rc:
            raise RuntimeError(M.dmi_last_error().decode())

    # every handle, call and event on one stream, so that the events time the work
    stream = torch.cuda.Stream()
    api.set_stream(stream.cuda_stream)
    torch.cuda.set_stream(stream)
    sp = C.c_void_p(stream.cuda_stream)
    meshes = [scenes.make_mesh("soup", a.tris), scenes.make_mesh("grid", a.tris)]
    mesh_of = np.arange(a.instances) % 2
    keys0, keys1 = moving_keys(a.instances, seed=1)
    keys0, keys1 = keys0.astype(np.float32), keys1.astype(np.float32)
    moving = MotionScene(M, api, meshes, mesh_of, keys0, keys1, np.float32)
    # the placement at tau = 0.5, as the motion call rounds it, for the static and the equal-keys scenes
    mid = moving.placement(np.full(a.instances, 0.5))[:, 0].astype(np.float32)
    static = Scene(S, api, moving.meshes, mesh_of, mid, np.float32)
    equal = MotionScene(M, api, moving.meshes, mesh_of, mid, mid, np.float32)
    rays = world_rays(np.concatenate([keys0, keys1]), a.width, a.height, np.float32)
    n = rays.shape[0]
    d_rays = cuda(rays)
    d_half = cuda(np.full(n, 0.5, np.float32))
    d_times = cuda(np.random.default_rng(5).uniform(0, 1, size=n).astype(np.float32))
    hits = [torch.empty((n, 4), dtype=torch.float32, device="cuda") for _ in range(3)]
    insts = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(3)]
    ws = torch.empty(64, dtype=torch.uint8, device="cuda")

    def run_static():
        check(S, S.dit_plain3f(C.c_void_p(static.top.handle), ptr(static.records), static.count, static.max_depth, ptr(d_rays), n,
                               ptr(hits[0]), ptr(insts[0]), ptr(ws), 64, sp))

    def run_equal():
        mcheck(M.dmi_plain3f(C.c_void_p(equal.top.handle), ptr(equal.records), equal.count, equal.max_depth, ptr(d_rays), ptr(d_half), n,
                             ptr(hits[1]), ptr(insts[1]), ptr(ws), 64, sp))

    def run_motion():
        mcheck(M.dmi_plain3f(C.c_void_p(moving.top.handle), ptr(moving.records), moving.count, moving.max_depth, ptr(d_rays),
                             ptr(d_times), n, ptr(hits[2]), ptr(insts[2]), ptr(ws), 64, sp))

    def run_frame():
        moving.prepare(sp)
        moving.top.refit_boxes(moving.boxes.data_ptr(), api.DEVICE_POINTERS)

    for f in (run_static, run_equal, run_motion):
        f()
    torch.cuda.synchronize()
    h0, h1, h2 = (host(h).view(np.uint32) for h in hits)
    i0, i1 = host(insts[0]), host(insts[1])
    same = (h0 == h1).all(axis=1) & (i0 == i1)
    assert same.mean() > 0.9999, f"{int((~same).sum())} rays differ between the static and the equal-keys motion call"
    hit_static, hit_motion = float((h0[:, 0] != 0xFFFFFFFF).mean()), float((h2[:, 0] != 0xFFFFFFFF).mean())

    def timed(f):
        f()
        torch.cuda.synchronize()
        times = []
        for _ in range(a.reps):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(stream)
            f()
            t1.record(stream)
            t1.synchronize()
            times.append(t0.elapsed_time(t1))
        return float(np.median(times))

    t = {"static": timed(run_static), "equal": timed(run_equal), "motion": timed(run_motion), "frame": timed(run_frame)}
    out = {"gpu": gpu, "instances": a.instances, "rays": n, "hit_fraction": {"static": hit_static, "motion": hit_motion},
           "equal_vs_static_differ": int((~same).sum()), "ms": {k: round(v, 3) for k, v in t.items()},
           "mrays_per_s": {k: round(n / t[k] / 1e3, 1) for k in ("static", "equal", "motion")}}
    print(f"# {gpu}")
    for k in ("static", "equal", "motion"):
        print(f"{k:8s} {t[k]:8.3f} ms  {n / t[k] / 1e3:8.1f} Mrays/s")
    print(f"frame    {t['frame']:8.3f} ms  (prepare_motion_instances + refit_boxes, {a.instances} instances)")
    print(json.dumps(out))
    static.top.destroy()
    equal.top.destroy()
    moving.destroy()
    api.set_stream(None)


if __name__ == "__main__":
    main()
