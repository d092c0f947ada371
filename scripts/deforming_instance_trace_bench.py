"""The deforming forms of DeviceView::trace_instances against the motion call and the two-launch workaround.

The scene: motion_instance_trace_bench.py's `--instances` copies (alternately of soup-64k and grid-64k, randomly rotated
and scaled on a grid of cells, each with a second placement key moved by up to one cell and turned by up to 30
degrees), of which every `--every`-th copy (16 of 256 by default) is instead a deforming soup-64k whose vertices move by
`--move` triangle sizes over the shutter (a smooth field: every vertex of a triangle moves alike, so triangles keep
their shape), and `--width` x `--height` primary rays from below, each at a random time in [0, 1].  Timed with CUDA
events on one stream, float, closest-hit, every hit accepted, median of `--reps` after a warm-up, for each `--move`:
  frozen     the motion trace_instances with the deforming copies frozen at tau = 0.5 (a static mesh of the vertices
             at 0.5): the cost of the scene without vertex motion (tests/device_motion_instance_kernels.cu dmi_plain3f)
  static     the deforming trace_instances over the same records, every bottom static (ddi_plain3f): the cost of the
             per-record branch of the new kernel
  shutter    the deforming copies as deforming bottoms on shutter boxes
  nodes      the deforming copies as deforming bottoms with motion nodes
  workaround the motion trace_instances over the static copies only, then one motion-node trace_triangles launch per
             deforming copy with the ray moved into its object space and a closest-hit merge (ddi_workaround3f)
  frame      one frame's preparation: the deforming mesh's prepare_motion_triangles, refit and prepare_motion_nodes,
             prepare_deforming_instances and the top refit
Before timing, `shutter` and `nodes` are checked to give the same closest hits (robust traversal is not used here, so
the count that differs is printed rather than asserted), and the hit fractions are printed.  Prints the card's name
and power limit with the numbers, and one JSON line.

    python scripts/deforming_instance_trace_bench.py [--instances 256] [--every 16] [--move 1 4] [--width 2048 --height 2048]
    python scripts/deforming_instance_trace_bench.py --ptxas    # registers and spills of the deforming kernels (no GPU)
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
    """Compiles tests/device_deforming_instance_kernels.cu with the library's flags and -Xptxas=-v into a temporary
    directory and prints registers and spills of the instance kernels under WithDeformingBottoms."""
    from bvh_b200 import build_ext
    flags = ["-std=c++20" if f == "-std=c++17" else f for f in build_ext.NVCC_FLAGS]
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, *flags, "-Xcompiler", "-march=x86-64-v3", "-Xptxas=-v", "-c", build_ext.DEFORMING_INSTANCE_KERNELS_SRC,
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
        if m and name and "WithDeformingBottoms" in name:
            spill = next((x for x in lines[i - 2:i] if "spill" in x), "")
            s = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", spill)
            kernel = re.match(r"void bvh::v2::cuda::(\w+)<(.*?), bvh::v2::cuda::detail::MotionShader<.*?\(anonymous namespace\)::(\w+)", name)
            g = (kernel.group(1), kernel.group(2), kernel.group(3)) if kernel else (name, "", "")
            rows.append((g, int(m.group(1)), s.group(1) if s else "0", s.group(2) if s else "0"))
    print("| kernel | T, flags | shader | registers | spill stores | spill loads |")
    print("|---|---|---|---|---|---|")
    for g, regs, st, ld in sorted(rows, key=lambda r: r[0]):
        print("| " + " | ".join(g) + f" | {regs} | {st} | {ld} |")


def moved(tris, move):
    """vertex keys: the soup at time 0 and moved by `move` triangle sizes along a smooth field at time 1"""
    v = tris.reshape(-1, 3, 3).astype(np.float64)
    size = float(np.median(np.linalg.norm(v[:, 1] - v[:, 0], axis=1)))
    c = v.mean(axis=1)
    field = np.stack([np.sin(2 * np.pi * c[:, 1]), np.cos(2 * np.pi * c[:, 0]), 0.5 * np.sin(2 * np.pi * c[:, 2])], axis=1)
    field /= np.maximum(np.linalg.norm(field, axis=1, keepdims=True), 1e-9)
    k1 = v + (move * size * field)[:, None, :]
    return np.ascontiguousarray(tris, np.float32), np.ascontiguousarray(k1.reshape(-1, 9), np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=256)
    ap.add_argument("--every", type=int, default=16)
    ap.add_argument("--tris", type=int, default=65536)
    ap.add_argument("--move", type=float, nargs="+", default=[1.0, 4.0])
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
    from tests.test_device_instance_trace_gpu import cuda, host, ptr, world_rays
    from tests.test_device_motion_instance_gpu import MotionScene, moving_keys

    api.lib()
    assert api.device_count() > 0, "needs a CUDA device"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True).stdout.strip()
    P, SZ = C.c_void_p, C.c_size_t
    M = C.CDLL(build_ext.build_device_motion_instance_tests())
    M.dmi_records3f.argtypes = [P, P, P, P, SZ, P, C.POINTER(SZ), P]
    M.dmi_prepare3f.argtypes = [P, SZ, SZ, P, P, P]
    M.dmi_placement3f.argtypes = [P, P, SZ, P, P]
    M.dmi_record_bytes3f.restype = SZ
    M.dmi_plain3f.argtypes = [P, P, SZ, SZ, P, P, SZ, P, P, P, SZ, P]
    M.dmi_last_error.restype = C.c_char_p
    D = C.CDLL(build_ext.build_device_deforming_instance_tests())
    D.ddi_records3f.argtypes = [P, P, P, P, P, P, P, P, SZ, P, C.POINTER(SZ), P]
    D.ddi_prepare3f.argtypes = [P, SZ, SZ, P, P, P]
    D.ddi_bottom3f.argtypes = [P, P, P, SZ, P, P, P, P, SZ, P]
    D.ddi_plain3f.argtypes = [P, P, SZ, SZ, P, P, SZ, P, P, P, SZ, P]
    D.ddi_workaround3f.argtypes = [P, P, SZ, SZ, P, P, P, P, P, P, SZ, P, P, SZ, P, P, P, SZ, P]
    for f in ("record_bytes3f", "motion_node_bytes3f"):
        getattr(D, f"ddi_{f}").restype = SZ
    D.ddi_last_error.restype = C.c_char_p

    def check(lib, rc, prefix):
        if rc:
            raise RuntimeError(getattr(lib, f"{prefix}_last_error")().decode())

    # every handle, call and event on one stream, so that the events time the work
    stream = torch.cuda.Stream()
    api.set_stream(stream.cuda_stream)
    torch.cuda.set_stream(stream)
    sp = C.c_void_p(stream.cuda_stream)
    soup, grid = scenes.make_mesh("soup", a.tris), scenes.make_mesh("grid", a.tris)
    static_meshes = [api.Bvh.build_triangles(np.ascontiguousarray(m, np.float32)) for m in (soup, grid)]
    count = a.instances
    deforming = np.arange(count) % a.every == a.every - 1
    keys0, keys1 = moving_keys(count, seed=1)
    keys0, keys1 = keys0.astype(np.float32), keys1.astype(np.float32)
    rays = world_rays(np.concatenate([keys0, keys1]), a.width, a.height, np.float32)
    n = rays.shape[0]
    d_rays = cuda(rays)
    d_times = cuda(np.random.default_rng(5).uniform(0, 1, size=n).astype(np.float32))
    ws = torch.empty(64, dtype=torch.uint8, device="cuda")
    hits = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    inst = torch.empty(n, dtype=torch.int32, device="cuda")
    results = {}

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

    for move in a.move:
        k0, k1 = moved(soup, move)
        frozen_tris = (0.5 * k0.astype(np.float64) + 0.5 * k1.astype(np.float64)).astype(np.float32)
        frozen = api.Bvh.build_triangles(frozen_tris)
        # the deforming mesh: a tree over prepare_motion_triangles' boxes, its motion nodes
        d_k0, d_k1 = cuda(k0), cuda(k1)
        nt = k0.shape[0]
        tboxes = torch.empty((nt, 6), dtype=torch.float32, device="cuda")
        tcentres = torch.empty((nt, 3), dtype=torch.float32, device="cuda")
        check(D, D.ddi_bottom3f(None, ptr(d_k0), ptr(d_k1), nt, ptr(tboxes), ptr(tcentres), None, None, 0, sp), "ddi")
        torch.cuda.synchronize()
        mesh = api.Bvh.build_boxes(tboxes.data_ptr(), tcentres.data_ptr(), count=nt, dtype=np.float32, flags=api.DEVICE_POINTERS)
        nodes = torch.zeros((mesh.node_count + 1) * D.ddi_motion_node_bytes3f(), dtype=torch.uint8, device="cuda")
        bws = torch.empty(2 * (mesh.node_count + 1) * 4 + 16, dtype=torch.uint8, device="cuda")

        def bottom_step():
            check(D, D.ddi_bottom3f(None, ptr(d_k0), ptr(d_k1), nt, ptr(tboxes), ptr(tcentres), None, None, 0, sp), "ddi")
            mesh.refit_boxes(tboxes.data_ptr(), api.DEVICE_POINTERS)
            check(D, D.ddi_bottom3f(C.c_void_p(mesh.handle), ptr(d_k0), ptr(d_k1), nt, None, None, ptr(nodes), ptr(bws), bws.numel(), sp),
                  "ddi")

        bottom_step()
        torch.cuda.synchronize()

        # meshes: 0 soup, 1 grid, 2 the frozen soup, 3 the deforming soup
        handles = (C.c_void_p * 4)(static_meshes[0].handle, static_meshes[1].handle, frozen.handle, mesh.handle)
        vk0 = (C.c_void_p * 4)(None, None, None, d_k0.data_ptr())
        vk1 = (C.c_void_p * 4)(None, None, None, d_k1.data_ptr())
        mn = (C.c_void_p * 4)(None, None, None, nodes.data_ptr())
        base_mesh = (np.arange(count) % 2).astype(np.uint32)

        def ddi_scene(kind):
            """records (kind of the deforming copies: 0 frozen static, 1 shutter boxes, 2 motion nodes), boxes, top"""
            mesh_of = np.where(deforming, 2 if kind == 0 else 3, base_mesh).astype(np.uint32)
            kinds = np.where(deforming, kind, 0).astype(np.int32)
            recs = torch.zeros(count * D.ddi_record_bytes3f(), dtype=torch.uint8, device="cuda")
            depth = SZ(0)
            torch.cuda.synchronize()
            check(D, D.ddi_records3f(handles, mesh_of.ctypes.data, kinds.ctypes.data, keys0.ctypes.data, keys1.ctypes.data, vk0, vk1, mn,
                                     count, ptr(recs), C.byref(depth), sp), "ddi")
            boxes = torch.empty((count, 6), dtype=torch.float32, device="cuda")
            centres = torch.empty((count, 3), dtype=torch.float32, device="cuda")
            check(D, D.ddi_prepare3f(ptr(recs), count, depth.value, ptr(boxes), ptr(centres), sp), "ddi")
            torch.cuda.synchronize()
            top = api.Bvh.build_boxes(boxes.data_ptr(), centres.data_ptr(), count=count, dtype=np.float32, flags=api.DEVICE_POINTERS)
            return recs, depth.value, boxes, centres, top

        def ddi_run(sc):
            recs, depth, _, _, top = sc
            check(D, D.ddi_plain3f(C.c_void_p(top.handle), ptr(recs), count, depth, ptr(d_rays), ptr(d_times), n, ptr(hits), ptr(inst),
                                   ptr(ws), 64, sp), "ddi")

        scenes_by_arm = {"static": ddi_scene(0), "shutter": ddi_scene(1), "nodes": ddi_scene(2)}
        mesh_list = [static_meshes[0], static_meshes[1], frozen]
        frozen_scene = MotionScene(M, api, mesh_list, np.where(deforming, 2, base_mesh), keys0, keys1, np.float32)
        static_only = MotionScene(M, api, static_meshes, base_mesh[~deforming], keys0[~deforming], keys1[~deforming], np.float32)
        def_ids = np.ascontiguousarray(np.nonzero(deforming)[0], np.uint32)
        nodes_recs = scenes_by_arm["nodes"][0]

        def run_frozen():
            check(M, M.dmi_plain3f(C.c_void_p(frozen_scene.top.handle), ptr(frozen_scene.records), frozen_scene.count, frozen_scene.max_depth,
                                   ptr(d_rays), ptr(d_times), n, ptr(hits), ptr(inst), ptr(ws), 64, sp), "dmi")

        def run_workaround():
            check(D, D.ddi_workaround3f(C.c_void_p(static_only.top.handle), ptr(static_only.records), static_only.count,
                                        static_only.max_depth, C.c_void_p(mesh.handle), ptr(d_k0), ptr(d_k1), ptr(nodes), ptr(nodes_recs),
                                        def_ids.ctypes.data, def_ids.size, ptr(d_rays), ptr(d_times), n, ptr(hits), ptr(inst), ptr(ws),
                                        64, sp), "ddi")

        def run_frame():
            recs, depth, boxes, centres, top = scenes_by_arm["nodes"]
            bottom_step()
            check(D, D.ddi_prepare3f(ptr(recs), count, depth, ptr(boxes), ptr(centres), sp), "ddi")
            top.refit_boxes(boxes.data_ptr(), api.DEVICE_POINTERS)

        # the closest hits of the two deforming bottom kinds, and the hit fractions
        out = {}
        for arm in ("shutter", "nodes"):
            ddi_run(scenes_by_arm[arm])
            torch.cuda.synchronize()
            out[arm] = (host(hits).view(np.uint32).copy(), host(inst).copy())
        run_workaround()
        torch.cuda.synchronize()
        out["workaround"] = (host(hits).view(np.uint32).copy(), host(inst).copy())
        differ = int((~((out["shutter"][0][:, :2] == out["nodes"][0][:, :2]).all(axis=1) & (out["shutter"][1] == out["nodes"][1]))).sum())
        hit_fraction = float((out["nodes"][0][:, 0] != 0xFFFFFFFF).mean())
        wk_t = out["workaround"][0][:, 1].view(np.float32)
        nd_t = out["nodes"][0][:, 1].view(np.float32)
        t_differ = int((wk_t.view(np.uint32) != nd_t.view(np.uint32)).sum())

        t = {"frozen": timed(run_frozen), "static": timed(lambda: ddi_run(scenes_by_arm["static"])),
             "shutter": timed(lambda: ddi_run(scenes_by_arm["shutter"])), "nodes": timed(lambda: ddi_run(scenes_by_arm["nodes"])),
             "workaround": timed(run_workaround), "frame": timed(run_frame)}
        results[str(move)] = {"ms": {k: round(v, 3) for k, v in t.items()},
                              "mrays_per_s": {k: round(n / v / 1e3, 1) for k, v in t.items() if k != "frame"},
                              "hit_fraction": hit_fraction, "shutter_vs_nodes_differ": differ, "workaround_t_differ": t_differ}
        print(f"# {gpu}; {count} copies, {int(deforming.sum())} deforming by {move} triangle sizes, {n} rays")
        for k in ("frozen", "static", "shutter", "nodes", "workaround"):
            print(f"{k:10s} {t[k]:8.3f} ms  {n / t[k] / 1e3:8.1f} Mrays/s")
        print(f"frame      {t['frame']:8.3f} ms  (bottom step + prepare_deforming_instances + top refit)")
        print(f"hit fraction {hit_fraction:.3f}; shutter vs nodes records differ on {differ} rays; workaround t differs on {t_differ}")
        for sc in scenes_by_arm.values():
            sc[4].destroy()
        frozen_scene.top.destroy()                          # (its meshes are shared: destroyed below)
        static_only.top.destroy()
        mesh.destroy()
        frozen.destroy()
    print(json.dumps({"gpu": gpu, "instances": count, "deforming": int(deforming.sum()), "rays": n, "by_move": results}))
    for m in static_meshes:
        m.destroy()
    api.set_stream(None)


if __name__ == "__main__":
    main()
