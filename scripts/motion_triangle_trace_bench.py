"""The motion form of DeviceView::trace_triangles (deforming meshes) against the static call on the same mesh.

Per scene (soup-1M and grid-1M, bvh_b200/scenes.py): key 0 is the mesh, key 1 the mesh moved by a smooth field of about
`--amplitude` triangle sizes (default 1: tests/test_device_motion_triangle_gpu.py moving_keys); `--width` x `--height` primary rays of the
scene's camera, in pixel order, each at a random time in [0, 1].  Timed with CUDA events, float, closest-hit, every hit
accepted, median of `--reps` after a warm-up (tests/device_motion_triangle_kernels.cu dmt_plain3f):
  static   trace_triangles on a tree built from the triangles at tau = 0.5 (triangle_at), triangles attached
  equal    the motion call with both keys the tau = 0.5 vertices (one pointer), on a tree from prepare_motion_triangles'
           boxes: the cost of loading and blending two keys per triangle test
  motion   the motion call with the moving keys at the rays' times, on the tree of their shutter boxes: adds the looser
           boxes
  frame    one frame of updates: prepare_motion_triangles + bvh3f_refit_boxes, against bvh3f_refit_triangles of the static
           tree, both stream-ordered with device pointers
  equal_nodes  the motion-node call (prepare_motion_nodes, two key boxes per child) with the equal keys: the cost of the
           blended inner step (tests/device_motion_nodes_kernels.cu dmn_plain3f)
  nodes    the motion-node call with the moving keys: each child's box at the ray's time, on the same topology
  nodes_frame  one frame of motion nodes: prepare_motion_nodes alone (the topology stays)
Before timing: `equal` must equal `static` bit for bit on every ray (with equal keys the boxes, so the tree, and the
triangles are the static ones), and `motion` must equal one thread per ray nesting DeviceView::intersect with a
triangle_at leaf on the first 1M rays; `equal_nodes` must equal `equal` bit for bit, and `nodes` one thread per ray through
a node_at node test on the first 1M rays.  Also prints traversal counts per ray (inner steps and triangle tests, one
thread per ray: the same decisions as the batched kernels) for the static tree, the shutter-box tree and the motion
nodes, and the card's name and power limit with the numbers, and one JSON line per scene.

    python scripts/motion_triangle_trace_bench.py [--tris 1000000] [--width 3163 --height 3163] [--reps 10] [--amplitude 1]
    python scripts/motion_triangle_trace_bench.py --ptxas    # registers and spills of the motion kernels (no GPU needed)
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


def kernel_row(name):
    """(kernel, "T, flags", static | motion | motion nodes, shader) of a demangled kernel name"""
    name = name.replace("(anonymous namespace)::", "").replace("bvh::v2::cuda::detail::", "")
    kernel = re.match(r"void bvh::v2::cuda::(\w+)<", name)
    body, depth, args, cur = name[kernel.end():], 0, [], ""
    for ch in body:                      # the template arguments, split at top-level commas
        if ch == "<":
            depth += 1
        elif ch == ">":
            if depth == 0:
                break
            depth -= 1
        if ch == "," and depth == 0:
            args.append(cur.strip())
            cur = ""
        else:
            cur += ch
    args.append(cur.strip())
    shader = args[-1]
    form = "motion" if shader.startswith("MotionShader<") else "static"
    if form == "motion":
        shader = shader[len("MotionShader<"):-1].split(",", 1)[1].strip()
    if shader.startswith("WithMotionNodes<"):
        form, shader = "motion nodes", shader[len("WithMotionNodes<"):-1].split(",", 1)[1].strip()
    return kernel.group(1), ", ".join(args[:-1]), form, shader


def ptxas_table():
    """Compiles tests/device_motion_triangle_kernels.cu and tests/device_motion_nodes_kernels.cu with the library's flags
    and -Xptxas=-v into a temporary directory and prints registers and spills of the triangle and path kernels, static,
    under a MotionShader and with motion nodes."""
    from bvh_b200 import build_ext
    flags = ["-std=c++20" if f == "-std=c++17" else f for f in build_ext.NVCC_FLAGS]
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    lines = []
    for src in (build_ext.MOTION_TRIANGLE_KERNELS_SRC, build_ext.MOTION_NODES_KERNELS_SRC):
        with tempfile.TemporaryDirectory() as tmp:
            res = subprocess.run([nvcc, *flags, "-Xcompiler", "-march=x86-64-v3", "-Xptxas=-v", "-c", src, "-o", os.path.join(tmp, "k.o")],
                                 capture_output=True, text=True)
        if res.returncode:
            sys.exit(res.stderr)
        lines += res.stderr.splitlines()
    rows, name = [], None
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        m = re.search(r"Used (\d+) registers", line)
        if m and name and ("device_view_triangle_kernel" in name or "device_view_path_kernel" in name):
            spill = next((x for x in lines[i - 2:i] if "spill" in x), "")
            s = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", spill)
            g = kernel_row(name)
            rows.append((g, int(m.group(1)), s.group(1) if s else "0", s.group(2) if s else "0"))
    print("| kernel | T, flags | form | shader | registers | spill stores | spill loads |")
    print("|---|---|---|---|---|---|---|")
    for g, regs, st, ld in sorted(set(rows), key=lambda r: r[0]):
        print("| " + " | ".join(g) + f" | {regs} | {st} | {ld} |")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=3163)
    ap.add_argument("--height", type=int, default=3163)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--scenes", default="soup,grid")
    ap.add_argument("--amplitude", type=float, default=1.0, help="key 1's motion, in triangle sizes")
    ap.add_argument("--ptxas", action="store_true")
    a = ap.parse_args()
    if a.ptxas:
        ptxas_table()
        return
    import torch
    import bvh_b200.api as api
    from bvh_b200 import build_ext, scenes
    from tests.test_device_motion_triangle_gpu import MOTION, PER_THREAD, Scene, cuda, deform, host, ptr, tri_size

    api.lib()
    assert api.device_count() > 0, "needs a CUDA device"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True).stdout.strip()
    P, SZ = C.c_void_p, C.c_size_t
    M = C.CDLL(build_ext.build_device_motion_triangle_tests())
    M.dmt_prepare3f.argtypes = [P, P, SZ, P, P, P]
    M.dmt_triangle_at3f.argtypes = [P, P, SZ, C.c_float, P, P]
    M.dmt_run3f.argtypes = [P, P, P, SZ, C.c_int, C.c_int, C.c_uint, P, P, SZ] + [P] * 7 + [P, SZ, P]
    M.dmt_plain3f.argtypes = [P, P, P, SZ, C.c_int, P, P, SZ, P, P, SZ, P]
    M.dmt_steps3f.argtypes = [P, P, P, SZ, C.c_int, P, P, SZ, P, P, P]
    M.dmt_last_error.restype = C.c_char_p
    N = C.CDLL(build_ext.build_device_motion_nodes_tests())
    N.dmn_prepare3f.argtypes = [P, P, P, SZ, P, P, SZ, P]
    N.dmn_run3f.argtypes = [P, P, P, SZ, P, SZ, C.c_int, C.c_int, C.c_uint, P, P, SZ] + [P] * 9 + [P, SZ, P]
    N.dmn_plain3f.argtypes = [P, P, P, SZ, P, SZ, P, P, SZ, P, P, SZ, P]
    N.dmn_last_error.restype = C.c_char_p

    def check(rc):
        if rc:
            raise RuntimeError(M.dmt_last_error().decode())

    def check_nodes(rc):
        if rc:
            raise RuntimeError(N.dmn_last_error().decode())

    def motion_nodes(scene):
        """prepare_motion_nodes of a scene's tree: (records, workspace, prepare)"""
        nc = scene.bvh.node_count
        nodes = torch.zeros((nc + 1) * 64, dtype=torch.uint8, device="cuda")
        bu = torch.empty(2 * (nc + 1) * 4, dtype=torch.uint8, device="cuda")

        def prepare():
            check_nodes(N.dmn_prepare3f(C.c_void_p(scene.bvh.handle), ptr(scene.k0), ptr(scene.k1), scene.count, ptr(nodes), ptr(bu),
                                        bu.numel(), sp))
        prepare()
        return nodes, nc, prepare

    # every handle, call and event on one stream, so that the events time the work
    stream = torch.cuda.Stream()
    api.set_stream(stream.cuda_stream)
    torch.cuda.set_stream(stream)
    sp = C.c_void_p(stream.cuda_stream)
    print(f"# {gpu}")
    for kind in a.scenes.split(","):
        tris = scenes.make_mesh(kind, a.tris)
        key0, key1 = tris, deform(tris, 1, a.amplitude * tri_size(tris))
        moving = Scene(M, api, key0, key1, stream=sp)
        mid = moving.triangle_at(0.5)                          # the vertices at tau = 0.5, as the motion call rounds them
        equal = Scene(M, api, mid, mid, same=True, stream=sp)
        static = api.Bvh.build_triangles(mid)
        d_mid = equal.k0
        count = tris.shape[0]
        rays = scenes.make_primary(kind, a.width, a.height)
        n = rays.shape[0]
        d_rays = cuda(rays)
        d_half = cuda(np.full(n, 0.5, np.float32))
        d_times = cuda(np.random.default_rng(5).uniform(0, 1, size=n).astype(np.float32))
        hits = [torch.empty((n, 4), dtype=torch.float32, device="cuda") for _ in range(5)]
        moving_nodes, node_count, run_nodes_frame = motion_nodes(moving)
        equal_nodes, equal_node_count, _ = motion_nodes(equal)
        ws = torch.empty(64, dtype=torch.uint8, device="cuda")

        def run_static():
            check(M.dmt_plain3f(C.c_void_p(static.handle), None, None, count, 1, ptr(d_rays), None, n, ptr(hits[0]), ptr(ws), 64, sp))

        def run_equal():
            check(M.dmt_plain3f(C.c_void_p(equal.bvh.handle), ptr(d_mid), ptr(d_mid), count, 0, ptr(d_rays), ptr(d_half), n,
                                ptr(hits[1]), ptr(ws), 64, sp))

        def run_motion():
            check(M.dmt_plain3f(C.c_void_p(moving.bvh.handle), ptr(moving.k0), ptr(moving.k1), count, 0, ptr(d_rays), ptr(d_times), n,
                                ptr(hits[2]), ptr(ws), 64, sp))

        def run_equal_nodes():
            check_nodes(N.dmn_plain3f(C.c_void_p(equal.bvh.handle), ptr(d_mid), ptr(d_mid), count, ptr(equal_nodes), equal_node_count,
                                      ptr(d_rays), ptr(d_half), n, ptr(hits[3]), ptr(ws), 64, sp))

        def run_nodes():
            check_nodes(N.dmn_plain3f(C.c_void_p(moving.bvh.handle), ptr(moving.k0), ptr(moving.k1), count, ptr(moving_nodes), node_count,
                                      ptr(d_rays), ptr(d_times), n, ptr(hits[4]), ptr(ws), 64, sp))

        def run_frame():
            moving.prepare(sp)
            moving.bvh.refit_boxes(moving.boxes.data_ptr(), api.DEVICE_POINTERS)

        def run_refit():
            static.refit_triangles(d_mid.data_ptr(), api.DEVICE_POINTERS)

        for f in (run_static, run_equal, run_motion, run_equal_nodes, run_nodes):
            f()
        torch.cuda.synchronize()
        h0, h1, h2, h3, h4 = (host(h).view(np.uint32) for h in hits)
        differ = int((~(h0 == h1).all(axis=1)).sum())
        assert differ == 0, f"{differ} rays differ between the static and the equal-keys motion call"
        differ = int((~(h1 == h3).all(axis=1)).sum())
        assert differ == 0, f"{differ} rays differ between the equal-keys motion call and its motion-node form"
        m = min(n, 1 << 20)
        ref = moving.run(PER_THREAD, d_rays, d_times, m, 0, 0, stream=sp)
        want = np.stack([ref[0].view(np.uint32), ref[1].view(np.uint32), ref[2].view(np.uint32), ref[3].view(np.uint32)], axis=1)
        bad = int((~(h2[:m] == want).all(axis=1)).sum())
        assert bad == 0, f"{bad} of {m} motion rays differ from the nested triangle_at reference"
        outs = [torch.empty(m, dtype=dt, device="cuda") for dt in (torch.int32, torch.float32, torch.float32, torch.float32)]
        inner, tests = (torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2))
        check_nodes(N.dmn_run3f(C.c_void_p(moving.bvh.handle), ptr(moving.k0), ptr(moving.k1), count, ptr(moving_nodes), node_count, 2, 0, 0,
                                ptr(d_rays), ptr(d_times), m, *[ptr(x) for x in outs], None, None, None, None, None, ptr(ws), 64, sp))
        torch.cuda.synchronize()
        want = np.stack([host(x).view(np.uint32) for x in outs], axis=1)
        bad = int((~(h4[:m] == want).all(axis=1)).sum())
        assert bad == 0, f"{bad} of {m} motion-node rays differ from the node_at reference"
        hit_static, hit_motion = float((h0[:, 0] != 0xFFFFFFFF).mean()), float((h2[:, 0] != 0xFFFFFFFF).mean())

        counts = {}
        for name, handle, k0, k1, motion, times in (("static", static.handle, None, None, 0, d_half),
                                                    ("motion", moving.bvh.handle, moving.k0, moving.k1, 1, d_times)):
            check(M.dmt_steps3f(C.c_void_p(handle), ptr(k0), ptr(k1), count, motion, ptr(d_rays), ptr(times), n, ptr(inner), ptr(tests), sp))
            torch.cuda.synchronize()
            counts[name] = {"inner_steps": round(float(host(inner).mean()), 2), "tri_tests": round(float(host(tests).mean()), 2)}
        check_nodes(N.dmn_run3f(C.c_void_p(moving.bvh.handle), ptr(moving.k0), ptr(moving.k1), count, ptr(moving_nodes), node_count, 2, 0, 0,
                                ptr(d_rays), ptr(d_times), n, None, None, None, None, None, None, None, ptr(inner), ptr(tests), ptr(ws), 64,
                                sp))
        torch.cuda.synchronize()
        counts["nodes"] = {"inner_steps": round(float(host(inner).mean()), 2), "tri_tests": round(float(host(tests).mean()), 2)}

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

        t = {"static": timed(run_static), "equal": timed(run_equal), "motion": timed(run_motion), "equal_nodes": timed(run_equal_nodes),
             "nodes": timed(run_nodes), "frame": timed(run_frame), "nodes_frame": timed(run_nodes_frame), "refit_triangles": timed(run_refit)}
        arms = ("static", "equal", "motion", "equal_nodes", "nodes")
        out = {"gpu": gpu, "scene": f"{kind}-{count}", "amplitude": a.amplitude, "rays": n,
               "hit_fraction": {"static": hit_static, "motion": hit_motion}, "per_ray": counts, "ms": {k: round(v, 3) for k, v in t.items()},
               "mrays_per_s": {k: round(n / t[k] / 1e3, 1) for k in arms}}
        print(f"## {kind}-{count}, {n} rays, amplitude {a.amplitude} triangle sizes")
        for k in arms:
            print(f"{k:12s} {t[k]:8.3f} ms  {n / t[k] / 1e3:8.1f} Mrays/s")
        print(f"frame    {t['frame']:8.3f} ms  (prepare_motion_triangles + refit_boxes); refit_triangles {t['refit_triangles']:.3f} ms")
        print(f"nodes_frame {t['nodes_frame']:8.3f} ms  (prepare_motion_nodes)")
        for k, c in counts.items():
            print(f"{k:8s} {c['inner_steps']:8.2f} inner steps  {c['tri_tests']:8.2f} triangle tests per ray")
        print(json.dumps(out))
        del moving_nodes, equal_nodes
        static.destroy()
        equal.destroy()
        moving.destroy()
    api.set_stream(None)


if __name__ == "__main__":
    main()
