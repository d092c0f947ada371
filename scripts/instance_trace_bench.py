"""DeviceView::trace_instances against the ways to trace the same scene without it.

The scene: `--instances` copies (alternately of soup-64k and grid-64k, each randomly rotated and scaled on a grid of
cells; 256 copies give about 16.8M placed triangles) and `--width` x `--height` primary rays from below, in pixel order.
Timed with CUDA events, float, closest-hit, every hit accepted, median of `--reps` after a warm-up:
  instances  trace_instances over the top tree of the copies (tests/device_instance_trace_kernels.cu dit_plain3f)
  flattened  trace_triangles over one tree built from all placed triangles in world space (dit_plain_triangles3f)
  nested     DeviceView::trace with a tracer whose leaf runs each copy's bottom tree through intersect with a per-thread
             stack (dit_nested_trace3f), what a caller writes without trace_instances
  frame      one rigid-motion frame of the top level: prepare_instances + bvh3f_refit_boxes, stream-ordered
Before timing, the records of `instances` and `nested` are checked equal bit for bit, and the (instance, id) of
`flattened` against them: the flattened triangles are rounded in world space, so a few rays may differ at edges and
ties; their count is printed.  Prints the card's name and power limit with the numbers, and one JSON line.

    python scripts/instance_trace_bench.py [--instances 256] [--width 2048 --height 2048] [--reps 10]
    python scripts/instance_trace_bench.py --ptxas      # registers and spills of the instance kernels (no GPU needed)
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
    """Compiles tests/device_instance_trace_kernels.cu with the library's flags and -Xptxas=-v into a temporary
    directory and prints registers and spills of every instance and triangle kernel."""
    from bvh_b200 import build_ext
    flags = ["-std=c++20" if f == "-std=c++17" else f for f in build_ext.NVCC_FLAGS]
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, *flags, "-Xcompiler", "-march=x86-64-v3", "-Xptxas=-v", "-c", build_ext.INSTANCE_TRACE_KERNELS_SRC,
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
        if m and name and ("instance_kernel" in name or "triangle_kernel" in name):
            spill = next((x for x in lines[i - 2:i] if "spill" in x), "")
            s = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", spill)
            kind = re.match(r"void bvh::v2::cuda::(\w+)<(\w+), (\w+), (\w+), (\w+), \(anonymous namespace\)::(\w+(?:<[^>]*>)?)", name)
            rows.append((kind.groups() if kind else (name,), int(m.group(1)), s.group(1) if s else "0", s.group(2) if s else "0"))
    print("| kernel | T | any | robust | last | shader | registers | spill stores | spill loads |")
    print("|---|---|---|---|---|---|---|---|---|")
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
    from bvh_b200 import scenes
    from tests.test_device_instance_trace_gpu import Scene, check, cuda, host, placements, ptr, world_rays, world_triangles

    api.lib()
    assert api.device_count() > 0, "needs a CUDA device"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True).stdout.strip()
    from bvh_b200 import build_ext
    L = C.CDLL(build_ext.build_device_instance_trace_tests())
    P, SZ = C.c_void_p, C.c_size_t
    for s in ("3f", "3d"):
        getattr(L, f"dit_records{s}").argtypes = [P, P, P, SZ, P, C.POINTER(SZ), P]
        getattr(L, f"dit_prepare{s}").argtypes = [P, SZ, SZ, P, P, P]
        getattr(L, f"dit_record_bytes{s}").restype = SZ
    L.dit_plain3f.argtypes = [P, P, SZ, SZ, P, SZ, P, P, P, SZ, P]
    L.dit_plain_triangles3f.argtypes = [P, P, SZ, P, P, SZ, P]
    L.dit_nested_trace3f.argtypes = [P, P, SZ, P, SZ, P, P, P, SZ, P]
    L.dit_last_error.restype = C.c_char_p

    # every handle, call and event on one stream, so that the events time the work
    stream = torch.cuda.Stream()
    api.set_stream(stream.cuda_stream)
    torch.cuda.set_stream(stream)
    sp = C.c_void_p(stream.cuda_stream)
    meshes = [scenes.make_mesh("soup", a.tris), scenes.make_mesh("grid", a.tris)]
    mats = placements(a.instances, seed=1)
    mesh_of = np.arange(a.instances) % 2
    scene = Scene(L, api, meshes, mesh_of, mats, np.float32)
    flat_tris = world_triangles(meshes, mesh_of, mats).reshape(-1, 9).astype(np.float32)
    flat = api.Bvh.build_triangles(flat_tris)
    offsets = np.concatenate([[0], np.cumsum([meshes[k].shape[0] for k in mesh_of])])
    rays = world_rays(mats, a.width, a.height, np.float32)
    n = rays.shape[0]
    d_rays = cuda(rays)
    hits = [torch.empty((n, 4), dtype=torch.float32, device="cuda") for _ in range(3)]
    insts = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2)]
    ws = torch.empty(64, dtype=torch.uint8, device="cuda")
    top = C.c_void_p(scene.top.handle)

    def run_instances():
        check(L, L.dit_plain3f(top, ptr(scene.records), scene.count, scene.max_depth, ptr(d_rays), n, ptr(hits[0]), ptr(insts[0]),
                               ptr(ws), 64, sp))

    def run_flat():
        check(L, L.dit_plain_triangles3f(C.c_void_p(flat.handle), ptr(d_rays), n, ptr(hits[1]), ptr(ws), 64, sp))

    def run_nested():
        check(L, L.dit_nested_trace3f(top, ptr(scene.records), scene.max_depth, ptr(d_rays), n, ptr(hits[2]), ptr(insts[1]), ptr(ws),
                                      64, sp))

    def run_frame():
        scene.prepare(sp)
        scene.top.refit_boxes(scene.boxes.data_ptr(), api.DEVICE_POINTERS)

    # outputs first: instances == nested bit for bit; flattened (instance, id) against them
    for f in (run_instances, run_flat, run_nested):
        f()
    torch.cuda.synchronize()
    h0, h1, h2 = (host(h).view(np.uint32) for h in hits)
    i0, i1 = host(insts[0]).view(np.uint32), host(insts[1]).view(np.uint32)
    assert (h0 == h2).all() and (i0 == i1).all(), "trace_instances and the nested tracer differ"
    hit = h0[:, 0] != 0xFFFFFFFF
    flat_id = np.where(hit, offsets[np.minimum(i0, a.instances - 1)] + h0[:, 0], 0xFFFFFFFF)
    differ = int((flat_id != h1[:, 0]).sum())
    assert differ <= n // 1000, f"{differ} rays differ between the flattened and the instanced scene"

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

    def tree_bytes(bvh):
        return bvh.node_count * 32 + bvh.prim_count * (4 + 48)

    t = {"instances": timed(run_instances), "flattened": timed(run_flat), "nested": timed(run_nested), "frame": timed(run_frame)}
    inst_bytes = sum(tree_bytes(m) for m in scene.meshes) + tree_bytes(scene.top) + scene.count * scene.rec_bytes
    out = {"gpu": gpu, "instances": a.instances, "placed_triangles": int(flat_tris.shape[0]), "rays": n,
           "hit_fraction": float(hit.mean()), "flat_differ": differ,
           "ms": {k: round(v, 3) for k, v in t.items()},
           "mrays_per_s": {k: round(n / t[k] / 1e3, 1) for k in ("instances", "flattened", "nested")},
           "bytes": {"instanced": int(inst_bytes), "flattened": int(tree_bytes(flat))}}
    print(f"# {gpu}")
    for k in ("instances", "flattened", "nested"):
        print(f"{k:10s} {t[k]:8.3f} ms  {n / t[k] / 1e3:8.1f} Mrays/s")
    print(f"frame      {t['frame']:8.3f} ms  (prepare_instances + refit_boxes, {a.instances} instances)")
    print(f"memory     instanced {inst_bytes / 2**20:.1f} MiB, flattened {tree_bytes(flat) / 2**20:.1f} MiB")
    print(json.dumps(out))
    flat.destroy()
    scene.destroy()
    api.set_stream(None)


if __name__ == "__main__":
    main()
