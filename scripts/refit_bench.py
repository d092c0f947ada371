"""Times a GPU refit against the host path it replaces, on 1M primitives.

    python scripts/refit_bench.py [--steps 20] [--warmup 3] [--n 1000000]

Prints the card's name and power limit, then one JSON line with the median of `steps` calls after `warmup` of
  refit_boxes_ms      bvh3f_refit_boxes, device pointers, on a tree over n sphere boxes (CUDA events on the handle's
                      stream around the call)
  refit_triangles_ms  bvh3f_refit_triangles, device pointers, on the n-triangle soup (CUDA events)
  host_path_ms        the same sphere refit without bvh3f_refit_boxes: leaf boxes written into the host mirror (one
                      NumPy assignment through the bvh3f_get_node pointer, what a C loop over bvh_node3f_set_bbox does),
                      bvh3f_refit (serial host pass), then the re-upload the next batched call makes (bvh3f_get_device_view
                      uploads like every batched call); host clock around the whole, which ends synchronised.  The leaf
                      boxes are folded from the primitive boxes before the timed region.
The work is the same in both sphere timings: after the last call the two trees are checked to be bit-identical.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

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


def sphere_boxes(n, seed):
    rng = np.random.default_rng(seed)
    centers = rng.random((n, 3), dtype=np.float32)
    radii = (0.5 + rng.random(n, dtype=np.float32)) * np.float32(0.5 / np.cbrt(n))
    return np.concatenate([centers - radii[:, None], centers + radii[:, None]], axis=1), centers


def leaf_bounds(index_values, prim_ids, boxes):
    """Leaf boxes (minx, maxx, ...) folded from primitive boxes in BVH order (BBox::extend); inner rows unused."""
    first, count = (index_values >> np.uint64(4)).astype(np.int64), (index_values & np.uint64(15)).astype(np.int64)
    big = np.finfo(np.float32).max
    lo = np.full((index_values.shape[0], 3), big, np.float32)
    hi = np.full((index_values.shape[0], 3), -big, np.float32)
    ids = prim_ids.astype(np.int64)
    for j in range(int(count.max())):
        m = count > j
        b = boxes[ids[first[m] + j]]
        lo[m] = np.where(lo[m] < b[:, :3], lo[m], b[:, :3])
        hi[m] = np.where(hi[m] > b[:, 3:], hi[m], b[:, 3:])
    out = np.zeros((index_values.shape[0], 6), np.float32)
    out[:, 0::2], out[:, 1::2] = lo, hi
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--n", type=int, default=1_000_000)
    args = ap.parse_args()

    import torch
    import bvh_b200.api as api
    from bvh_b200 import scenes
    api.set_device(0)
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream()
    api.set_stream(stream.cuda_stream)                    # the handles' work and the timing events on one stream
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

    n = args.n
    boxes, centers = sphere_boxes(n, seed=1)
    moved, _ = sphere_boxes(n, seed=2)                    # every sphere somewhere else: the leaf boxes all change
    spheres = api.Bvh.build(boxes, centers)
    d_moved = torch.from_numpy(moved).cuda()
    row = {"n": n, "refit_boxes_ms": timed(lambda: spheres.refit_boxes(d_moved.data_ptr(), api.DEVICE_POINTERS))}

    tris = scenes.soup(n)
    soup = api.Bvh.build_triangles(tris)
    d_verts = torch.from_numpy(tris + np.float32(0.001)).cuda()
    row["refit_triangles_ms"] = timed(lambda: soup.refit_triangles(d_verts.data_ptr(), api.DEVICE_POINTERS))
    soup.destroy()

    host = api.Bvh.build(boxes, centers)
    _, index_values, prim_ids = host.arrays()
    leaves = np.nonzero((index_values & 15) != 0)[0]
    new_leaf_bounds = leaf_bounds(index_values, prim_ids, moved)[leaves]
    rec = np.dtype([("bounds", np.float32, 6), ("index", np.uint32)])
    count = index_values.shape[0]

    def host_path():
        base = host._f("get_node")(host.handle, 0)
        mirror = np.ctypeslib.as_array((C.c_char * (count * rec.itemsize)).from_address(base)).view(rec)
        mirror["bounds"][leaves] = new_leaf_bounds
        host.refit()
        host.device_view()

    ms = []
    for k in range(args.warmup + args.steps):
        t0 = time.perf_counter()
        host_path()
        if k >= args.warmup:
            ms.append(1e3 * (time.perf_counter() - t0))
    row["host_path_ms"] = float(np.median(ms))
    same = (spheres.arrays()[0].view(np.uint32) == host.arrays()[0].view(np.uint32)).all()
    row["host_path_over_refit_boxes"] = row["host_path_ms"] / row["refit_boxes_ms"]
    row["trees_bit_identical"] = bool(same)
    row["card"], row["power_limit"] = name, power
    print(json.dumps(row), flush=True)
    spheres.destroy(); host.destroy()
    api.set_stream(None)
    if not same:
        raise SystemExit("the GPU refit and the host path gave different trees")
    return row


if __name__ == "__main__":
    main()
