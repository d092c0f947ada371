"""Times DeviceView::traverse_bottom_up and the refit built on the same climb, on 1M sphere boxes (float).

    python scripts/bottom_up_bench.py [--steps 20] [--warmup 3] [--n 1000000] [--baseline-lib OTHER/libbvh_c.so]

Prints the card's name and power limit, then one JSON line with the median of `steps` calls after `warmup` of
  refit_boxes_ms       bvh3f_refit_boxes, device pointers, every sphere moved (CUDA events on the handle's stream).  With
                       --baseline-lib, the refit is timed in child processes that alternate between that library and
                       this tree's (BVH_B200_LIB), three rounds each: refit_boxes_ms then lists this build's three medians
                       and baseline_refit_boxes_ms the other's, and trees_identical says whether both builds refitted
                       to the same bits
  count_box_ms         the pass with subtree primitive counts and box unions (tests/device_bottom_up.h CountBox)
  mass_ms              the pass with subtree mass and centre of mass (MassCentre)
  barnes_hut_ms        the softened potential at every particle, theta = 0.5, through traverse_top_down with the
                       three-argument node test (Potential), one thread per particle
  barnes_hut_query_ms  the same potential as one batch through DeviceView::query (tests/device_query_batch_kernels.cu)
  *_bvh_order_ms       both again with the particles queried in BVH order (query i takes particle prim_ids[i])
                       instead of their random original order
                       Before each pair is timed, its potentials are checked equal bit for bit (barnes_hut_match,
                       barnes_hut_bvh_order_match)
The passes include their link kernel and workspace set-up; they run the test kernels of tests/device_bottom_up_kernels.cu
(built by build()).
"""
import argparse
import ctypes as C
import hashlib
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


def sphere_boxes(n, seed):
    rng = np.random.default_rng(seed)
    centers = rng.random((n, 3), dtype=np.float32)
    radii = (0.5 + rng.random(n, dtype=np.float32)) * np.float32(0.5 / np.cbrt(n))
    return np.concatenate([centers - radii[:, None], centers + radii[:, None]], axis=1), centers


def setup():
    import torch
    import bvh_b200.api as api
    api.set_device(0)
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream()
    api.set_stream(stream.cuda_stream)                    # the handles' work and the timing events on one stream
    return torch, api, stream


def timer(torch, stream, steps, warmup):
    def timed(fn):
        for _ in range(warmup):
            fn()
        ms = []
        for _ in range(steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fn()
            b.record(stream)
            b.synchronize()
            ms.append(a.elapsed_time(b))
        return float(np.median(ms))
    return timed


def refit_only(args):
    """One library's refit timing and a digest of the refitted tree, as one JSON line."""
    torch, api, stream = setup()
    timed = timer(torch, stream, args.steps, args.warmup)
    boxes, centers = sphere_boxes(args.n, seed=1)
    moved, _ = sphere_boxes(args.n, seed=2)
    bvh = api.Bvh.build(boxes, centers)
    d_moved = torch.from_numpy(moved).cuda()
    ms = timed(lambda: bvh.refit_boxes(d_moved.data_ptr(), api.DEVICE_POINTERS))
    bounds, index, ids = bvh.arrays()
    digest = hashlib.sha256(bounds.tobytes() + index.tobytes() + ids.tobytes()).hexdigest()[:16]
    print(json.dumps({"refit_boxes_ms": ms, "tree": digest}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--baseline-lib", default="")
    ap.add_argument("--refit-only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.refit_only:
        return refit_only(args)

    torch, api, stream = setup()
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    timed = timer(torch, stream, args.steps, args.warmup)
    n = args.n
    row = {"n": n}

    if args.baseline_lib:
        this_lib = os.path.join(ROOT, "bvh_b200", "libbvh_c.so")
        runs = {"this": [], "baseline": []}
        for _ in range(3):
            for which, lib in (("baseline", os.path.abspath(args.baseline_lib)), ("this", this_lib)):
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--refit-only", "--n", str(n), "--steps",
                                      str(args.steps), "--warmup", str(args.warmup)], env=dict(os.environ, BVH_B200_LIB=lib),
                                     capture_output=True, text=True, check=True).stdout
                runs[which].append(json.loads(out.strip().splitlines()[-1]))
        row["refit_boxes_ms"] = [r["refit_boxes_ms"] for r in runs["this"]]
        row["baseline_refit_boxes_ms"] = [r["refit_boxes_ms"] for r in runs["baseline"]]
        row["trees_identical"] = len({r["tree"] for r in runs["this"] + runs["baseline"]}) == 1

    from bvh_b200 import build_ext
    bu = C.CDLL(build_ext.build_device_bottom_up_tests())
    P, SZ = C.c_void_p, C.c_size_t
    bu.bu_workspace_bytes3f.argtypes = [P, C.POINTER(C.c_size_t)]
    bu.bu_count_box3f.argtypes = [P, P, SZ, P, P, P]
    bu.bu_mass3f.argtypes = [P, P, SZ, P, P, P, P]
    bu.bu_potential3f.argtypes = [P, P, P, P, P, P, SZ, C.c_float, C.c_float, P, P]
    bu.bu_last_error.restype = C.c_char_p

    boxes, centers = sphere_boxes(n, seed=1)
    moved, _ = sphere_boxes(n, seed=2)
    bvh = api.Bvh.build(boxes, centers)
    if not args.baseline_lib:
        d_moved = torch.from_numpy(moved).cuda()
        row["refit_boxes_ms"] = timed(lambda: bvh.refit_boxes(d_moved.data_ptr(), api.DEVICE_POINTERS))
    bvh.refit_boxes(boxes)                                # the boxes the passes read
    h = C.c_void_p(bvh.handle)
    nbytes = C.c_size_t(0)
    assert bu.bu_workspace_bytes3f(h, C.byref(nbytes)) == 0
    nodes = bvh.node_count
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device="cuda")
    d_boxes, d_pos = torch.from_numpy(boxes).cuda(), torch.from_numpy(centers).cuda()
    d_mass = torch.from_numpy((0.5 + np.random.default_rng(3).random(n)).astype(np.float32)).cuda()
    counts = torch.empty(nodes, dtype=torch.int32, device="cuda")
    node_boxes = torch.empty((nodes, 6), dtype=torch.float32, device="cuda")
    node_mass = torch.empty(nodes, dtype=torch.float32, device="cuda")
    node_centre = torch.empty((nodes, 3), dtype=torch.float32, device="cuda")
    phi = torch.empty(n, dtype=torch.float32, device="cuda")

    def ok(rc):
        assert rc == 0, bu.bu_last_error()

    row["count_box_ms"] = timed(lambda: ok(bu.bu_count_box3f(h, ws.data_ptr(), nbytes.value, d_boxes.data_ptr(), counts.data_ptr(),
                                                             node_boxes.data_ptr())))
    row["mass_ms"] = timed(lambda: ok(bu.bu_mass3f(h, ws.data_ptr(), nbytes.value, d_pos.data_ptr(), d_mass.data_ptr(),
                                                   node_mass.data_ptr(), node_centre.data_ptr())))
    eps2 = float((0.1 / np.cbrt(n)) ** 2)
    dqb = C.CDLL(build_ext.build_device_query_batch_tests())
    dqb.dqb_potential3f.argtypes = [P, P, P, P, P, P, SZ, C.c_float, C.c_float, P, P, P, SZ, P]
    dqb.dqb_last_error.restype = C.c_char_p
    ok(bu.bu_mass3f(h, ws.data_ptr(), nbytes.value, d_pos.data_ptr(), d_mass.data_ptr(), node_mass.data_ptr(),
                    node_centre.data_ptr()))
    cursor = torch.empty(8, dtype=torch.uint8, device="cuda")
    phi_query = torch.empty(n, dtype=torch.float32, device="cuda")

    def per_thread(points):
        ok(bu.bu_potential3f(h, d_pos.data_ptr(), d_mass.data_ptr(), node_mass.data_ptr(), node_centre.data_ptr(),
                             points.data_ptr(), n, 0.25, eps2, phi.data_ptr(), None))

    def batch(points):
        rc = dqb.dqb_potential3f(h, d_pos.data_ptr(), d_mass.data_ptr(), node_mass.data_ptr(), node_centre.data_ptr(),
                                 points.data_ptr(), n, 0.25, eps2, phi_query.data_ptr(), None, cursor.data_ptr(), 8, None)
        assert rc == 0, dqb.dqb_last_error()

    bvh_order = torch.from_numpy(bvh.arrays()[2].astype(np.int64)).cuda()
    for suffix, points in (("", d_pos), ("_bvh_order", d_pos[bvh_order].contiguous())):
        per_thread(points)
        batch(points)
        torch.cuda.synchronize()
        row[f"barnes_hut{suffix}_match"] = bool(torch.equal(phi.view(torch.int32), phi_query.view(torch.int32)))
        row[f"barnes_hut{suffix}_ms"] = timed(lambda: per_thread(points))
        row[f"barnes_hut_query{suffix}_ms"] = timed(lambda: batch(points))
    torch.cuda.synchronize()
    bounds = bvh.arrays()[0]
    row["count_box_matches_tree"] = bool((node_boxes.cpu().numpy().view(np.uint32) == bounds.view(np.uint32)).all())
    row["root_count"] = int(counts[0].item())
    row["card"], row["power_limit"] = name, power
    print(json.dumps(row))
    bvh.destroy()


if __name__ == "__main__":
    main()
