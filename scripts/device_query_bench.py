"""Times a build from device-resident boxes and two queries written on DeviceView::traverse_top_down, on 1M spheres.

    python scripts/device_query_bench.py [--steps 20] [--warmup 3] [--n 1000000]

Prints the card's name and power limit, then one JSON line with the median of `steps` calls after `warmup` of
  build_boxes_ms    bvh3f_build_boxes on n sphere boxes and centres already on the device (BVH_DEVICE_POINTERS); host
                    clock around the call, which ends with the build's own synchronisation
  build_host_ms     bvh3f_build on the same values in host arrays (the copy to the device included); same clock
  overlap_ms        the broad phase: every sphere's box queried against the tree, counting the overlapping boxes
                    (tests/device_query_kernels.cu overlap_kernel, one thread per query), with the per-thread array stack
                    (`_array`) and the shared-memory stack (`_shared`); CUDA events on the handle's stream
  nearest_ms        the nearest sphere centre to each of n random points in the unit cube (nearest_kernel), both stacks;
                    CUDA events
  overlap_ms_query, nearest_ms_query  the same two queries as batches through DeviceView::query on the persistent
                    scheduler (tests/device_query_batch_kernels.cu); before they are timed, their outputs are checked equal
                    to the per-thread kernels' (query_matches_per_thread)
and the number of overlapping pairs the broad phase found (each unordered pair of distinct spheres once).  Nothing is
written to the tree except the test kernels' build under tests/_build when it is stale.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--n", type=int, default=1_000_000)
    args = ap.parse_args()

    import torch
    import bvh_b200.api as api
    from bvh_b200 import build_ext
    from tests.test_device_query_gpu import sphere_boxes
    dq = C.CDLL(build_ext.build_device_query_tests())
    P, SZ = C.c_void_p, C.c_size_t
    dq.dq_overlap3f.argtypes = [P, P, P, SZ, C.c_int, P, P, P, P, P]
    dq.dq_nearest3f.argtypes = [P, P, P, SZ, C.c_int, P, P, P, P, P]
    dq.dq_last_error.restype = C.c_char_p
    dqb = C.CDLL(build_ext.build_device_query_batch_tests())
    dqb.dqb_query3f.argtypes = [P, C.c_int, C.c_int, C.c_int, P, P, SZ, P, P, P, P, P, P, P, SZ, P]
    dqb.dqb_last_error.restype = C.c_char_p
    api.set_device(0)
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream()
    api.set_stream(stream.cuda_stream)                    # the handles' work and the timing events on one stream
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)

    def host_timed(fn):
        ms = []
        for k in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            bvh = fn()
            t1 = time.perf_counter()
            bvh.destroy()
            if k >= args.warmup:
                ms.append(1e3 * (t1 - t0))
        return float(np.median(ms))

    def event_timed(fn):
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
    boxes, centers = sphere_boxes(n, np.float32)
    d_boxes, d_centers = torch.from_numpy(boxes).cuda(), torch.from_numpy(centers).cuda()
    torch.cuda.synchronize()
    row = {"n": n}
    row["build_boxes_ms"] = host_timed(lambda: api.Bvh.build_boxes(d_boxes.data_ptr(), d_centers.data_ptr(), count=n,
                                                                   dtype=np.float32, flags=api.DEVICE_POINTERS))
    row["build_host_ms"] = host_timed(lambda: api.Bvh.build(boxes, centers))

    bvh = api.Bvh.build_boxes(d_boxes.data_ptr(), d_centers.data_ptr(), count=n, dtype=np.float32, flags=api.DEVICE_POINTERS)
    counts = torch.zeros(n, dtype=torch.int32, device="cuda")
    ids = torch.zeros(n, dtype=torch.int32, device="cuda")
    dist2 = torch.zeros(n, dtype=torch.float32, device="cuda")
    points = torch.from_numpy(np.random.default_rng(2).random((n, 3), dtype=np.float32)).cuda()

    def check(rc):
        if rc:
            raise RuntimeError(dq.dq_last_error().decode())

    for stack, label in ((0, "array"), (1, "shared")):
        row[f"overlap_ms_{label}"] = event_timed(lambda: check(dq.dq_overlap3f(
            C.c_void_p(bvh.handle), d_boxes.data_ptr(), d_boxes.data_ptr(), n, stack, counts.data_ptr(), None, None, None, None)))
        row[f"overlap_pairs_{label}"] = (int(counts.sum().item()) - n) // 2      # a box overlaps itself
        row[f"nearest_ms_{label}"] = event_timed(lambda: check(dq.dq_nearest3f(
            C.c_void_p(bvh.handle), d_centers.data_ptr(), points.data_ptr(), n, stack, ids.data_ptr(), dist2.data_ptr(),
            None, None, None)))
    # the same queries through DeviceView::query: outputs checked equal to the per-thread kernels' first, then timed
    ws = torch.empty(8, dtype=torch.uint8, device="cuda")
    idsums = torch.zeros(n, dtype=torch.int64, device="cuda")

    def batch(kind, prims, queries, r0, r1):
        rc = dqb.dqb_query3f(C.c_void_p(bvh.handle), kind, 0, 0, prims.data_ptr(), queries.data_ptr(), n, r0.data_ptr(),
                             r1.data_ptr(), None, None, None, None, ws.data_ptr(), 8, None)
        if rc:
            raise RuntimeError(dqb.dqb_last_error().decode())

    check(dq.dq_overlap3f(C.c_void_p(bvh.handle), d_boxes.data_ptr(), d_boxes.data_ptr(), n, 0, counts.data_ptr(),
                          idsums.data_ptr(), None, None, None))
    check(dq.dq_nearest3f(C.c_void_p(bvh.handle), d_centers.data_ptr(), points.data_ptr(), n, 0, ids.data_ptr(),
                          dist2.data_ptr(), None, None, None))
    want = [t.clone() for t in (counts, idsums, ids, dist2)]
    q_counts, q_idsums, q_ids, q_dist2 = (torch.zeros_like(t) for t in want)
    batch(0, d_boxes, d_boxes, q_counts, q_idsums)
    batch(1, d_centers, points, q_ids, q_dist2)
    torch.cuda.synchronize()
    row["query_matches_per_thread"] = all(bool(torch.equal(a, b)) for a, b in
                                          zip(want[:3] + [want[3].view(torch.int32)],
                                              [q_counts, q_idsums, q_ids, q_dist2.view(torch.int32)]))
    row["overlap_ms_query"] = event_timed(lambda: batch(0, d_boxes, d_boxes, q_counts, q_idsums))
    row["nearest_ms_query"] = event_timed(lambda: batch(1, d_centers, points, q_ids, q_dist2))
    row["depth"] = bvh.depth
    row["card"], row["power_limit"] = name, power
    print(json.dumps(row), flush=True)
    bvh.destroy()
    api.set_stream(None)
    return row


if __name__ == "__main__":
    main()
