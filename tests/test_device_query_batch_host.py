"""DeviceView::query (include/bvh/v2/cuda/intersect.cuh) compiled by g++ as host code, no GPU needed.

On the golden trees of the unmodified reference and on a one-primitive tree, a recording querier makes per query the
node and leaf calls Bvh<Node>::traverse_top_down of the C++ surface makes, with the same arguments in the same order, for
overlap, containment with IsAnyHit, a nearest search whose leaf shrinks the radius the node test reads, reject-all and
accept-all, with the two-argument and the three-argument node function (tests/device_query_batch_host_test.cpp).  start
and finish run once per query, an empty batch makes no call, and the scheduling settings are 8 / 8."""
import os
import re
import subprocess

import numpy as np
import pytest

from tests.conftest import golden
from tests.test_device_query_host import queries, tri_boxes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDES = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "bvh_b200", "csrc")]
OVERLAP, CONTAINS, NEAREST, REJECT_ALL, ACCEPT_ALL = range(5)


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "device_query_batch_host_test")
    src = os.path.join(ROOT, "tests", "device_query_batch_host_test.cpp")
    csrc = os.path.join(ROOT, "bvh_b200", "csrc")
    deps = [src, os.path.join(ROOT, "tests", "device_queries.h"), os.path.join(ROOT, "include", "bvh", "v2", "cuda", "intersect.cuh"),
            os.path.join(ROOT, "include", "bvh", "v2", "b200_surface.h"), os.path.join(ROOT, "include", "bvh_b200_device.h")]
    deps += [os.path.join(csrc, f) for f in ("traverse_core.cuh", "core.cuh", "persistent_core.cuh", "trace_plan.h")]
    if not os.path.exists(out) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(out):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["g++", "-std=gnu++20", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-Wall", "-Werror",
                               *INCLUDES, src, "-o", out])
    return out


def run_case(exe, tmp_path, bounds, index, prim_ids, boxes, qs):
    dtype = boxes.dtype
    rec = np.dtype([("bounds", dtype, 6), ("index", np.uint32 if dtype == np.float32 else np.uint64)])
    nodes = np.zeros(bounds.shape[0], rec)
    nodes["bounds"], nodes["index"] = bounds, index
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(np.array([nodes.shape[0], prim_ids.shape[0], qs.shape[0]], np.uint64).tobytes())
        f.write(nodes.tobytes())
        f.write(np.asarray(prim_ids, np.uint64).tobytes())
        f.write(np.ascontiguousarray(boxes).tobytes())
        f.write(np.ascontiguousarray(qs).tobytes())
    res = subprocess.run([exe, str(path), "d" if dtype == np.float64 else "f"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "empty batch ok, small workspace throws, null workspace throws" in res.stdout, res.stdout
    lines = {}
    for line in res.stdout.splitlines():
        m = re.match(r"kind (\d) form (\d) mismatches 0 events (\d+) starts_ok 1 finishes_ok 1$", line)
        if m:
            lines[int(m[1]), int(m[2])] = int(m[3])
    assert len(lines) == 10, res.stdout
    return lines


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "box12_f32", "soup1k_f64"])
def test_call_sequences_match_reference(exe, tmp_path, name):
    g = golden(name)
    boxes = tri_boxes(g["tris"])
    qs = queries(boxes, boxes.dtype)
    index = g["ref_index"].astype(np.uint64)
    events = run_case(exe, tmp_path, g["ref_bounds"], index, g["ref_prim_ids"], boxes, qs)
    leaves = int(((index & 15) != 0).sum())
    m = qs.shape[0]
    assert events[ACCEPT_ALL, 0] == m * (2 * leaves - 1)            # every inner node and every leaf, once
    assert events[REJECT_ALL, 1] == m                               # the root's node call only
    for kind in (OVERLAP, CONTAINS, NEAREST):
        assert events[kind, 0] == events[kind, 1] > m, kind


def test_one_primitive_tree(exe, tmp_path):
    """The root is a leaf: every query gets one leaf call and no node call."""
    boxes = np.array([[0, 0, 0, 1, 1, 1]], np.float32)
    bounds = np.array([[0, 1, 0, 1, 0, 1]], np.float32)
    qs = queries(np.concatenate([boxes, boxes + 0.5]), np.float32, m=40)
    events = run_case(exe, tmp_path, bounds, np.array([1], np.uint64), np.array([0], np.uint64), boxes, qs)
    for key, count in events.items():
        assert count == 40, key


def test_plan_query(exe):
    out = subprocess.run([exe, "plan"], capture_output=True, text=True, check=True).stdout.strip()
    assert out == "refill_min 8 inner_budget 8"
