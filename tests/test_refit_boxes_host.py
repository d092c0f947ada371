"""bvhNN_refit_boxes without a GPU: the exported symbols, the header, the Python binding's checks, and the refit pass of
bvh_b200/csrc/refit_core.cuh compiled by g++ (tests/refit_host_test.cpp) on trees the reference built, against the
plain-C restatement of the reference's refit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDES = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "bvh_b200", "csrc")]
LIB = os.path.join(ROOT, "bvh_b200", "libbvh_c.so")


def fold_leaf_boxes(index_values, prim_ids, boxes, dtype):
    """Node bounds (minx, maxx, ...) with every leaf's box folded from its primitives' boxes in BVH order the way
    BBox::extend does it (robust_min / robust_max, accumulator first, from +-max); inner nodes are zero."""
    index_values = np.asarray(index_values, np.uint64)
    first, count = (index_values >> np.uint64(4)).astype(np.int64), (index_values & np.uint64(15)).astype(np.int64)
    big = np.finfo(dtype).max
    lo = np.full((index_values.shape[0], 3), big, dtype)
    hi = np.full((index_values.shape[0], 3), -big, dtype)
    ids = np.asarray(prim_ids, np.int64)
    for j in range(int(count.max())):
        m = count > j
        b = boxes[ids[first[m] + j]]
        lo[m] = np.where(lo[m] < b[:, :3], lo[m], b[:, :3])
        hi[m] = np.where(hi[m] > b[:, 3:], hi[m], b[:, 3:])
    out = np.zeros((index_values.shape[0], 6), dtype)
    out[:, 0::2], out[:, 1::2] = lo, hi
    out[count == 0] = 0
    return out


def random_boxes(n, dtype, seed):
    """Boxes around points of the unit cube, a tenth of them points (min == max) and a twentieth far outside."""
    rng = np.random.default_rng(seed)
    c = rng.random((n, 3))
    h = 0.01 * rng.random((n, 3))
    h[rng.random(n) < 0.1] = 0
    far = rng.random(n) < 0.05
    c[far] += rng.choice([-1e6, 1e6, 1e30], size=(int(far.sum()), 3))
    return np.concatenate([c - h, c + h], axis=1).astype(dtype)


@pytest.fixture(scope="module")
def exe():
    out = os.path.join(ROOT, "tests", "_build", "refit_host_test")
    src = os.path.join(ROOT, "tests", "refit_host_test.cpp")
    deps = [src] + [os.path.join(ROOT, "bvh_b200", "csrc", f) for f in ("refit_core.cuh", "build_core.cuh", "core.cuh")]
    if not os.path.exists(out) or max(os.path.getmtime(d) for d in deps) > os.path.getmtime(out):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["g++", "-std=gnu++20", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-Wall", "-Werror",
                               *INCLUDES, src, "-o", out])
    return out


def host_refit(exe, tmp_path, index_values, prim_ids, boxes, order):
    dtype = boxes.dtype
    path, out_path = tmp_path / "case.bin", tmp_path / "out.bin"
    with open(path, "wb") as f:
        f.write(np.array([index_values.shape[0], prim_ids.shape[0], order.shape[0]], np.uint64).tobytes())
        f.write(np.asarray(index_values, np.uint64).tobytes())
        f.write(np.asarray(prim_ids, np.uint64).tobytes())
        f.write(np.ascontiguousarray(boxes).tobytes())
        f.write(np.asarray(order, np.uint64).tobytes())
    res = subprocess.run([exe, str(path), "d" if dtype == np.float64 else "f", str(out_path)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return np.fromfile(out_path, dtype).reshape(-1, 6)


def bits(a):
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


@pytest.mark.parametrize("key", ["optimize_3f_300", "optimize_3f_3000", "optimize_3d_300", "optimize_3d_3000"])
def test_pass_matches_reference_refit(exe, tmp_path, oracle, key):
    """Leaves processed in index order and in a shuffled order (the GPU's arrival order is arbitrary): both equal the
    reference's refit of the folded leaf boxes, bit for bit."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "reference_trees.npz"))
    index_values, prim_ids = g[key + "_index"].astype(np.uint64), g[key + "_ids"].astype(np.uint64)
    dtype = np.float32 if "_3f_" in key else np.float64
    boxes = random_boxes(prim_ids.shape[0], dtype, seed=len(key) + prim_ids.shape[0])
    tree = oracle.from_arrays(fold_leaf_boxes(index_values, prim_ids, boxes, dtype), index_values, prim_ids)
    oracle.refit(tree)
    want = tree.arrays()[0]
    rng = np.random.default_rng(11)
    for order in (np.arange(index_values.shape[0]), rng.permutation(index_values.shape[0])):
        got = host_refit(exe, tmp_path, index_values, prim_ids, boxes, order)
        assert (bits(got) == bits(want)).all(), f"{key}: first difference at node {np.nonzero(bits(got) != bits(want))[0][:4]}"


def test_pass_on_one_leaf_tree(exe, tmp_path):
    """The root is a leaf: its box is the fold of all primitives' boxes."""
    boxes = random_boxes(5, np.float32, seed=1)
    index_values, prim_ids = np.array([5], np.uint64), np.array([3, 0, 4, 1, 2], np.uint64)
    got = host_refit(exe, tmp_path, index_values, prim_ids, boxes, np.array([0]))
    assert (bits(got) == bits(fold_leaf_boxes(index_values, prim_ids, boxes, np.float32))).all()


def test_library_exports_refit_boxes():
    if not os.path.exists(LIB):
        from bvh_b200 import build_ext
        build_ext.build()
    lib = C.CDLL(LIB)
    assert hasattr(lib, "bvh3f_refit_boxes") and hasattr(lib, "bvh3d_refit_boxes")


def test_device_header_compiles_as_c11():
    src = ("#include <bvh_b200_device.h>\n"
           "int (*f)(struct bvh3f*, const struct bvh_bbox3f*, size_t, unsigned) = bvh3f_refit_boxes;\n"
           "int (*d)(struct bvh3d*, const struct bvh_bbox3d*, size_t, unsigned) = bvh3d_refit_boxes;\n"
           "int main(void) { return 0; }\n")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), "-x", "c", "-"],
                   input=src, text=True, check=True)


def test_binding_raises_without_a_tree():
    """No CPU fallback: without a device there is no handle, and the call fails loudly; a malformed array is refused
    before it reaches the library."""
    from bvh_b200 import api
    bvh = object.__new__(api.Bvh)
    bvh.handle, bvh.dtype, bvh.s = None, np.dtype(np.float32), "3f"
    with pytest.raises(api.BvhError, match="null handle"):
        bvh.refit_boxes(np.zeros((4, 6), np.float32))
    with pytest.raises(ValueError):
        bvh.refit_boxes(np.zeros((4, 3), np.float32))
