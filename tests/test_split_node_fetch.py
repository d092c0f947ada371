"""For float closest-hit rays the traversal step tests the x/y half of each child box first and loads the z half only
when that half does not already reject the box (traverse_core.cuh inner_step; other rays load whole nodes).  These tests check that it takes the decision of the full box
test: which children are hit, which is entered first and which index is pushed, on adversarial rays and boxes, and
that whole traversals keep the reference's hits and step counters, on the host emulation and on the GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from bvh_b200 import scenes
from oracle.pyoracle import ANY_HIT, ROBUST, TIE_LOWEST_ID
from tests.conftest import golden
from tests.helpers import ROOT, aligned_zeros, assert_hits_equal, hits_tuple

MODES = [("closest", TIE_LOWEST_ID), ("any", ANY_HIT | TIE_LOWEST_ID), ("robust", ROBUST | TIE_LOWEST_ID)]


@pytest.fixture(scope="module")
def step_lib():
    src = os.path.join(ROOT, "tests", "split_step_check.cpp")
    out_dir = os.path.join(ROOT, "tests", "_build")
    out = os.path.join(out_dir, "libsplit_step_check.so")
    csrc = os.path.join(ROOT, "bvh_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("core.cuh", "traverse_core.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(out_dir, exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fPIC", "-shared",
                               "-x", "c++", "-I", csrc, src, "-o", out])
    lib = C.CDLL(out)
    for s in ("3f", "3d"):
        getattr(lib, f"split_step_check_{s}").argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]
    return lib


def adversarial_cases(dtype, m, seed):
    """Sibling pairs and rays where the halves matter: axis-parallel rays (zero and -0 direction components, whose
    fast slab test meets inf - inf), rays starting on box faces, degenerate, inverted and unbounded boxes, tiny
    direction components (clamped inverse), and tmin / tmax set exactly to a box face."""
    rng = np.random.RandomState(seed)
    big = np.finfo(dtype).max
    org = rng.uniform(-1, 1, (m, 3)).astype(dtype)
    d = rng.uniform(-1, 1, (m, 3)).astype(dtype)
    pick = rng.randint(0, 6, (m, 3))
    d[pick == 0] = 0.0
    d[pick == 1] = -0.0
    d[pick == 2] = np.sign(d[pick == 2]) * dtype(1e-30 if dtype == np.float64 else 1e-9)
    lo = rng.uniform(-1.5, 1.5, (m, 2, 3)).astype(dtype)
    hi = lo + rng.uniform(0, 1, (m, 2, 3)).astype(dtype)
    kind = rng.randint(0, 8, (m, 2, 3))
    on_face = kind == 0                                       # a face through the ray's origin
    lo[on_face] = np.broadcast_to(org[:, None, :], lo.shape)[on_face]
    hi[kind == 1] = lo[kind == 1]                             # flat
    inverted = kind == 2                                      # empty along that axis
    lo[inverted], hi[inverted] = hi[inverted], lo[inverted] - dtype(0.25)
    lo[kind == 3], hi[kind == 3] = -np.inf, np.inf            # unbounded
    hi[kind == 4] = big
    nodes = aligned_zeros((3 * m, 8), dtype)
    view = nodes.reshape(m, 3, 8)
    view[:, 1:, 0:6:2], view[:, 1:, 1:6:2] = lo, hi
    it = np.uint32 if dtype == np.float32 else np.uint64
    ids = view[:, 1:, 6].view(it)
    ids[:, 0] = (np.arange(m, dtype=it) * 2 + 7) << 4        # any distinct inner / leaf indices
    ids[:, 1] = ((np.arange(m, dtype=it) * 2 + 8) << 4) | 3
    rays = np.zeros((m, 8), dtype)
    rays[:, 0:3], rays[:, 3:6] = org, d
    rays[:, 6] = np.where(rng.rand(m) < 0.5, dtype(0.0), dtype(-0.0))
    rays[:, 7] = rng.choice(np.array([np.inf, big, 0.5, 2.0], dtype), m)
    face = rng.randint(0, 3, m).astype(np.uint8)              # 1: tmax on a far plane, 2: tmin on a near plane
    return nodes, rays, face


@pytest.mark.parametrize("robust", [False, True])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_split_step_takes_the_full_test_decision(step_lib, dtype, robust):
    m = 200_000
    nodes, rays, face = adversarial_cases(dtype, m, seed=3 + robust)
    out = np.zeros((m, 4), np.uint64)
    fn = getattr(step_lib, "split_step_check_3f" if dtype == np.float32 else "split_step_check_3d")
    fn(nodes.ctypes.data, rays.ctypes.data, face.ctypes.data, m, int(robust), out.ctypes.data)
    bad = np.nonzero((out[:, 0] != out[:, 2]) | (out[:, 1] != out[:, 3]))[0]
    assert bad.size == 0, f"{bad.size} steps differ from the full test, first {bad[:8]}"
    # the cases cover every outcome: both children, one, none, and both orders
    top, pushed = out[:, 2], out[:, 3]
    it = np.uint32 if dtype == np.float32 else np.uint64
    ids = nodes.reshape(m, 3, 8)[:, 1:, 6].view(it).astype(np.uint64)
    both = pushed != np.uint64(np.iinfo(it).max)              # nothing pushed: all ones of the index type
    assert (both & (top == ids[:, 1])).any() and (both & (top == ids[:, 0])).any()
    assert (~both & (top == ids[:, 0])).any() and (~both & (top == ids[:, 1])).any()
    assert (~both & (top != ids[:, 0]) & (top != ids[:, 1])).any()


def adversarial_rays(tris, m, dtype, seed):
    rng = np.random.RandomState(seed)
    lo, hi = tris.reshape(-1, 3).min(axis=0), tris.reshape(-1, 3).max(axis=0)
    rays = np.zeros((m, 8), dtype)
    rays[:, 0:3] = rng.uniform(lo - 0.1, hi + 0.1, (m, 3))
    rays[:, 3:6] = rng.uniform(-1, 1, (m, 3))
    pick = rng.randint(0, 5, (m, 3))
    rays[:, 3:6][pick == 0] = 0.0
    rays[:, 3:6][pick == 1] = -0.0
    snap = rng.rand(m) < 0.3                                  # origins on vertex coordinates: rays in box faces
    v = tris.reshape(-1, 3)[rng.randint(0, tris.shape[0] * 3, m)]
    axis = rng.randint(0, 3, m)
    rays[snap, axis[snap]] = v[snap, axis[snap]]
    rays[:, 6] = np.where(rng.rand(m) < 0.5, 0.0, -0.0)
    rays[:, 7] = rng.choice(np.array([np.inf, np.finfo(dtype).max, 0.3], dtype), m)
    return rays


@pytest.mark.parametrize("name", ["soup2k_f32", "grid2k_f32", "soup1k_f64"])
def test_golden_trees_keep_hits_and_counters(emul, oracle, name):
    """Whole traversals of the reference's own trees with the split step: hits and step counters of the oracle."""
    g = golden(name)
    tris = g["tris"]
    tree = emul.from_reference(g["ref_bounds"], g["ref_index"], g["ref_prim_ids"], tris)
    otree = oracle.from_arrays(g["ref_bounds"], g["ref_index"], g["ref_prim_ids"])
    oracle.set_triangles(otree, tris)
    for rays in (g["rays"], adversarial_rays(tris, 20000, tris.dtype, seed=5)):
        for mode, flags in MODES:
            got = emul.trace(tree, rays, flags)
            want = oracle.trace(otree, rays, flags=flags, stats=True)
            assert_hits_equal(got[:4], want[:4], f"{name}/{mode}")
            assert (got[4] == want[4]).all(), f"{name}/{mode}: step counters differ"


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n,dtype", [("soup", 20000, np.float32), ("grid", 20000, np.float32), ("soup", 8000, np.float64)])
def test_gpu_split_step_keeps_hits_and_counters(gpu_lib, oracle, kind, n, dtype):
    """The device kernels with the split step (persistent and statistics kernels) on adversarial rays: the oracle's
    hits and step counters on the GPU-built tree."""
    api = gpu_lib
    tris = scenes.make_mesh(kind, n, dtype=dtype)
    bvh = api.Bvh.build_triangles(tris)
    bounds, index_values, prim_ids = bvh.arrays()
    otree = oracle.from_arrays(bounds, index_values, prim_ids)
    oracle.set_triangles(otree, tris)
    rays = adversarial_rays(tris, 50000, dtype, seed=7)
    for mode, oflags in MODES:
        flags = (api.ANY_HIT if oflags & ANY_HIT else 0) | (api.ROBUST if oflags & ROBUST else 0)
        want = oracle.trace(otree, rays, flags=oflags, stats=True)
        hits, st = bvh.intersect_rays(rays, flags=flags, stats=True)
        assert_hits_equal(hits_tuple(hits), want[:4], f"{kind}/{mode}/stats kernel")
        assert (st["inner_steps"] == want[4][:, 0]).all() and (st["prim_tests"] == want[4][:, 2]).all()
        assert_hits_equal(hits_tuple(bvh.intersect_rays(rays, flags=flags)), want[:4], f"{kind}/{mode}/persistent")
    bvh.destroy()
