"""The GPU LBVH build against the NumPy model of tests/lattice_reference.py (pytest -m gpu).

The model fixes the whole Quality Low tree of a lattice scene from its Morton keys alone: primitive order, node ranges,
node boxes and depth.  It is checked against the host emulation in tests/test_build_reference_host.py.  Here the GPU
tree must equal it at the sizes where the build's parallel decomposition changes:
  2048-key radix sort tiles (kRsTile)                    2047, 2048, 2049
  8-tile look-back windows of the one-sweep sort         16383, 16384, 16385, 18433 (the window loop wraps above 16384)
  64-, 128-, 256-leaf blocks of the hierarchy kernel     63 ... 257
  2048-pair compaction tiles (kCompactTile)              2049 (2048 pairs), 2^21 + 2^11 + 1
  1024-thread single-block compaction scan               2^21 + 2^11 + 1 (1025 tiles: two rounds)
  automatic 63-bit keys and 8 sort passes                2^22 - 1 (30-bit) and 2^22 (63-bit)
and with key patterns that stress the sorts: equal keys (the rank of equal digits must be stable), keys that differ in
one radix digit only (every key of a tile in one bin in the other passes), input in and against key order."""
import math

import numpy as np
import pytest

from bvh_b200 import scenes
from tests import lattice_reference as L
from tests.helpers import assert_hits_equal, hits_tuple

pytestmark = pytest.mark.gpu

PATTERNS = ("distinct", "one_cell", "cells16", "low_digit", "high_digit", "sorted", "reversed")
SIZES = (1, 2, 3, 63, 64, 65, 127, 128, 129, 255, 256, 257, 2047, 2048, 2049, 16383, 16384, 16385, 18433, 300_007)
# the model takes seconds per scene at these sizes: a few patterns each
LARGE = ((2 ** 21 + 2 ** 11 + 1, ("distinct", "reversed", "low_digit")), (2 ** 22 - 1, ("one_cell", "high_digit")),
         (2 ** 22, ("distinct", "reversed", "high_digit")))
CASES = [(n, p) for n in SIZES for p in PATTERNS] + [(n, p) for n, ps in LARGE for p in ps]


def _check(bvh, ref, oracle, collapsed=False, prim_boxes=None, what=""):
    bounds, index_values, prim_ids = bvh.arrays()
    try:
        L.check_tree(ref, bounds, index_values, prim_ids, bvh.depth, collapsed=collapsed, prim_boxes=prim_boxes)
    except AssertionError as e:
        raise AssertionError(f"{what}: {e}") from None
    tree = oracle.from_arrays(bounds, index_values, prim_ids)
    assert oracle.check_invariants(tree, 8 if collapsed else 1) == 0, what


def _lattice(pattern, n, bits, dtype, seed=None):
    centres, extent = L.lattice_scene(pattern, n, bits, seed=n if seed is None else seed)
    boxes = L.boxes_around(centres, dtype)
    return centres.astype(dtype), boxes, L.Reference(centres, extent, bits, boxes)


@pytest.mark.parametrize("n,pattern", CASES)
def test_gpu_build_is_the_reference_tree(gpu_lib, oracle, n, pattern):
    """Boxes + centres, float, the automatic key width: with min_leaf_size = max_leaf_size = 1 the tree is the model's,
    node for node; with the default leaf settings every node is a node of the model (up to 300k primitives)."""
    api = gpu_lib
    bits = 63 if n >= 1 << 22 else 30
    centres, boxes, ref = _lattice(pattern, n, bits, np.float32)
    bvh = api.Bvh.build_boxes(boxes, centres, quality="low", min_leaf_size=1, max_leaf_size=1)
    assert bvh.get_property("morton_bits") == bits
    _check(bvh, ref, oracle, what=f"{pattern}, n={n}")
    if pattern == "one_cell" and n > 2:
        assert ref.depth <= math.ceil(math.log2(n)) + 2            # the index tie-break balances the run of equal keys
    if n <= 300_007:
        bvh = api.Bvh.build_boxes(boxes, centres, quality="low")
        _check(bvh, ref, oracle, collapsed=True, what=f"{pattern}, n={n}, default leaves")


@pytest.mark.parametrize("n", [1, 3, 65, 129, 257, 2049, 16385, 18433, 300_007])
def test_gpu_build_is_the_reference_tree_double(gpu_lib, oracle, n):
    """Double trees (the hierarchy kernel's 256-leaf blocks fall back to 128 for them)."""
    api = gpu_lib
    for pattern in ("distinct", "reversed", "low_digit"):
        centres, boxes, ref = _lattice(pattern, n, 30, np.float64)
        bvh = api.Bvh.build_boxes(boxes, centres, quality="low", min_leaf_size=1, max_leaf_size=1)
        _check(bvh, ref, oracle, what=f"{pattern}, n={n}, double")


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", [3, 129, 2049, 18433])
def test_gpu_build_from_triangles_is_the_reference_tree(gpu_lib, oracle, n, dtype):
    """Triangle input: the build computes each centre as ((v0 + v1) + v2) * fl(1/3); the scene's triangles put it on
    the lattice point exactly, so the same model applies, with the triangles' boxes."""
    api = gpu_lib
    for pattern in ("distinct", "cells16"):
        centres, extent = L.lattice_scene(pattern, n, 30, seed=n)
        tris = L.triangles_around(centres, dtype)
        ref = L.Reference(centres, extent, 30, L.triangle_boxes(tris))
        bvh = api.Bvh.build_triangles(tris, quality="low", min_leaf_size=1, max_leaf_size=1)
        _check(bvh, ref, oracle, what=f"{pattern}, n={n}, triangles")


def _rays_at(tris, m, seed):
    """m rays from random points around the scene to random points inside random triangles, and a few that miss."""
    rng = np.random.default_rng(seed)
    v = tris.reshape(-1, 3, 3).astype(np.float64)
    pick = rng.integers(0, v.shape[0], m)
    w = rng.dirichlet((1.0, 1.0, 1.0), m)
    target = np.einsum("mk,mkd->md", w, v[pick])
    org = target + rng.normal(size=(m, 3)) * (1.0 + rng.uniform(0, 8, (m, 1)))
    rays = np.zeros((m, 8))
    rays[:, :3], rays[:, 3:6], rays[:, 7] = org, target - org, 10.0
    rays[: m // 10, 3:6] = -rays[: m // 10, 3:6]                # pointing away
    return rays.astype(tris.dtype)


@pytest.mark.parametrize("n", [65, 4099])
def test_deep_chain_with_wide_keys(gpu_lib, oracle, n):
    """63-bit keys with one bit set each (cells 1, 2, 4, ... along the three axes, duplicated up to n): a caterpillar
    of about 63 levels above the duplicates' balanced runs.  The reported depth is the model's, and ROBUST rays through
    the tree find what brute force finds."""
    api = gpu_lib
    centres, extent = L.lattice_scene("chain", n, 63, seed=n)
    tris = L.triangles_around(centres, np.float32)
    ref = L.Reference(centres, extent, 63, L.triangle_boxes(tris))
    assert ref.depth >= 60
    api.set_option("morton_bits", 63)
    try:
        bvh = api.Bvh.build_triangles(tris, quality="low", min_leaf_size=1, max_leaf_size=1)
    finally:
        api.set_option("morton_bits", 0)
    assert bvh.get_property("morton_bits") == 63
    _check(bvh, ref, oracle, what=f"chain, n={n}")
    rays = _rays_at(tris, 400, seed=n)
    assert_hits_equal(hits_tuple(bvh.intersect_rays(rays, flags=api.ROBUST)), oracle.brute_force(tris, rays), f"chain, n={n}")


SWITCH_CASES = [(65, "reversed"), (129, "cells16"), (257, "reversed"), (2049, "low_digit"), (16385, "high_digit"),
                (18433, "reversed"), (300_007, "distinct")]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n,pattern", SWITCH_CASES)
def test_every_build_switch_gives_the_reference_tree(gpu_lib, oracle, n, pattern, dtype):
    """Every combination of sort_onesweep (one-sweep sort with decoupled look-back / histogram-scan-scatter passes),
    hierarchy (global flags only / 64- / 128- / 256-leaf blocks, 256 for float only) and morton_bits (30 / 63) gives
    the model's tree, not merely the same tree as the other combinations."""
    api = gpu_lib
    hierarchies = (0, 64, 128, 256) if dtype == np.float32 else (0, 64, 128)
    try:
        for bits in (30, 63):
            centres, boxes, ref = _lattice(pattern, n, bits, dtype)
            api.set_option("morton_bits", bits)
            for onesweep in (0, 1):
                api.set_option("sort_onesweep", onesweep)
                for hierarchy in hierarchies:
                    api.set_option("hierarchy", hierarchy)
                    bvh = api.Bvh.build_boxes(boxes, centres, quality="low", min_leaf_size=1, max_leaf_size=1)
                    assert bvh.get_property("morton_bits") == bits
                    _check(bvh, ref, oracle, what=f"{pattern}, n={n}, sort_onesweep {onesweep}, hierarchy {hierarchy}, {bits}-bit keys")
    finally:
        api.set_option("morton_bits", 0)
        api.set_option("sort_onesweep", 1)
        api.set_option("hierarchy", 128)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", [2049, 16385, 300_007])
def test_refit_boxes_are_the_reference_boxes(gpu_lib, oracle, n, dtype):
    """refit_boxes with new random boxes (in the original primitive order): topology and prim_ids stay, and every node
    box is the min / max of the new boxes over its range, bit for bit; with and without leaf collapse."""
    api = gpu_lib
    centres, boxes, ref = _lattice("reversed", n, 30, dtype)
    rng = np.random.default_rng(n)
    lo = rng.uniform(-50, 50, (n, 3)).astype(dtype)
    new = np.ascontiguousarray(np.concatenate([lo, lo + rng.uniform(0, 3, (n, 3)).astype(dtype)], axis=1))
    for leaves in ({"min_leaf_size": 1, "max_leaf_size": 1}, {}):
        bvh = api.Bvh.build_boxes(boxes, centres, quality="low", **leaves)
        collapsed = not leaves
        _check(bvh, ref, oracle, collapsed=collapsed, what=f"n={n}, before the refit")
        _, index_before, ids_before = bvh.arrays()
        bvh.refit_boxes(new)
        _, index_after, ids_after = bvh.arrays()
        assert np.array_equal(index_after, index_before) and np.array_equal(ids_after, ids_before)
        _check(bvh, ref, oracle, collapsed=collapsed, prim_boxes=new, what=f"n={n}, refit")


@pytest.mark.parametrize("quality", ["medium", "high"])
@pytest.mark.parametrize("n", [64, 65, 2049, 16385])
def test_treelet_qualities_keep_the_reference_tree_above_the_treelets(gpu_lib, oracle, n, quality):
    """Quality Medium / High rebuild every maximal subtree of at most 64 primitives by SAH.  Above those treelets the
    tree is the model's: every node of more than 64 primitives is a node of the model with the model's box, and each
    treelet holds the primitives of its range in the model.  The result is a valid BVH whose ROBUST answers are brute
    force's."""
    api = gpu_lib
    centres, extent = L.lattice_scene("cells16" if n < 2049 else "distinct", n, 30, seed=n)
    tris = L.triangles_around(centres, np.float32)
    ref = L.Reference(centres, extent, 30, L.triangle_boxes(tris))
    bvh = api.Bvh.build_triangles(tris, quality=quality)
    bounds, index_values, prim_ids = bvh.arrays()
    prim_ids = prim_ids.astype(np.int64)
    assert np.array_equal(np.sort(prim_ids), np.arange(n))
    first, count, levels = L.tree_ranges(index_values, n)
    above = np.nonzero(count > 64)[0]
    node = ref.find(first[above], count[above])
    assert (node >= 0).all(), "a node above the treelets is not a node of the model"
    assert (bounds[above].view(np.uint32) == ref.boxes[node].view(np.uint32)).all(), "a box above the treelets differs from the model's"
    # the children below the nodes of > 64 primitives partition the positions: same primitives in each part
    is_above = count > 64
    child = (index_values >> np.uint64(4)).astype(np.int64)
    parts = np.concatenate([child[above], child[above] + 1]) if above.size else np.zeros(1, np.int64)
    parts = parts[~is_above[parts]]
    assert count[parts].sum() == n
    segment = np.zeros(n, np.int64)
    segment[first[parts]] = 1
    segment = np.cumsum(segment)
    assert np.array_equal(prim_ids[np.lexsort((prim_ids, segment))], ref.order[np.lexsort((ref.order, segment))])
    assert oracle.check_invariants(oracle.from_arrays(bounds, index_values, prim_ids), 8) == 0
    rays = _rays_at(tris, 400, seed=n)
    assert_hits_equal(hits_tuple(bvh.intersect_rays(rays, flags=api.ROBUST)), oracle.brute_force(tris, rays), f"{quality}, n={n}")


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_sorted_rays_at_sort_tile_edges(gpu_lib, dtype):
    """SORT_RAYS orders the batch by the one-sweep radix sort of the build, over 30-bit keys of the ray origins.  The
    planner sorts batches of 2^16 rays and more (trace_plan.h), so the counts are 2^16 plus the tile edges: whole
    2048-key tiles, one key more or less, whole 8-tile look-back windows and one more.  Every hit record must be written
    and be bit-identical to the unsorted call's; a third of the rays share one origin (equal keys)."""
    api = gpu_lib
    tris = scenes.soup(30_000, seed=6).astype(dtype)
    bvh = api.Bvh.build_triangles(tris)
    big = scenes.incoherent_rays(tris.astype(np.float32), (1 << 16) + 18433, seed=2).astype(dtype)
    big[::3, :3] = big[0, :3]
    for m in [(1 << 16) + d for d in (0, 1, 2047, 2048, 2049, 16384, 16385, 18433)]:
        rays = np.ascontiguousarray(big[:m])
        out = []
        for flags in (0, api.SORT_RAYS):
            hits = np.empty(m, api.HIT3F if dtype == np.float32 else api.HIT3D)
            hits.view(np.uint8)[:] = 0xA5
            bvh.intersect_rays(rays, hits=hits, flags=flags)
            ids = hits["prim_id"].astype(np.uint64)
            assert ((ids < tris.shape[0]) | (ids == np.uint64(api.INVALID_ID if dtype == np.float32 else 2 ** 64 - 1))).all(), (m, flags)
            out.append(hits)
        assert np.array_equal(out[1].view(np.uint8), out[0].view(np.uint8)), m
