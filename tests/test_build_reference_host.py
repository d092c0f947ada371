"""The NumPy model of the Quality Low LBVH build (tests/lattice_reference.py) against the host emulation of the device
code, before the GPU build is compared with it (tests/test_build_reference_gpu.py), and the model's checker against
corrupted copies of a correct tree.

The model and the emulation agree on every key pattern in both key widths: without leaf collapse the emulated tree is
the max-Cartesian tree of the split weights, node for node, and with the default leaf settings every node of the
collapsed tree is a node of that tree.  The model therefore describes the algorithm, not one implementation of it."""
import math

import numpy as np
import pytest

from tests import lattice_reference as L

SIZES = (1, 2, 3, 17, 65, 300, 5000)


@pytest.mark.parametrize("bits", [30, 63])
@pytest.mark.parametrize("pattern", L.PATTERNS)
def test_model_is_the_emulated_tree(emul, pattern, bits):
    """min_leaf = max_leaf = 1: the emulated tree is the model's, node for node (order, ranges, boxes, depth); default
    leaf settings: every leaf and inner node of the collapsed tree is a node of the model, with the model's box."""
    for n in SIZES:
        for dtype in (np.float32, np.float64):
            centres, extent = L.lattice_scene(pattern, n, bits, seed=n)
            boxes = L.boxes_around(centres, dtype)
            ref = L.Reference(centres, extent, bits, boxes)
            for min_leaf, max_leaf in ((1, 1), (1, 8)):
                tree = emul.build(bboxes=boxes, centers=centres.astype(dtype), min_leaf=min_leaf, max_leaf=max_leaf,
                                  morton_bits=bits, quality="low")
                bounds, index_values = emul.compact(tree)
                try:
                    L.check_tree(ref, bounds, index_values, tree["prim_ids"], tree["depth"], collapsed=max_leaf > 1)
                except AssertionError as e:
                    raise AssertionError(f"{pattern}, n={n}, {np.dtype(dtype).name}, leaves {min_leaf}..{max_leaf}: {e}") from None


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_model_is_the_emulated_tree_of_triangles(emul, dtype):
    """Triangle input: the build computes the centres itself; the scene's triangles put them on the lattice points
    exactly (asserted by triangles_around), so the same model applies, with the triangles' boxes."""
    for pattern in ("distinct", "cells16", "reversed"):
        for n in (3, 129, 3000):
            centres, extent = L.lattice_scene(pattern, n, 30, seed=n)
            tris = L.triangles_around(centres, dtype)
            ref = L.Reference(centres, extent, 30, L.triangle_boxes(tris))
            tree = emul.build(tris=tris, min_leaf=1, max_leaf=1, quality="low")
            bounds, index_values = emul.compact(tree)
            L.check_tree(ref, bounds, index_values, tree["prim_ids"], tree["depth"])


def test_model_keys_are_the_library_morton_codes(emul):
    """The model's bit interleave, written out bit by bit, against the library's (build_core.cuh spread_bits_*)."""
    rng = np.random.default_rng(5)
    for bits, encode in ((30, emul.lib.emul_morton30), (63, emul.lib.emul_morton63)):
        axis_bits = L.AXIS_BITS[bits]
        cells = rng.integers(0, 1 << axis_bits, size=(2000, 3))
        cells[:3] = [[0, 0, 0], [(1 << axis_bits) - 1] * 3, [1 << (axis_bits - 1), 1, 0]]
        want = np.array([encode(*map(int, c)) for c in cells], np.uint64)
        assert np.array_equal(L.interleave(cells[:, 0], cells[:, 1], cells[:, 2], axis_bits), want)


@pytest.mark.parametrize("bits", [30, 63])
def test_model_shapes(bits):
    """What the key patterns are for: one cell gives a balanced run (depth about log2 n, plus the two corners), the
    chain of single-bit keys a deep caterpillar, the digit patterns keys that differ in one radix digit only."""
    n = 5000
    centres, extent = L.lattice_scene("one_cell", n, bits)
    assert L.Reference(centres, extent, bits, L.boxes_around(centres, np.float32)).depth <= math.ceil(math.log2(n)) + 2
    centres, extent = L.lattice_scene("chain", 3 * L.AXIS_BITS[bits] + 2, bits)
    assert L.Reference(centres, extent, bits, L.boxes_around(centres, np.float32)).depth >= 3 * L.AXIS_BITS[bits]
    top = 24 if bits == 30 else 56                                  # lowest bit of the last radix digit (4 / 8 passes)
    corner = L.lattice_keys(np.array([[extent] * 3]), extent, bits)[0]
    for pattern, mask in (("low_digit", np.uint64(0xFF)), ("high_digit", np.uint64(0xFF) << np.uint64(top))):
        centres, extent = L.lattice_scene(pattern, n, bits)
        keys = L.lattice_keys(centres, extent, bits)
        keys = keys[keys != corner]
        assert (keys & ~mask).max() == 0 and np.unique(keys).size > 32, pattern


def _rotate_split(bounds, index_values, ref, prim_boxes):
    """Moves one split by one position: a node over sorted positions [l, l + 2] split after l + 1 (children: an inner
    node over the leaves l, l + 1, and the leaf l + 2) is rebuilt split after l (children: the leaf l, and an inner node
    over the leaves l + 1, l + 2), with every box recomputed, so the tree stays a valid BVH of correct boxes."""
    bounds, index_values = bounds.copy(), index_values.copy()
    count = (index_values & np.uint64(15)).astype(np.int64)
    first = (index_values >> np.uint64(4)).astype(np.int64)
    pb = np.asarray(prim_boxes)[ref.order]
    box = lambda *pos: np.stack([pb[list(pos), :3].min(axis=0), pb[list(pos), 3:].max(axis=0)], axis=1).ravel()
    leaf = lambda pos: np.uint64(pos << 4 | 1)
    for node in np.nonzero(count == 0)[0]:
        for a, b in ((first[node], first[node] + 1), (first[node] + 1, first[node])):
            if count[a] == 0 and count[b] == 1:
                d = first[a]
                if count[d] == 1 and count[d + 1] == 1:
                    l = min(first[d], first[d + 1])
                    if first[b] == l + 2:
                        index_values[a], index_values[b] = leaf(l), index_values[a]
                        index_values[d], index_values[d + 1] = leaf(l + 1), leaf(l + 2)
                        bounds[a], bounds[b] = box(l), box(l + 1, l + 2)
                        bounds[d], bounds[d + 1] = box(l + 1), box(l + 2)
                        return bounds, index_values
    raise AssertionError("no node of the shape to rotate")


@pytest.mark.parametrize("corruption,check", [("swap two equal-key prim_ids", "order"), ("move one split by one position", "topology"),
                                              ("widen one node bound by one ulp", "boxes"), ("drop one level of the depth", "depth")])
def test_checker_names_each_corruption(emul, oracle, corruption, check):
    """The checker is sensitive to each kind of error a build kernel could make, and names it: a corrupted copy of a
    correct tree (emulated, 300 primitives in 16 cells, no leaf collapse) fails exactly the named check."""
    centres, extent = L.lattice_scene("cells16", 300, 30, seed=3)
    boxes = L.boxes_around(centres, np.float32)
    ref = L.Reference(centres, extent, 30, boxes)
    tree = emul.build(bboxes=boxes, centers=centres.astype(np.float32), min_leaf=1, max_leaf=1, quality="low")
    bounds, index_values = emul.compact(tree)
    prim_ids, depth = tree["prim_ids"].astype(np.int64), tree["depth"]
    L.check_tree(ref, bounds, index_values, prim_ids, depth)
    if check == "order":
        i = int(np.nonzero(ref.keys[1:] == ref.keys[:-1])[0][0])
        prim_ids[[i, i + 1]] = prim_ids[[i + 1, i]]
    elif check == "topology":
        bounds, index_values = _rotate_split(bounds, index_values, ref, boxes)
        assert oracle.check_invariants(oracle.from_arrays(bounds, index_values, prim_ids), 1) == 0   # still a valid BVH
    elif check == "boxes":
        node = int(np.nonzero((index_values & np.uint64(15)) == 0)[0][7])
        bounds[node, 2] = np.nextafter(bounds[node, 2], np.float32(-np.inf))
    else:
        depth -= 1
    with pytest.raises(AssertionError, match=f"^{check}:"):
        L.check_tree(ref, bounds, index_values, prim_ids, depth)
