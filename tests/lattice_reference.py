"""A NumPy model of the Quality Low LBVH build, exact on scenes whose Morton keys are known in advance.

Every primitive centre of a lattice scene is an integer point of [0, E]^3, with one centre at (0, 0, 0) and one at
(E, E, E), E a power of two.  The build's grid transform (build_core.cuh make_grid_xform, cubic cells) then has
scale = dim / E and offset 0, both exact (dim = 2^10 cells per axis for 30-bit keys, 2^21 for 63-bit keys), so the cell
of a centre c is min(c * dim / E, dim - 1) and every key is an integer function of the input.  From the keys alone,
with no code of the library:

1. order     the BVH order of the primitives is argsort(keys, stable): equal keys keep their input order, because
             the first radix pass ranks the identity permutation stably and every later pass is stable;
2. topology  the split between sorted neighbours k and k + 1 weighs delta(k) = (keys[k] ^ keys[k+1], k ^ (k+1)),
             compared lexicographically (build_core.cuh delta_at).  Two equal weights always have a larger one
             between them (equal XORs of sorted keys: the common prefix above their top bit must change in
             between; equal position XORs: the ruler sequence), so the tree without leaf collapse is the max-Cartesian
             tree of delta: the node of split k covers the sorted positions from (nearest larger weight on the left) + 1
             to (nearest larger weight on the right);
3. boxes     every node's box is the min / max of the boxes of the primitives in its range;
4. depth     the number of levels that hold inner nodes (tests/test_host_emulation.py _tree_depth).

check_tree compares a built tree with the model and names the first check that fails.
"""
import numpy as np

# lattice extent per key width: one cell per lattice step
EXTENT = {30: 1 << 10, 63: 1 << 21}
AXIS_BITS = {30: 10, 63: 21}

PATTERNS = ("distinct", "one_cell", "cells16", "low_digit", "high_digit", "sorted", "reversed", "chain")


# ---- keys -----------------------------------------------------------------------------------------------------------
def _spread_byte():
    """bit i of a byte -> bit 3i"""
    table = np.zeros(256, np.uint64)
    for b in range(256):
        table[b] = sum(((b >> i) & 1) << (3 * i) for i in range(8))
    return table


_SPREAD_BYTE = _spread_byte()


def interleave(x, y, z, axis_bits):
    """Morton key: bit i of x, y, z goes to key bit 3i, 3i + 1, 3i + 2 (a byte of a coordinate at a time)."""
    key = np.zeros(np.shape(x), np.uint64)
    for axis, v in enumerate((x, y, z)):
        v = np.asarray(v, np.uint64) & np.uint64((1 << axis_bits) - 1)
        for low in range(0, axis_bits, 8):
            key |= _SPREAD_BYTE[(v >> np.uint64(low)) & np.uint64(255)] << np.uint64(3 * low + axis)
    return key


def lattice_keys(centres, extent, key_bits):
    """Keys of integer centres in [0, extent]^3 under the build's cubic grid (extent and cell count powers of two)."""
    c = np.asarray(centres, np.int64)
    assert c.min() >= 0 and c.max() <= extent
    dim = 1 << AXIS_BITS[key_bits]
    cells = c * (dim // extent) if dim >= extent else c // (extent // dim)
    cells = np.minimum(cells, dim - 1)
    return interleave(cells[:, 0], cells[:, 1], cells[:, 2], AXIS_BITS[key_bits])


def _distinct(values):
    """the distinct values, sorted"""
    v = np.sort(values)
    return v[np.concatenate([[True], v[1:] != v[:-1]])]


# ---- scenes ---------------------------------------------------------------------------------------------------------
def lattice_scene(pattern, n, key_bits, seed=0):
    """Integer centres (n, 3) of one key pattern, and the lattice extent E.  Every scene of two or more centres holds
    the corners (0, 0, 0) and (E, E, E), which fix the grid; the rest follow the pattern:
      distinct    distinct random cells, random input order
      one_cell    every other centre in one cell (the index tie-break must balance the run)
      cells16     16 distinct cells, heavily duplicated
      low_digit   keys that differ only in their lowest 8-bit radix digit
      high_digit  keys that differ only in their highest radix digit (bits 24-31 / 56-63)
      sorted      random cells with many duplicates, input already in key order
      reversed    the same in reverse key order (equal keys must still come out in input order)
      chain       cells 2^i along each axis (keys with one bit set each: a tree of about 3 log2 E levels),
                  duplicated up to n"""
    E = EXTENT[key_bits]
    rng = np.random.default_rng(seed)
    corners = np.array([[0, 0, 0], [E, E, E]], np.int64)
    if n <= 2:
        return corners[:n].copy(), E
    m = n - 2
    if pattern == "distinct":
        # distinct cells of [1, E - 2]^3 (never a corner's cell)
        pick = _distinct(rng.integers(0, (E - 2) ** 3, size=m + m // 8 + 16, dtype=np.int64))
        while pick.size < m:
            pick = _distinct(np.concatenate([pick, rng.integers(0, (E - 2) ** 3, size=m, dtype=np.int64)]))
        pick = rng.permutation(pick)[:m]
        body = np.stack([pick % (E - 2), pick // (E - 2) % (E - 2), pick // (E - 2) ** 2], axis=1) + 1
    elif pattern == "one_cell":
        body = np.repeat(rng.integers(1, E - 1, size=(1, 3)), m, axis=0)
    elif pattern == "cells16":
        body = rng.integers(1, E - 1, size=(16, 3))[rng.integers(0, 16, size=m)]
    elif pattern == "low_digit":
        # x, y < 8 and z < 4: key bits 0..7 only
        body = np.stack([rng.integers(0, 8, m), rng.integers(0, 8, m), rng.integers(0, 4, m)], axis=1)
    elif pattern == "high_digit":
        # multiples of E / 4: cell bits 8, 9 (30-bit) or 19, 20 (63-bit), key bits 24..29 or 57..62
        body = rng.integers(0, 4, size=(m, 3)) * (E // 4)
    elif pattern in ("sorted", "reversed"):
        pool = rng.integers(1, E - 1, size=(max(1, m // 3), 3))
        body = pool[rng.integers(0, pool.shape[0], size=m)]
    elif pattern == "chain":
        steps = np.int64(1) << np.arange(AXIS_BITS[key_bits], dtype=np.int64)
        chain = np.zeros((3 * steps.size, 3), np.int64)
        for axis in range(3):
            chain[axis * steps.size:(axis + 1) * steps.size, axis] = steps
        body = chain[np.arange(m) % chain.shape[0]]
    else:
        raise ValueError(pattern)
    centres = np.concatenate([corners, np.asarray(body, np.int64)])
    if pattern in ("sorted", "reversed"):
        centres = centres[np.argsort(lattice_keys(centres, E, key_bits), kind="stable")]
        if pattern == "reversed":
            centres = centres[::-1]
    else:
        centres = centres[rng.permutation(n)]
    return np.ascontiguousarray(centres), E


def boxes_around(centres, dtype, half=0.25):
    """(n, 6) boxes as min3, max3: the centre +- half, exact in both scalar types."""
    c = np.asarray(centres, dtype)
    return np.ascontiguousarray(np.concatenate([c - dtype(half), c + dtype(half)], axis=1))


def triangles_around(centres, dtype):
    """(n, 9) triangles whose centre, computed as the build does (tri_bounds_center: ((v0 + v1) + v2) * fl(1/3)), is
    exactly the lattice point; asserted here in the build's own scalar type and order of operations."""
    c = np.asarray(centres, dtype)
    h = dtype(0.5)
    v0 = c + np.array([h, 0, 0], dtype)
    v1 = c + np.array([0, h, 0], dtype)
    v2 = c - np.array([h, h, 0], dtype)
    third = dtype(1.0 / 3.0)
    centre = ((v0 + v1) + v2) * third
    assert centre.dtype == dtype and np.array_equal(centre, c), "triangle centres are not the lattice points"
    return np.ascontiguousarray(np.concatenate([v0, v1, v2], axis=1))


def triangle_boxes(tris):
    """(n, 6) min3, max3 boxes of (n, 9) triangles (min / max are exact)."""
    v = tris.reshape(-1, 3, 3)
    return np.ascontiguousarray(np.concatenate([v.min(axis=1), v.max(axis=1)], axis=1))




# ---- the model ------------------------------------------------------------------------------------------------------
def _larger(hi, lo, a, b):
    """weight of split a > weight of split b (lexicographic)"""
    return (hi[a] > hi[b]) | ((hi[a] == hi[b]) & (lo[a] > lo[b]))


def _nearest_larger(hi, lo, step):
    """For every split k, the nearest split in direction `step` (-1 / +1) with a larger weight, or -1 / m if none.
    Pointer jumping: a neighbour that is not larger than k hands over its own current candidate, and everything in
    between is not larger than k either."""
    m = hi.size
    near = np.arange(m, dtype=np.int64) + step
    todo = np.arange(m, dtype=np.int64)
    while todo.size:
        j = near[todo]
        inside = (j >= 0) & (j < m)
        todo, j = todo[inside], j[inside]
        keep = ~_larger(hi, lo, j, todo)
        todo = todo[keep]
        near[todo] = near[j[keep]]
    return near


class Reference:
    """The expected Quality Low tree (no leaf collapse) of a lattice scene.  Nodes: leaf i (0 <= i < n) is sorted
    position i, inner node n + k is split k; first / count are their ranges of sorted positions."""

    def __init__(self, centres, extent, key_bits, prim_boxes):
        keys = lattice_keys(centres, extent, key_bits)
        n = self.n = keys.size
        self.order = np.argsort(keys, kind="stable")
        self.keys = keys[self.order]
        first = np.concatenate([np.arange(n, dtype=np.int64), np.zeros(n - 1, np.int64)])
        last = first.copy()
        self.levels = []                          # split indices of the inner nodes, root level first
        if n > 1:
            k = np.arange(n - 1, dtype=np.int64)
            hi = self.keys[:-1] ^ self.keys[1:]
            lo = (k ^ (k + 1)).astype(np.uint64)
            left, right = _nearest_larger(hi, lo, -1), _nearest_larger(hi, lo, +1)
            first[n:], last[n:] = left + 1, right
            # the parent of split k is the smaller of its two nearest larger neighbours
            has_l, has_r = left >= 0, right < n - 1
            l_, r_ = np.where(has_l, left, 0), np.where(has_r, right, 0)
            up = np.where(has_l & has_r, np.where(_larger(hi, lo, l_, r_), r_, l_), np.where(has_l, l_, np.where(has_r, r_, -1)))
            # children: the left child of split k covers [first, k], the right one [k + 1, last]; a one-position range is
            # the leaf itself, a longer one the split whose parent is k
            lchild, rchild = k.copy(), k + 1
            child = np.nonzero(up >= 0)[0]
            is_left = child < up[child]
            lchild[up[child[is_left]]] = n + child[is_left]
            rchild[up[child[~is_left]]] = n + child[~is_left]
            # (fails if two equal weights had no larger one between them: they would claim the same child slot)
            assert (up < 0).sum() == 1 and np.array_equal(first[lchild], first[n:]) and np.array_equal(last[lchild], k) and \
                np.array_equal(first[rchild], k + 1) and np.array_equal(last[rchild], last[n:]), \
                "the split weights do not define a binary tree"
            self.lchild, self.rchild = lchild, rchild
            frontier = np.nonzero(up < 0)[0]
            while frontier.size:
                self.levels.append(frontier)
                kids = np.concatenate([lchild[frontier], rchild[frontier]])
                frontier = np.sort(kids[kids >= n] - n)     # in position order: the box pass then reads memory in order
        self.depth = len(self.levels)
        self.first, self.count = first, last - first + 1
        self.boxes = self.node_boxes(prim_boxes)

    def find(self, first, count):
        """The model node of each range (first, count) of sorted positions, -1 where the model has no such node."""
        codes = (self.first << 32) + self.count
        by_code = np.argsort(codes)
        want = (np.asarray(first, np.int64) << 32) + np.asarray(count, np.int64)
        at = np.minimum(np.searchsorted(codes[by_code], want), codes.size - 1)
        return np.where(codes[by_code[at]] == want, by_code[at], -1)

    def node_boxes(self, prim_boxes):
        """(2n - 1, 6) node boxes as minx, maxx, miny, maxy, minz, maxz: the min / max of the primitive boxes of the
        node's range, computed level by level from the leaves up as the union of the two children (min and max are
        exact: this is the range's min / max bit for bit).  Internally the mins are negated, so a union is one max."""
        pb = np.asarray(prim_boxes)[self.order]
        n = self.n
        acc = np.empty((2 * n - 1, 6), pb.dtype)
        acc[:n, :3], acc[:n, 3:] = -pb[:, :3], pb[:, 3:]
        for k in reversed(self.levels):
            acc[n + k] = np.maximum(acc[self.lchild[k]], acc[self.rchild[k]])
        boxes = np.empty_like(acc)
        boxes[:, 0::2], boxes[:, 1::2] = -acc[:, :3], acc[:, 3:]
        return boxes


# ---- a built tree ---------------------------------------------------------------------------------------------------
def tree_ranges(index_values, prim_count):
    """Ranges of sorted positions of every node of a tree in the reference layout (root at 0, inner index = first
    child of an adjacent pair, leaf index = first primitive << 4 | count): (first, count, inner nodes level by level
    from the root)."""
    iv = np.asarray(index_values, np.uint64)
    m = iv.size
    count = (iv & np.uint64(15)).astype(np.int64)
    first = (iv >> np.uint64(4)).astype(np.int64)
    lo, hi = first.copy(), first + count - 1
    levels, reached, frontier = [], [], np.zeros(1, np.int64)
    while frontier.size:
        reached.append(frontier)
        inner = frontier[count[frontier] == 0]
        assert (first[inner] + 1 < m).all() and len(levels) < 256, "structure: a child index is out of range, or a cycle"
        if inner.size:
            levels.append(inner)
        frontier = np.concatenate([first[inner], first[inner] + 1])
    assert (np.bincount(np.concatenate(reached), minlength=m) == 1).all(), "structure: not every node is reached once from the root"
    leaves = count > 0
    assert (lo[leaves] >= 0).all() and (hi[leaves] < prim_count).all(), "structure: a leaf range is out of range"
    for inner in reversed(levels):
        c = first[inner]
        lo[inner] = np.minimum(lo[c], lo[c + 1])
        hi[inner] = np.maximum(hi[c], hi[c + 1])
    return lo, hi - lo + 1, levels


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype.itemsize == 4 else np.uint64)


def check_tree(ref, bounds, index_values, prim_ids, depth, collapsed=False, prim_boxes=None):
    """Compares a built tree (reference-layout arrays and its reported depth) with the model; raises AssertionError
    naming the first check that fails: order, topology, boxes or depth.
      collapsed=False  the tree must BE the model's tree (built with min_leaf_size = max_leaf_size = 1);
      collapsed=True   every node must be a node of the model (the SAH leaf collapse only prunes), and the reported
                       depth that of the tree itself;
      prim_boxes       the primitive boxes the node boxes must be made of (default: those the model was made with).
    The two trees are walked together from the root: the model node of a built node is the model child with the same
    first position (children may sit in either order: the larger box goes first)."""
    n = ref.n
    prim_ids = np.asarray(prim_ids).astype(np.int64)
    bad = np.nonzero(prim_ids != ref.order)[0]
    assert bad.size == 0, f"order: prim_ids differ from the stable key order at {bad.size} positions, first {bad[:4]} " \
                          f"(got {prim_ids[bad[:4]]}, want {ref.order[bad[:4]]})"
    first, count, levels = tree_ranges(index_values, n)
    child = (np.asarray(index_values, np.uint64) >> np.uint64(4)).astype(np.int64)
    model = np.full(first.size, -1, np.int64)
    model[0] = n + int(ref.levels[0][0]) if n > 1 else 0
    for inner in levels:
        k = model[inner]
        assert (k >= n).all(), f"topology: built inner node {int(inner[k < n][0])} covers a single position of the reference tree"
        lc, rc = ref.lchild[k - n], ref.rchild[k - n]
        c0_left = first[child[inner]] == ref.first[lc]
        model[np.where(c0_left, child[inner], child[inner] + 1)] = lc
        model[np.where(c0_left, child[inner] + 1, child[inner])] = rc
    bad = np.nonzero((first != ref.first[model]) | (count != ref.count[model]))[0]
    if bad.size:
        i = int(bad[0])
        raise AssertionError(f"topology: {bad.size} built nodes differ from the reference tree, first node {i}: (first, count) "
                             f"({int(first[i])}, {int(count[i])}), reference ({int(ref.first[model[i]])}, {int(ref.count[model[i]])})")
    if not collapsed:
        assert first.size == 2 * n - 1, f"topology: {first.size} nodes, the reference tree has {2 * n - 1}"
    boxes = ref.boxes if prim_boxes is None else ref.node_boxes(prim_boxes)
    want = boxes[model]
    diff = np.nonzero((_bits(np.asarray(bounds)) != _bits(want)).any(axis=1))[0]
    if diff.size:
        i = int(diff[0])
        raise AssertionError(f"boxes: {diff.size} node boxes are not the min / max of their range; node {i} "
                             f"({int(first[i])}, {int(count[i])}): {np.asarray(bounds)[i]} vs {want[i]}")
    want_depth = len(levels) if collapsed else ref.depth
    assert depth == want_depth and len(levels) == want_depth, \
        f"depth: reported {depth}, the tree has {len(levels)} inner levels, expected {want_depth}"
