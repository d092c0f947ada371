"""Scenes far from the unit cube, without a GPU: meshes moved far from the origin, scaled down to 1e-20 and up to 1e20,
flat meshes with rays lying in and crossing their plane, a tiny cluster among huge triangles, surface rays with negative
and infinite tmin, a mesh whose boundary lies just past a cell of the 4-wide tree's quantisation grid, and double
precision at 1e9 and 1e-200.  The device code compiled by g++ (tests/host_emul.cpp) must
equal the oracle on its own tree in every mode, counters included; the watertight ROBUST traversal and the compressed
4-wide tree must equal brute force.  tests/test_coordinate_ranges_gpu.py checks the CUDA kernels against the same
expectations, so a failure there points at the device code and not at these assumptions.

Why the yardsticks are what they are: far from the origin the reference's FAST slab test is not watertight on many rays
(at offset 1e6 it misses about a third of the hits brute force finds), so the fast binary traversal is compared with the
oracle on the same tree, never with brute force.  On a flat mesh a ray crossing a shared edge hits two coplanar
triangles at the same t and which one is reported depends on the tree, so there brute force is the yardstick only for
rays whose closest hit is unique in t."""
import numpy as np
import pytest

from bvh_b200 import scenes
from oracle.pyoracle import ANY_HIT, ROBUST, TIE_LOWEST_ID
from tests.helpers import INVALID, assert_hits_equal
from tests.test_refit_boxes_host import fold_leaf_boxes

MODES = (("lowest", TIE_LOWEST_ID), ("last", 0), ("any", ANY_HIT | TIE_LOWEST_ID), ("robust", ROBUST | TIE_LOWEST_ID))

N_TRIS = 20000
# name -> (unit-range scene, offset, scale, dtype)
FAMILIES = {
    "offset_1e3": ("soup", 1e3, 1.0, np.float32),
    "offset_1e5": ("soup", 1e5, 1.0, np.float32),
    "offset_-3e5": ("soup", -3e5, 1.0, np.float32),
    "offset_1e6": ("soup", 1e6, 1.0, np.float32),
    "scale_1e-20": ("soup", 0.0, 1e-20, np.float32),
    "scale_1e-6": ("soup", 0.0, 1e-6, np.float32),
    "scale_1e6": ("soup", 0.0, 1e6, np.float32),
    "scale_1e20": ("soup", 0.0, 1e20, np.float32),
    "flat_soup": ("flat_soup", 0.0, 1.0, np.float32),
    "flat_grid": ("flat_grid", 0.0, 1.0, np.float32),
    "tiny_cluster_huge_tris": ("mix", 0.0, 1.0, np.float32),
    "surface_rays_tmin": ("ao", 0.0, 1.0, np.float32),
    "cell_boundary": ("cell_boundary", 0.0, 1.0, np.float32),
    "f64_offset_1e9": ("soup", 1e9, 1.0, np.float64),
    "f64_scale_1e-200": ("soup", 0.0, 1e-200, np.float64),
}
# every triangle in one plane (or, for cell_boundary, a wall and soups clipped flat against their boxes): equal-t ties
# between coplanar neighbours depend on the tree
COPLANAR = {"flat_soup", "flat_grid", "cell_boundary"}


def _axis_rays(rng, m, plane_axis, plane, in_plane):
    """m axis-parallel rays over [0,1]^2 of the other two axes, half of them on the 1/100 lattice (the flat grid's
    vertex lines): crossing the plane `plane_axis = plane` from 0.5 away, or (in_plane) lying in it."""
    other = [a for a in range(3) if a != plane_axis]
    rays = np.zeros((m, 8))
    rays[:, other[0]] = rng.uniform(0, 1, m)
    rays[:, other[1]] = rng.uniform(0, 1, m)
    rays[: m // 2, other] = np.round(rays[: m // 2, other] * 100) / 100
    if in_plane:
        rays[:, plane_axis] = plane
        along = other[0] if in_plane == 1 else other[1]
        rays[:, along] = -0.5
        rays[:, 3 + along] = 1.0
    else:
        rays[:, plane_axis] = plane + 0.5
        rays[:, 3 + plane_axis] = -1.0
    rays[:, 7] = np.inf
    return rays


def _unit_scene(kind, n):
    """(triangles, rays) of a scene in or near the unit cube, in float64.  Infinite tmax is stored as inf."""
    rng = np.random.RandomState(3)
    if kind == "soup":
        tris = scenes.soup(n, seed=3, dtype=np.float64)
        rays = scenes.make_primary("soup", 97, 95, dtype=np.float64)
    elif kind == "flat_soup":
        tris = scenes.soup(n, seed=3, dtype=np.float64)
        tris[:, 2::3] = 0.5
        rays = np.concatenate([scenes.make_primary("soup", 80, 80, dtype=np.float64),
                               _axis_rays(rng, 2000, 2, 0.5, 0), _axis_rays(rng, 1000, 2, 0.5, 1), _axis_rays(rng, 1000, 2, 0.5, 2)])
    elif kind == "flat_grid":
        tris = scenes.grid(n, dtype=np.float64)
        tris[:, 1::3] = 0.0
        rays = np.concatenate([scenes.make_primary("grid", 80, 80, dtype=np.float64),
                               _axis_rays(rng, 2000, 1, 0.0, 0), _axis_rays(rng, 1000, 1, 0.0, 1), _axis_rays(rng, 1000, 1, 0.0, 2)])
    elif kind == "mix":
        # the unit soup shrunk to 1e-4 at (1000, 1000, 1000) and its camera with it, plus ten triangles 1e4 across
        # around it; at 1000 a float32 ulp is 6e-5, so the cluster's triangles collapse onto a few lattice points
        tris = scenes.soup(n - 10, seed=3, dtype=np.float64) * 1e-4 + 1000.0
        c = 1000.0 + rng.uniform(-2e3, 2e3, (10, 1, 3))
        huge = (c + rng.uniform(-0.5, 0.5, (10, 3, 3)) * 1e4).reshape(10, 9)
        tris = np.concatenate([tris, huge])
        rays = scenes.make_primary("soup", 97, 95, dtype=np.float64)
        rays[:, 0:3] = rays[:, 0:3] * 1e-4 + 1000.0
        rays[:, 6:8] *= 1e-4
    elif kind == "cell_boundary":
        # x from -1 to 1.5, with a wall of triangles at x = 2^-25 closing the negative half: the root's 4-wide node has
        # its origin at -1 and cells of 2^-6, and 2^-25 - (-1) rounds to 1.0 = 64 cells exactly, so the wide quantisation
        # must round the upper bounds of the children holding the wall up by one more cell.  Short rays start at
        # x = 2^-22 and reach the wall but not x = 0 (rays from exactly 2^-24 would lose their offset to rounding
        # against the node origin); the soup camera looks at the rest.
        def box_soup(count, seed, lo, hi):
            t = np.clip(scenes.soup(count, seed=seed, dtype=np.float64), 0, 1).reshape(count, 3, 3)
            return (np.array(lo) + t * (np.array(hi) - np.array(lo))).reshape(count, 9)
        g = np.arange(31) / 30
        y, z = np.meshgrid(g, g, indexing="ij")
        p = np.stack([np.full_like(y, 2.0 ** -25), y, z], -1)
        wall = np.concatenate([np.concatenate([p[:-1, :-1], p[1:, :-1], p[1:, 1:]], -1),
                               np.concatenate([p[:-1, :-1], p[1:, 1:], p[:-1, 1:]], -1)]).reshape(-1, 9)
        tris = np.concatenate([box_soup(6000, 1, (-1, 0, 0), (-0.5, 1, 1)), box_soup(6000, 2, (-0.4, 0, 0), (-0.1, 1, 1)), wall,
                               box_soup(n - 12000 - wall.shape[0], 3, (0.5, 0, 0), (1.5, 1, 1))])
        short = np.zeros((5000, 8))
        short[:, 0] = 2.0 ** -22
        short[:, 1:3] = rng.uniform(0.05, 0.95, (5000, 2))
        short[:, 3] = -1.0
        short[:, 4:6] = rng.uniform(-0.1, 0.1, (5000, 2))
        short[:, 7] = 0.9 * 2.0 ** -22
        rays = np.concatenate([short, scenes.make_primary("soup", 71, 71, dtype=np.float64)])
    elif kind == "ao":
        # surface rays (pushed 1e-3 off a triangle, tmax 0.25) with tmin 0, -1 and -inf: negative tmin reaches behind
        # the origin, to the triangle the ray starts from
        tris = scenes.soup(n, seed=3, dtype=np.float64)
        rays = scenes.incoherent_rays(tris, 9999, seed=3)
        rays[1::3, 6] = -1.0
        rays[2::3, 6] = -np.inf
    else:
        raise ValueError(kind)
    rays = rays.astype(np.float64)
    rays[rays[:, 7] >= np.finfo(np.float32).max, 7] = np.inf
    return tris, rays


def ranged(kind, n, offset=0.0, scale=1.0, dtype=np.float32):
    """A unit-range scene moved to `offset` and scaled by `scale`: triangles and ray origins as x * scale + offset,
    directions unchanged, tmin and tmax times scale (tmax clamped to the dtype's max), all in float64 and rounded once."""
    tris, rays = _unit_scene(kind, n)
    tris = tris * scale + offset
    rays[:, 0:3] = rays[:, 0:3] * scale + offset
    with np.errstate(over="ignore"):
        rays[:, 6:8] *= scale
    rays[:, 7] = np.minimum(rays[:, 7], np.finfo(dtype).max)
    return np.ascontiguousarray(tris.astype(dtype)), np.ascontiguousarray(rays.astype(dtype))


def family(name):
    kind, offset, scale, dtype = FAMILIES[name]
    return ranged(kind, N_TRIS, offset, scale, dtype)


def brute_force_unique(oracle, tris, rays):
    """Brute force's closest hits (lowest id among equal t) and which rays have a closest hit that is unique in t (or
    none): the same scan over the triangles in reverse order, which keeps the highest id among equal t, agrees there."""
    bf = oracle.brute_force(tris, rays)
    rev = oracle.brute_force(np.ascontiguousarray(tris[::-1]), rays)[0]
    rev = np.where(rev == INVALID, INVALID, tris.shape[0] - 1 - rev.astype(np.int64)).astype(np.uint32)
    return bf, bf[0] == rev


# At scale 1e-20 the triangle test runs on subnormals, which the CPU computes about a hundred times slower: brute force
# checks every eighth ray there, so that a family costs seconds rather than minutes.
BRUTE_FORCE_STRIDE = {"scale_1e-20": 8}
_brute_force_cache = {}


def family_brute_force(oracle, name):
    """(ray selection, brute force on those rays, unique-in-t mask) of a family, computed once per process."""
    if name not in _brute_force_cache:
        tris, rays = family(name)
        sel = np.arange(0, rays.shape[0], BRUTE_FORCE_STRIDE.get(name, 1))
        _brute_force_cache[name] = (sel,) + brute_force_unique(oracle, tris, rays[sel])
    return _brute_force_cache[name]


def pick(hits, sel):
    return tuple(np.asarray(x)[sel] for x in hits[:4])


def leaf_boxes_contained(tree, wide):
    """Dequantise the box of every leaf child of every wide node in position space (origin + q * cell, float32) and
    compare with the binary leaf it was quantised from: returns the number of leaf boxes that do not enclose it."""
    words = wide.view(np.uint32)
    nodes = tree["nodes"]
    index = nodes.view(np.uint32)[:, 6]
    leaf = np.nonzero(index & 15)[0]
    order = np.argsort(index[leaf])
    keys, slots = index[leaf][order], leaf[order]
    origin = words[:, 0:3].view(np.float32)
    cell = ((words[:, 3:4] >> np.array([0, 8, 16], np.uint32)) & 0xFF) << 23
    cell = cell.astype(np.uint32).view(np.float32)
    count = (words[:, 3] >> 24) & 0xFF
    bad = 0
    for c in range(4):
        ref = words[:, 10 + c]
        sel = np.nonzero((c < count) & ((ref & 15) != 0))[0]
        pos = np.searchsorted(keys, ref[sel])
        assert (keys[pos] == ref[sel]).all()
        b = nodes[slots[pos]][:, :6]
        ql = ((words[sel, 4:7] >> np.uint32(8 * c)) & 0xFF).astype(np.float32)
        qh = ((words[sel, 7:10] >> np.uint32(8 * c)) & 0xFF).astype(np.float32)
        flat = cell[sel] == 0                                      # exponent 0: a flat axis, every child on the origin
        lo = np.where(flat, origin[sel], origin[sel] + ql * cell[sel])
        hi = np.where(flat, origin[sel], origin[sel] + qh * cell[sel])
        bad += int(((lo > b[:, 0::2]) | (hi < b[:, 1::2])).any(axis=1).sum())
    return bad


@pytest.mark.parametrize("name", list(FAMILIES))
def test_emulation_equals_the_oracle_at_range(emul, oracle, name):
    """Both build qualities: a valid reference tree, and the device traversal code equal to the oracle on it in every
    mode, counters included; ROBUST equal to brute force except on coplanar meshes."""
    tris, rays = family(name)
    for quality in ("low", "high"):
        tree = emul.build(tris=tris, quality=quality)
        bounds, index_values = emul.compact(tree)
        otree = oracle.from_arrays(bounds, index_values, tree["prim_ids"])
        assert oracle.check_invariants(otree, 8) == 0
        before = otree.arrays()[0]
        oracle.refit(otree)
        assert (otree.arrays()[0] == before).all()
        oracle.set_triangles(otree, tris)
        for mode, flags in MODES:
            got = emul.trace(tree, rays, flags)
            want = oracle.trace(otree, rays, flags=flags, stats=True)
            assert_hits_equal(got[:4], want[:4], f"{name}/{quality}/{mode}")
            assert (got[4] == want[4]).all(), f"{name}/{quality}/{mode}: counters"
    sel, bf, unique = family_brute_force(oracle, name)
    robust = pick(emul.trace(tree, rays, ROBUST | TIE_LOWEST_ID), sel)
    if name in COPLANAR:
        assert_hits_equal(pick(robust, unique), pick(bf, unique), f"{name}: robust vs brute force")
    else:
        assert_hits_equal(robust, bf, f"{name}: robust vs brute force")


@pytest.mark.parametrize("name", [f for f in FAMILIES if FAMILIES[f][3] == np.float32])
def test_wide_tree_is_conservative_at_range(emul, oracle, name):
    """The compressed 4-wide tree over the library's default tree: every leaf box encloses its binary leaf in position
    space, closest hits equal brute force wherever brute force's hit is unique in t, any-hit finds a hit exactly where
    brute force does."""
    tris, rays = family(name)
    tree = emul.build(tris=tris, quality="high")
    wide, levels = emul.wide_build(tree)
    assert 1 <= levels <= 60                    # the device collapses up to 60 levels and falls back to binary beyond
    assert leaf_boxes_contained(tree, wide) == 0
    sel, bf, unique = family_brute_force(oracle, name)
    got = emul.wide_trace(tree, wide, rays, 0)
    assert_hits_equal(pick(pick(got, sel), unique), pick(bf, unique), f"{name}: wide vs brute force")
    occl = emul.wide_trace(tree, wide, rays, 1)[0][sel]
    assert ((occl != INVALID) == (bf[0] != INVALID)).all(), f"{name}: wide any-hit verdict"
    # the same wide tree when the binary one is read back in the reference's layout (what the GPU test rebuilds)
    bounds, index_values = emul.compact(tree)
    again = emul.from_reference(bounds, index_values, tree["prim_ids"], tris)
    wide2, _ = emul.wide_build(again)
    assert_hits_equal(emul.wide_trace(again, wide2, rays, 0)[:4], got[:4], f"{name}: wide from the reference layout")


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_wide_morton_keys_far_from_the_origin(emul, oracle, dtype):
    """63-bit Morton keys at offset 1e6: a valid tree on which the traversal code equals the oracle."""
    tris, rays = ranged("soup", N_TRIS, 1e6, 1.0, dtype)
    tree = emul.build(tris=tris, morton_bits=63, quality="high")
    bounds, index_values = emul.compact(tree)
    otree = oracle.from_arrays(bounds, index_values, tree["prim_ids"])
    assert oracle.check_invariants(otree, 8) == 0
    oracle.set_triangles(otree, tris)
    for mode, flags in MODES:
        assert_hits_equal(emul.trace(tree, rays, flags)[:4], oracle.trace(otree, rays, flags=flags), f"63-bit/{mode}")


def moved_vertices(tris, scale, seed=4):
    """Every triangle moved by up to 0.02 * scale per axis, in float64 and rounded once."""
    rng = np.random.RandomState(seed)
    n = tris.shape[0]
    return np.ascontiguousarray((tris.astype(np.float64).reshape(n, 3, 3) + rng.uniform(-0.02, 0.02, (n, 1, 3)) * scale)
                                .reshape(n, 9).astype(tris.dtype))


def grown_boxes(oracle, tris):
    """The triangles' boxes (min3, max3) grown by 1 % of their extent on every side, in float64 and rounded once."""
    bb = oracle.tri_bboxes_centers(tris)[0].astype(np.float64)
    ext = bb[:, 3:] - bb[:, :3]
    return np.ascontiguousarray(np.concatenate([bb[:, :3] - 0.01 * ext, bb[:, 3:] + 0.01 * ext], axis=1).astype(tris.dtype))


def refitted_bounds(oracle, index_values, prim_ids, boxes):
    """What a refit must leave: leaf boxes folded from the primitive boxes, inner boxes by the reference's refit."""
    want = fold_leaf_boxes(index_values, prim_ids, boxes, boxes.dtype)
    tree = oracle.from_arrays(want, index_values, prim_ids)
    oracle.refit(tree)
    return tree.arrays()[0]


@pytest.mark.parametrize("name", ["offset_1e5", "scale_1e6"])
def test_refit_at_range(emul, oracle, name):
    """A tree refitted to moved vertices (and to boxes grown by 1 %): ROBUST and the rebuilt wide tree equal brute force
    on the moved mesh."""
    tris, rays = family(name)
    tree = emul.build(tris=tris, quality="high")
    _, index_values = emul.compact(tree)
    prim_ids = tree["prim_ids"]
    moved = moved_vertices(tris, FAMILIES[name][2])
    bf, unique = brute_force_unique(oracle, moved, rays)
    assert unique.all()
    for boxes in (oracle.tri_bboxes_centers(moved)[0], grown_boxes(oracle, moved)):
        bounds = refitted_bounds(oracle, index_values, prim_ids, boxes)
        refitted = emul.from_reference(bounds, index_values, prim_ids, moved)
        assert_hits_equal(emul.trace(refitted, rays, ROBUST | TIE_LOWEST_ID)[:4], bf, f"{name}: refit robust")
        wide, _ = emul.wide_build(refitted)
        assert_hits_equal(emul.wide_trace(refitted, wide, rays, 0)[:4], bf, f"{name}: refit wide")
