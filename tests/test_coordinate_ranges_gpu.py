"""GPU build and traversal on scenes far from the unit cube (pytest -m gpu): the families of
tests/test_coordinate_ranges_host.py, whose expectations that file pins on the host.

* Build: the GPU tree, read back through the reference accessors, equals the host emulation's node for node (bounds
  bits, index words, primitive ids, depth) and is a valid reference tree.
* Binary kernels: every kernel in every mode equals the oracle traversing the downloaded tree bit for bit, counters
  included.  Far from the origin the reference's fast slab test is not watertight, so the fast modes are compared with
  the oracle on the same tree only; the watertight ROBUST mode must also equal brute force, except on coplanar meshes,
  where equal-t ties across shared edges depend on the tree.
* Wide kernel: its closest hits equal the host emulation of the same wide tree bit for bit, and equal brute force
  wherever brute force's hit is unique in t (the wide tree's claim of being conservative, checked directly); any-hit
  finds a hit exactly where brute force does.
* Refit: after moving the vertices (and after a refit from grown boxes) the bounds are the reference's refit of the
  new leaf boxes, and the rebuilt wide tree and ROBUST still answer as above on the moved mesh."""
import numpy as np
import pytest

from oracle.pyoracle import ANY_HIT as O_ANY, ROBUST as O_ROBUST, TIE_LOWEST_ID as O_LOWEST
from tests.helpers import INVALID, assert_hits_equal, hits_tuple
from tests.test_coordinate_ranges_host import (COPLANAR, FAMILIES, N_TRIS, brute_force_unique, family, family_brute_force,
                                               grown_boxes, moved_vertices, pick, ranged, refitted_bounds)

pytestmark = pytest.mark.gpu

WIDE_MAX_LEVELS = 60          # levels of the device's wide collapse; a deeper tree is traced by the binary kernels


def modes(api):
    """(name, oracle flags, C-ABI flags)"""
    return (("lowest", O_LOWEST, 0), ("last", 0, api.TIE_LAST_VISITED),
            ("any", O_ANY | O_LOWEST, api.ANY_HIT), ("robust", O_ROBUST | O_LOWEST, api.ROBUST))


def check_build(bvh, emul, oracle, tris, what, **build_args):
    """The GPU tree equals the host emulation's node for node and is a valid reference tree; returns its arrays."""
    bounds, index_values, prim_ids = bvh.arrays()
    etree = emul.build(tris=tris, **build_args)
    eb, ei = emul.compact(etree)
    assert eb.shape == bounds.shape, what
    assert (eb.view(np.uint8) == bounds.view(np.uint8)).all() and (ei == index_values).all(), f"{what}: nodes"
    assert (etree["prim_ids"] == prim_ids).all() and bvh.depth == etree["depth"], f"{what}: primitive ids / depth"
    tree = oracle.from_arrays(bounds, index_values, prim_ids)
    assert oracle.check_invariants(tree, 8) == 0, what
    return bounds, index_values, prim_ids


def check_wide(api, bvh, emul, tris, rays, sel, bf, unique, what):
    """KERNEL_WIDE against the host emulation of the wide tree derived from the downloaded binary tree, and against
    brute force (on the rays `sel`)."""
    bounds, index_values, prim_ids = bvh.arrays()
    etree = emul.from_reference(bounds, index_values, prim_ids, tris)
    wide, levels = emul.wide_build(etree)
    got = hits_tuple(bvh.intersect_rays(rays, flags=api.KERNEL_WIDE))
    if levels > WIDE_MAX_LEVELS:
        assert bvh.get_property("wide_nodes") == 0 and bvh.properties()["last_kernel"] != "trace_wide_kernel", what
        assert_hits_equal(got, hits_tuple(bvh.intersect_rays(rays)), f"{what}: binary fallback")
        return
    assert bvh.properties()["last_kernel"] == "trace_wide_kernel", what
    assert bvh.get_property("wide_nodes") == wide.shape[0] > 0, what
    assert_hits_equal(got, emul.wide_trace(etree, wide, rays, 0)[:4], f"{what}: wide kernel vs emulation")
    assert_hits_equal(pick(pick(got, sel), unique), pick(bf, unique), f"{what}: wide kernel vs brute force")
    occl = bvh.intersect_rays(rays, flags=api.KERNEL_WIDE | api.ANY_HIT)["prim_id"].astype(np.uint32)[sel]
    assert ((occl != INVALID) == (bf[0] != INVALID)).all(), f"{what}: wide any-hit verdict"


@pytest.mark.parametrize("name", list(FAMILIES))
def test_gpu_build_equals_the_emulation_at_range(gpu_lib, oracle, emul, name):
    tris, _ = family(name)
    for quality in ("low", "high"):
        bvh = gpu_lib.Bvh.build_triangles(tris, quality=quality)
        check_build(bvh, emul, oracle, tris, f"{name}/{quality}", quality=quality)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_gpu_wide_morton_keys_far_from_the_origin(gpu_lib, oracle, emul, dtype):
    """The 63-bit key path at offset 1e6: the emulation's tree, and the oracle's answers on it."""
    api = gpu_lib
    tris, rays = ranged("soup", N_TRIS, 1e6, 1.0, dtype)
    api.set_option("morton_bits", 63)
    try:
        bvh = api.Bvh.build_triangles(tris)
    finally:
        api.set_option("morton_bits", 0)
    assert bvh.get_property("morton_bits") == 63
    tree = oracle.from_arrays(*check_build(bvh, emul, oracle, tris, "63-bit keys", morton_bits=63, quality="high"))
    oracle.set_triangles(tree, tris)
    for mode, oflags, flags in modes(api):
        assert_hits_equal(hits_tuple(bvh.intersect_rays(rays, flags=flags)), oracle.trace(tree, rays, flags=oflags), f"63-bit/{mode}")


@pytest.mark.parametrize("name", list(FAMILIES))
def test_gpu_binary_kernels_equal_the_oracle_at_range(gpu_lib, oracle, name):
    api = gpu_lib
    tris, rays = family(name)
    bvh = api.Bvh.build_triangles(tris)
    tree = oracle.from_arrays(*bvh.arrays())
    oracle.set_triangles(tree, tris)
    for mode, oflags, flags in modes(api):
        want = oracle.trace(tree, rays, flags=oflags, stats=True)
        for kernel in (0,) + api.KERNELS:
            assert_hits_equal(hits_tuple(bvh.intersect_rays(rays, flags=flags | kernel)), want[:4], f"{name}/{mode}/{kernel}")
        hits, st = bvh.intersect_rays(rays, flags=flags, stats=True)
        assert_hits_equal(hits_tuple(hits), want[:4], f"{name}/{mode}/stats")
        for k, counter in enumerate(("inner_steps", "leaves", "prim_tests")):
            assert (st[counter] == want[4][:, k]).all(), f"{name}/{mode}: {counter}"
    sel, bf, unique = family_brute_force(oracle, name)
    robust = pick(hits_tuple(bvh.intersect_rays(rays, flags=api.ROBUST)), sel)
    keep = unique if name in COPLANAR else np.ones(sel.shape[0], bool)
    assert_hits_equal(pick(robust, keep), pick(bf, keep), f"{name}: robust vs brute force")


@pytest.mark.parametrize("name", list(FAMILIES))
def test_gpu_wide_kernel_is_conservative_at_range(gpu_lib, oracle, emul, name):
    api = gpu_lib
    tris, rays = family(name)
    bvh = api.Bvh.build_triangles(tris)
    if tris.dtype != np.float32:
        # the compressed wide tree is float only: the flag falls back to the exact binary traversal
        got = bvh.intersect_rays(rays, flags=api.KERNEL_WIDE)
        assert bvh.get_property("wide_nodes") == 0 and bvh.properties()["last_kernel"] != "trace_wide_kernel"
        assert np.array_equal(got.view(np.uint8), bvh.intersect_rays(rays).view(np.uint8))
        return
    sel, bf, unique = family_brute_force(oracle, name)
    check_wide(api, bvh, emul, tris, rays, sel, bf, unique, name)


@pytest.mark.parametrize("name", ["offset_1e5", "scale_1e6"])
def test_gpu_refit_at_range(gpu_lib, oracle, emul, name):
    """refit_triangles after the vertices moved a little, then refit_boxes with boxes grown by 1 %: same topology,
    bounds equal to the leaf-box fold plus the reference's refit, the rebuilt wide tree equal to its emulation and to
    brute force, ROBUST equal to brute force on the moved mesh."""
    api = gpu_lib
    tris, rays = family(name)
    bvh = api.Bvh.build_triangles(tris)
    bvh.intersect_rays(rays[:64], flags=api.KERNEL_WIDE)            # derive the wide tree: every refit must rebuild it
    assert bvh.get_property("wide_nodes") > 0
    _, index_before, ids_before = bvh.arrays()
    moved = moved_vertices(tris, FAMILIES[name][2])
    bf, unique = brute_force_unique(oracle, moved, rays)
    sel = np.arange(rays.shape[0])
    for how, boxes in (("refit_triangles", oracle.tri_bboxes_centers(moved)[0]), ("refit_boxes", grown_boxes(oracle, moved))):
        if how == "refit_triangles":
            bvh.refit_triangles(moved)
        else:
            bvh.refit_boxes(boxes)
        bounds, index_values, prim_ids = bvh.arrays()
        assert (index_values == index_before).all() and (prim_ids == ids_before).all(), how
        want = refitted_bounds(oracle, index_values, prim_ids, boxes)
        assert (want.view(np.uint8) == bounds.view(np.uint8)).all(), f"{name}/{how}: bounds"
        assert_hits_equal(hits_tuple(bvh.intersect_rays(rays, flags=api.ROBUST)), bf, f"{name}/{how}: robust vs brute force")
        check_wide(api, bvh, emul, moved, rays, sel, bf, unique, f"{name}/{how}")
