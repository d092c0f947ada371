"""Stores what the tests that compare with the original project compared against, so that they run without it:

    BVH_REFERENCE_DIR=<checkout of madmann91/bvh> python -c "import __graft_entry__ as g; g.build()"
    python tests/golden/make_reference_digests.py

Needs oracle/_ref (the unmodified reference compiled in place).  Writes, next to this script:
  reference_digests.json  SHA-256 digests (tests/helpers.py digest) of the reference's outputs
  reference_trees.npz     topology (node index words, primitive order) of the trees the reference built that the
                          tests feed to this library; tests/helpers.py reference_tree rebuilds their exact bytes
"""
import ctypes as C
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from bvh_b200 import scenes  # noqa: E402
from oracle.pyoracle import Ref  # noqa: E402
from tests import test_c_abi_2d as T2  # noqa: E402
from tests import test_optimize as TO  # noqa: E402
from tests import test_oracle_pinning as TP  # noqa: E402
from tests.helpers import digest, reference_tree  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
ref = Ref()
tmp = tempfile.mkdtemp()
digests, trees = {}, {}


def topology(blob, dim, dtype, key, boxes):
    nodes, ids = TO.parse(blob, dim, dtype)
    trees[key + "_index"] = nodes["index"].astype(np.uint32)
    trees[key + "_ids"] = ids.astype(np.uint32)
    np.savez_compressed(os.path.join(OUT, "reference_trees.npz"), **trees)
    assert reference_tree(key, boxes, dim, dtype) == blob, f"{key}: the stored topology does not rebuild the reference's tree"


# -- test_oracle_pinning: builders, refit, Morton codes ---------------------------------------------------
sec = digests["builders"] = {}
for kind, n, dtype in [("soup", 3000, np.float32), ("grid", 3000, np.float32), ("soup", 1500, np.float64)]:
    for quality in ("low", "medium"):
        tris = scenes.make_mesh(kind, n, dtype=dtype)
        bb, cc = ref.tri_bboxes_centers(tris)
        tr = ref.build(bb, cc, quality=quality, threads=-1)
        bounds, idx, ids = tr.arrays()
        d = {"bounds": digest(bounds), "index": digest(idx), "prim_ids": digest(ids),
             "serialized": digest(np.frombuffer(ref.serialize(tr), np.uint8))}
        ref.set_triangles(tr, tris)
        rays = scenes.make_primary(kind, 96, 96, dtype=dtype)
        for mode, flags in TP.MODES:
            for name, a in zip(("ids", "t", "u", "v", "stats"), ref.trace(tr, rays, flags=flags, stats=True)):
                d[f"{mode}_{name}"] = digest(a)
        sec[f"{kind}_{n}_{np.dtype(dtype).name}_{quality}"] = d

tris = scenes.soup(2000)
bb, cc = ref.tri_bboxes_centers(tris)
tr = ref.build(bb, cc, quality="medium", threads=-1)
bounds, idx, ids = tr.arrays()
rng = np.random.RandomState(3)
leaf = (idx & 15) != 0
noisy = bounds.copy()
noisy[leaf] += rng.uniform(-0.01, 0.01, size=noisy[leaf].shape).astype(np.float32)
noisy[~leaf] = 0
b = ref.from_arrays(noisy, idx, ids)
ref.refit(b)
digests["refit"] = {"tree": {"bounds": digest(bounds), "index": digest(idx), "prim_ids": digest(ids)},
                    "refitted_bounds": digest(b.arrays()[0])}

rng = np.random.RandomState(7)
m32, m64 = [], []
for _ in range(500):
    x, y, z = (int(v) for v in rng.randint(0, 1 << 10, 3))
    m32.append(ref.morton_encode(x, y, z, 32))
    x, y, z = (int(v) for v in rng.randint(0, 1 << 21, 3))
    m64.append(ref.morton_encode(x, y, z, 64))
digests["morton"] = {"morton32": digest(np.array(m32, np.uint64)), "morton64": digest(np.array(m64, np.uint64))}

# -- test_optimize: the reference C library's Medium tree, before and after its ReinsertionOptimizer -------------
cref = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libbvh_c_ref.so"))
sec = digests["optimize"] = {}
for s, dim, dtype in [("3f", 3, np.float32), ("3d", 3, np.float64), ("2f", 2, np.float32), ("2d", 2, np.float64)]:
    for n in (300, 3000):
        rf = TO.bind(cref, s)
        boxes, centers = TO.scene(dim, n, dtype, 7 + n)
        cfg = TO.Config(1, 1, 8, 1024)
        tree = rf("build")(None, boxes.ctypes.data, centers.ctypes.data, n, C.byref(cfg))
        before = TO.save_bytes(rf, tree, os.path.join(tmp, "before.bin"))
        pool = cref.bvh_thread_pool_create(4)
        rf("optimize")(pool if n > 100 else None, tree)
        cref.bvh_thread_pool_destroy(pool)
        after = TO.save_bytes(rf, tree, os.path.join(tmp, "after.bin"))
        rf("destroy")(tree)
        key = f"optimize_{s}_{n}"
        topology(before, dim, dtype, key, boxes)
        sec[key] = {"after": digest(np.frombuffer(after, np.uint8))}

# -- test_c_abi_2d: a 2-D tree built, traversed, refitted and saved by the reference C library ---------------
sec = digests["c_abi_2d"] = {}
for s in ("2f", "2d"):
    api = T2.Api2(os.path.join(ROOT, "oracle", "_ref", "libbvh_c_ref.so"), s)
    boxes, centers, rays = T2.scene2(700, 3, api.dtype)
    rb = api.build(boxes, centers)
    path = os.path.join(tmp, f"tree_{s}.bin")
    api.save(rb, path)
    key = f"c_abi_2d_{s}"
    topology(open(path, "rb").read(), 2, api.dtype, key, boxes)
    ids = api.prim_ids(rb)
    d = {"nodes": digest(T2.node_array(api.nodes(rb)))}
    for variant in ("intersect_ray", "intersect_ray_any", "intersect_ray_robust", "intersect_ray_any_robust"):
        d[variant] = digest(T2.trace_array(api.trace(rb, rays, boxes, ids, variant)))
    T2.grow_leaves_and_refit(api, rb)
    d["refitted_nodes"] = digest(T2.node_array(api.nodes(rb)))
    api.save(rb, path)
    d["refitted_file"] = digest(np.frombuffer(open(path, "rb").read(), np.uint8))
    api.f("destroy")(rb)
    sec[key] = d

with open(os.path.join(OUT, "reference_digests.json"), "w") as f:
    json.dump(digests, f, indent=1, sort_keys=True)
    f.write("\n")
print("trees:", {k: v.shape for k, v in trees.items()})
