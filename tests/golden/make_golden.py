"""Generates the committed golden vectors from the UNMODIFIED reference (oracle/_ref/libbvh_ref.so, built by
__graft_entry__.build() when BVH_REFERENCE_DIR names a checkout of madmann91/bvh):

    BVH_REFERENCE_DIR=<checkout> python tests/golden/make_golden.py

Outputs (small .npz files next to this script):
  kat_simple_example.npz   reference test/simple_example.cpp: 2 triangles, 1 ray -> prim 1 (BVH order), t=1, u=-0, v=0.5
  kat_serialize.npz        reference test/serialize.cpp: the 44-byte file of the 2-triangle BVH
  kat_cornell.npz          reference test/scenes/cornell_box.obj (36 triangles, fan-triangulated like
                           test/load_obj.cpp:57-96) through DefaultBuilder High: 37 nodes, and the
                           1024x1024 pinhole render of test/CMakeLists.txt:15-24: 1 027 152 hits
  soup2k_f32.npz, grid2k_f32.npz, soup1k_f64.npz, box12_f32.npz
                           seeded scenes (bvh_b200/scenes.py) with closest-hit (canonical tie-break and
                           reference last-visited), any-hit and robust results + per-ray step counts
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from bvh_b200 import scenes  # noqa: E402
from oracle.pyoracle import ANY_HIT, ROBUST, TIE_LOWEST_ID, Ref  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
ref = Ref()


def load_obj_tris(path):
    verts, tris = [], []
    for line in open(path):
        tok = line.split()
        if not tok:
            continue
        if tok[0] == "v":
            verts.append([float(x) for x in tok[1:4]])
        elif tok[0] == "f":
            idx = []
            for t in tok[1:]:
                i = int(t.split("/")[0])
                idx.append(i - 1 if i > 0 else len(verts) + i)
            for k in range(1, len(idx) - 1):          # triangle fan
                tris.append(verts[idx[0]] + verts[idx[k]] + verts[idx[k + 1]])
    return np.asarray(tris, np.float32)


def trace_all(tree, rays):
    out = {}
    for name, fl in (("lowest", TIE_LOWEST_ID), ("last", 0), ("any", ANY_HIT | TIE_LOWEST_ID),
                     ("robust", ROBUST | TIE_LOWEST_ID)):
        ids, t, u, v, st = ref.trace(tree, rays, flags=fl, stats=True)
        out.update({f"{name}_ids": ids, f"{name}_t": t, f"{name}_u": u, f"{name}_v": v, f"{name}_stats": st})
    return out


def scene_fixture(name, tris, rays, quality="high"):
    bb, cc = ref.tri_bboxes_centers(tris)
    tree = ref.build(bb, cc, quality=quality, threads=0)
    ref.set_triangles(tree, tris)
    bounds, index_values, prim_ids = tree.arrays()
    data = dict(tris=tris, rays=rays, bboxes=bb, centers=cc, ref_bounds=bounds, ref_index=index_values,
                ref_prim_ids=prim_ids, ref_serialized=np.frombuffer(ref.serialize(tree), np.uint8))
    data.update(trace_all(tree, rays))
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **data)
    print(name, "tris", tris.shape[0], "rays", rays.shape[0], "nodes", tree.node_count,
          "hits", int((data["lowest_ids"] != 0xFFFFFFFF).sum()))


# -- known answers of the reference's own tests -------------------------------------------------
two = np.array([[1, -1, 1, 1, 1, 1, -1, 1, 1], [1, -1, 1, -1, -1, 1, -1, 1, 1]], np.float32)
bb, cc = ref.tri_bboxes_centers(two)
tree = ref.build(bb, cc, quality="high", threads=0)           # pool overload, falls to serial (n < 1024)
ref.set_triangles(tree, two)
ray = np.array([[0, 0, 0, 0, 0, 1, 0, 100]], np.float32)
ids, t, u, v = ref.trace(tree, ray, flags=0)
_, _, prim_ids = tree.arrays()
slot = int(np.nonzero(prim_ids == ids[0])[0][0])
np.savez(os.path.join(OUT, "kat_simple_example.npz"), tris=two, ray=ray, bvh_order_prim=slot, orig_id=ids, t=t, u=u, v=v)
print("simple_example: primitive", slot, "distance", t[0], "u", u[0], "v", v[0])
tree2 = ref.build(bb, cc, quality="high", threads=-1)         # serialize.cpp uses the serial overload, default config
blob = ref.serialize(tree2)
np.savez(os.path.join(OUT, "kat_serialize.npz"), tris=two, bboxes=bb, centers=cc, blob=np.frombuffer(blob, np.uint8))
print("serialize:", len(blob), "bytes", blob.hex())

cornell = load_obj_tris(os.path.join(os.environ["BVH_REFERENCE_DIR"], "test", "scenes", "cornell_box.obj"))
bb, cc = ref.tri_bboxes_centers(cornell)
tree = ref.build(bb, cc, quality="high", threads=0)
ref.set_triangles(tree, cornell)
rays = scenes.primary_rays(1024, 1024, eye=(0, 1, 2), direction=(0, 0, -1), up=(0, 1, 0))
ids, t, u, v = ref.trace(tree, rays, flags=0, threads=0)
packed = np.packbits(ids != 0xFFFFFFFF)
np.savez_compressed(os.path.join(OUT, "kat_cornell.npz"), tris=cornell, node_count=tree.node_count,
                    hit_count=int((ids != 0xFFFFFFFF).sum()), hit_mask=packed,
                    ids_crc=np.uint64(int(ids.astype(np.uint64).sum())))
print("cornell: tris", cornell.shape[0], "nodes", tree.node_count, "hits", int((ids != 0xFFFFFFFF).sum()))

# -- seeded scenes --------------------------------------------------------------------------------
scene_fixture("soup2k_f32", scenes.soup(2000), scenes.make_primary("soup", 64, 64))
scene_fixture("grid2k_f32", scenes.grid(2048), scenes.make_primary("grid", 64, 64))
scene_fixture("box12_f32", scenes.box12(), scenes.make_primary("box12", 8, 8))
scene_fixture("soup1k_f64", scenes.soup(1000, dtype=np.float64), scenes.make_primary("soup", 48, 48, dtype=np.float64))
t64 = scenes.soup(1500)
scene_fixture("soup_incoherent_f32", t64, scenes.incoherent_rays(t64, 4096))
