#!/usr/bin/env python
"""Node loads per traversal step when a child's second 16-byte half is loaded only if its first half does not already
reject the box.  CPU only: replays the stack machine (scripts/split_fetch_count.cpp) on the host-emulated High tree,
which equals the GPU-built tree node for node, with bench.py's scenes, seeds and cameras at full size.

    python scripts/split_fetch_count.py [--configs c2/soup c2/grid c3/soup c5/soup] [--rays-stride S]

A float node is two 16-byte halves: [minx maxx miny maxy] and [minz maxz index spare] (double: two 32-byte halves,
two loads each).  For every child box test the replay records whether the x/y half alone rejects the box, whether the
z half alone does, and whether the full test hits it.  Loads per step (counted in halves, 4 without the split):
  (a) x/y half first;  (b) z half first;  (c) x/y first until the ray has a hit, z first afterwards.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tests.helpers import HostEmul, _ptr  # noqa: E402


def counter_lib(tmp: str):
    src = os.path.join(ROOT, "scripts", "split_fetch_count.cpp")
    out = os.path.join(tmp, "libsplit_fetch_count.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                           "-x", "c++", "-I", os.path.join(ROOT, "bvh_b200", "csrc"), src, "-o", out])
    lib = C.CDLL(out)
    for s in ("3f", "3d"):
        getattr(lib, f"count_split_fetch_{s}").argtypes = [C.c_void_p] * 4 + [C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def count(lib, emul, config: str, kind: str, stride: int):
    cfg = bench.CONFIGS[config]
    tris = bench.make_tris(cfg, kind)
    rays = np.ascontiguousarray(bench.make_rays(cfg, kind, tris)[::stride])
    tree = emul.build(tris=tris, quality="high", morton_bits=63 if tris.shape[0] >= 1 << 22 else 30)
    out = np.zeros(16, np.uint64)
    steps = np.zeros(1, np.uint64)
    s = "3f" if tris.dtype == np.float32 else "3d"
    getattr(lib, f"count_split_fetch_{s}")(_ptr(tree["nodes"]), _ptr(tree["tris"]), _ptr(tree["prim_ids"]), _ptr(rays),
                                          rays.shape[0], int(cfg["any_hit"]), _ptr(out), _ptr(steps))
    return rays.shape[0], int(steps[0]), out.reshape(2, 2, 2, 2).astype(np.float64)   # [has_hit, xy_rej, z_rej, hit]


def report(name: str, m: int, steps: int, c: np.ndarray) -> None:
    tests = c.sum()
    xy, z = c[:, 1].sum(), c[:, :, 1].sum()
    both = c[:, 1, 1].sum()
    only3 = c[:, 0, 0, 0].sum()
    hit = c[..., 1].sum()
    # loads in halves per child test: 1, plus 1 unless the first-loaded half rejects
    a = tests + (tests - xy)
    b = tests + (tests - z)
    pc = c[0].sum() + (c[0].sum() - c[0, 1].sum()) + c[1].sum() + (c[1].sum() - c[1, :, 1].sum())
    base = 2 * tests
    print(f"{name}: {m} rays, {steps / m:.2f} inner steps per ray, {tests:.0f} child tests "
          f"({c[1].sum() / tests:.1%} after the ray's first hit)")
    print(f"  rejected by x/y half {xy / tests:.1%}, by z half {z / tests:.1%} (by both {both / tests:.1%}), "
          f"only by all three axes {only3 / tests:.1%}, hit {hit / tests:.1%}")
    for label, loads in (("(a) x/y first", a), ("(b) z first", b), ("(c) x/y until hit, then z", pc)):
        print(f"  {label:28s} {2 * loads / tests:.3f} loads per step (4.000 without the split): {1 - loads / base:6.1%} fewer")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["c2/soup", "c2/grid", "c3/soup", "c5/soup"])
    ap.add_argument("--rays-stride", type=int, default=1, help="replay every S-th ray only (1: all of them)")
    args = ap.parse_args()
    emul = HostEmul()
    with tempfile.TemporaryDirectory() as tmp:
        lib = counter_lib(tmp)
        for item in args.configs:
            config, kind = item.split("/")
            report(item, *count(lib, emul, config, kind, args.rays_stride))


if __name__ == "__main__":
    main()
