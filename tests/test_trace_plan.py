"""Which traversal kernel a batched call runs, and with which scheduling settings (bvh_b200/csrc/trace_plan.h, compiled
with g++ into a temporary library; needs no GPU), and the values bvh_set_option refuses."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from bvh_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PERSISTENT_TMA, PERSISTENT, SIMPLE, STATS, PAIR, WIDE = 1, 2, 3, 4, 5, 6

SHIM = r"""
#include "trace_plan.h"
using namespace bvhb200;
// out = {kernel, sort_rays, refill_min, inner_budget}
extern "C" void plan(unsigned flags, int stats, int is_float, int wide_tree, int gather, unsigned long long n, int variant,
                     int use_wide, uint32_t refill_min, uint32_t inner_budget, uint32_t wide_budget, uint32_t* out) {
    const TracePlan p = plan_trace({ flags, stats != 0, is_float != 0, wide_tree != 0, gather != 0, n, variant, use_wide,
                                     refill_min, inner_budget, wide_budget });
    out[0] = (uint32_t)p.kernel; out[1] = p.sort_rays; out[2] = p.refill_min; out[3] = p.inner_budget;
}
"""


class Planner:
    def __init__(self, out_dir):
        lib = os.path.join(out_dir, "libtrace_plan.so")
        subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-fPIC", "-shared", "-x", "c++", "-I",
                        os.path.join(ROOT, "bvh_b200", "csrc"), "-", "-o", lib], input=SHIM, text=True, check=True)
        self.lib = C.CDLL(lib)
        self.lib.plan.argtypes = [C.c_uint, C.c_int, C.c_int, C.c_int, C.c_int, C.c_ulonglong, C.c_int, C.c_int,
                                  C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]

    def plan_trace(self, flags=0, stats=False, is_float=True, wide_tree=True, gather=False, n=1 << 20, variant=0, use_wide=0,
                   refill_min=0, inner_budget=0, wide_budget=4):
        """(kernel, sort_rays, refill_min, inner_budget) for one batched call."""
        out = np.zeros(4, np.uint32)
        self.lib.plan(flags, stats, is_float, wide_tree, gather, n, variant, use_wide, refill_min, inner_budget, wide_budget,
                      out.ctypes.data_as(C.c_void_p))
        return int(out[0]), bool(out[1]), int(out[2]), int(out[3])


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    return Planner(str(tmp_path_factory.mktemp("trace_plan")))


def kernel(planner, flags=0, **request):
    return planner.plan_trace(flags, **request)[0]


def test_kernel_names_match_the_property_report():
    assert api.KERNEL_NAMES[PERSISTENT_TMA] == "trace_persistent_kernel<kTma=true>"
    assert api.KERNEL_NAMES[PERSISTENT] == "trace_persistent_kernel<kTma=false>"
    assert api.KERNEL_NAMES[WIDE] == "trace_wide_kernel"


def test_statistics_win_over_every_flag(planner):
    for flags in (0, api.KERNEL_SIMPLE, api.KERNEL_WIDE, api.KERNEL_PAIR, api.KERNEL_TMA, api.KERNEL_SIMPLE | api.KERNEL_PAIR):
        assert kernel(planner, flags, stats=True) == STATS, flags
        assert kernel(planner, flags, stats=True, use_wide=1) == STATS, flags


def test_simple_comes_next(planner):
    for flags in (api.KERNEL_SIMPLE, api.KERNEL_SIMPLE | api.KERNEL_WIDE, api.KERNEL_SIMPLE | api.KERNEL_PAIR,
                  api.KERNEL_SIMPLE | api.KERNEL_TMA):
        assert kernel(planner, flags) == SIMPLE, flags
    assert kernel(planner, api.KERNEL_SIMPLE, use_wide=1, variant=1) == SIMPLE


def test_wide_kernel_rules(planner):
    assert kernel(planner, api.KERNEL_WIDE) == WIDE
    assert kernel(planner, api.KERNEL_WIDE | api.KERNEL_PAIR) == WIDE               # an explicit wide flag beats the pair flag
    assert kernel(planner, api.KERNEL_WIDE | api.ANY_HIT) == WIDE
    assert kernel(planner, 0, use_wide=1) == WIDE
    for binary in (api.KERNEL_PAIR, api.KERNEL_NO_TMA, api.KERNEL_TMA):           # use_wide yields to an explicit binary kernel
        assert kernel(planner, binary, use_wide=1) != WIDE, binary
    for order_sensitive in (api.TIE_LAST_VISITED, api.ROBUST):
        assert kernel(planner, api.KERNEL_WIDE | order_sensitive) == PERSISTENT
        assert kernel(planner, order_sensitive, use_wide=1) == PERSISTENT
    assert kernel(planner, api.KERNEL_WIDE, is_float=False) == PERSISTENT
    assert kernel(planner, 0, use_wide=1, is_float=False) == PERSISTENT
    assert kernel(planner, api.KERNEL_WIDE, wide_tree=False) == PERSISTENT          # the tree cannot be collapsed
    assert kernel(planner, api.KERNEL_WIDE | api.KERNEL_PAIR, wide_tree=False) == PAIR
    assert kernel(planner, 0, use_wide=0) == PERSISTENT


def test_pair_then_persistent(planner):
    assert kernel(planner, api.KERNEL_PAIR) == PAIR
    assert kernel(planner, api.KERNEL_PAIR | api.KERNEL_TMA) == PAIR
    assert kernel(planner, api.KERNEL_PAIR, is_float=False) == PAIR
    assert kernel(planner, api.KERNEL_PAIR, variant=1) == PAIR
    assert kernel(planner, 0) == PERSISTENT
    assert kernel(planner, api.KERNEL_NO_TMA) == PERSISTENT
    assert kernel(planner, api.KERNEL_TMA) == PERSISTENT_TMA
    assert kernel(planner, api.KERNEL_TMA | api.KERNEL_NO_TMA) == PERSISTENT_TMA
    assert kernel(planner, 0, variant=1) == PERSISTENT_TMA
    assert kernel(planner, 0, variant=1, is_float=False) == PERSISTENT_TMA
    assert kernel(planner, api.KERNEL_NO_TMA, variant=1) == PERSISTENT           # the flag beats the switch


def test_sort_rules(planner):
    big = 1 << 20
    sort = lambda flags, **q: planner.plan_trace(flags | api.SORT_RAYS, **{"n": big, **q})
    assert sort(0)[:2] == (PERSISTENT, True)
    assert sort(api.KERNEL_WIDE)[:2] == (WIDE, True)
    assert sort(api.KERNEL_TMA)[:2] == (PERSISTENT, True)                    # a sorted run is not contiguous: no bulk copies
    assert sort(0, variant=1)[:2] == (PERSISTENT, True)
    assert sort(api.KERNEL_PAIR)[:2] == (PAIR, False)
    assert sort(api.KERNEL_SIMPLE)[:2] == (SIMPLE, False)
    assert sort(0, stats=True)[:2] == (STATS, False)
    assert sort(0, gather=True)[:2] == (PERSISTENT, False)
    assert sort(api.KERNEL_TMA, gather=True)[:2] == (PERSISTENT_TMA, False)
    assert sort(0, n=(1 << 16) - 1)[1] is False
    assert sort(0, n=1 << 16)[1] is True
    assert sort(0, n=0xFFFFFFFE)[1] is True
    assert sort(0, n=0xFFFFFFFF)[1] is False
    assert planner.plan_trace(0, n=big)[1] is False


def test_auto_refill_and_budget(planner):
    settings = lambda flags=0, **q: planner.plan_trace(flags, **q)[2:]
    assert settings() == (14, 4)                                             # closest-hit, binary persistent kernels
    assert settings(api.KERNEL_TMA) == (14, 4)
    assert settings(api.ROBUST | api.TIE_LAST_VISITED) == (14, 4)
    assert settings(api.ANY_HIT) == (8, 8)
    assert settings(api.KERNEL_PAIR) == (8, 8)
    assert settings(api.KERNEL_WIDE) == (8, 4)                                # the wide kernel always takes wide_budget
    assert settings(api.KERNEL_WIDE, wide_budget=0xFFFFFFFF) == (8, 0xFFFFFFFF)
    assert settings(api.KERNEL_WIDE, inner_budget=2) == (8, 4)
    assert settings(refill_min=3, inner_budget=5) == (3, 5)                   # set explicitly: every kernel
    assert settings(api.KERNEL_PAIR | api.ANY_HIT, refill_min=3, inner_budget=0xFFFFFFFF) == (3, 0xFFFFFFFF)
    assert settings(api.KERNEL_WIDE, refill_min=20) == (20, 4)


def test_set_option_rejects_variants_it_does_not_name():
    """bvh_set_option: "variant" is 0 (streaming ray loads) or 1 (TMA-staged rays); any other value would select a kernel
    it does not name, so it is an error."""
    path = os.path.join(ROOT, "bvh_b200", "libbvh_c.so")
    if not os.path.exists(path):
        import bvh_b200.build_ext as b
        b.build()
    library = C.CDLL(path)
    library.bvh_set_option.argtypes = [C.c_char_p, C.c_long]
    library.bvh_last_error.restype = C.c_char_p
    for bad in (-1, 2, 3, 1 << 40):
        assert library.bvh_set_option(b"variant", bad) != 0, bad
        assert b"variant" in library.bvh_last_error()
    assert library.bvh_set_option(b"variant", 1) == 0 and library.bvh_set_option(b"variant", 0) == 0
