// bvh_b200/csrc/refit_core.cuh — the bottom-up pass (reference Bvh::traverse_bottom_up, bvh.h:184-208) and the refit
// built on it (Bvh::refit, bvh.h:210-218), shared by the CUDA kernels of lbvh_build.cu, DeviceView::traverse_bottom_up
// (include/bvh/v2/cuda/intersect.cuh) and the host-side tests of the pass (tests/refit_host_test.cpp,
// tests/device_bottom_up_host_test.cpp).
//
// Two steps over the device node array (slot = reference index + 1, slot 0 unused):
//   refit_link       one call per slot: parent[child slot] = parent slot for the two children of an inner node, and
//                    the slot's arrival counter cleared;
//   climb_from_leaf  one call per slot, after every refit_link: a leaf calls leaf(i, begin, end), then climbs.  At each
//                    parent the first child to arrive stops, the second calls inner(i, left) and climbs on (i, left:
//                    reference indices; the right child is left + 1).  Every inner node's call comes once, after both
//                    of its children's, so a result that combines only the children's values does not depend on the
//                    order in which the leaves are processed.
// refit_from_leaf is the climb whose leaf folds its primitives' boxes into the empty box in BVH order (BBox::extend,
// bbox.h:23-27: robust_min / robust_max with the accumulator first, starting from +-max) and whose inner node unions the
// two child boxes in the reference's order (left.extend(right), bvh.h:213-217).  Where a leaf's primitive boxes come from
// is the caller's: `box_of(k, id, bmin, bmax)` gives the box of BVH slot k, whose original primitive id is id (BoxSource
// below: per-primitive boxes; lbvh_build.cu: triangles).
#pragma once

#include "build_core.cuh"

#if defined(__CUDACC__)
#include <cuda/atomic>
#endif

namespace bvhb200 {

// Per-primitive boxes in the original primitive order, struct bvh_bboxNN (min xyz, max xyz).
template <typename T> struct BoxSource {
    const T* boxes;
    BVH_HD void operator()(uint32_t, uint32_t id, T bmin[3], T bmax[3]) const {
        const T* b = boxes + 6 * (size_t)id;
        for (int a = 0; a < 3; ++a) {
#if defined(__CUDA_ARCH__)
            bmin[a] = __ldg(b + a); bmax[a] = __ldg(b + 3 + a);
#else
            bmin[a] = b[a]; bmax[a] = b[3 + a];
#endif
        }
    }
};

template <typename T>
BVH_HD void refit_link(const DevNode<T>* __restrict__ nodes, size_t slots, size_t i, uint32_t* __restrict__ parent,
                       int* __restrict__ flags) {
    flags[i] = 0;
    const auto index = nodes[i].index;
    if (index_count(index) == 0) {
        const size_t first = (size_t)index_first(index) + 1;          // device slot of the left child
        if (first + 1 < slots) { parent[first] = (uint32_t)i; parent[first + 1] = (uint32_t)i; }
    }
    if (i == 1) parent[1] = 0;
}

// The sibling's record was written by another thread (another SM on the device): read it through L2.
template <typename T> BVH_HD DevNode<T> refit_load_child(const DevNode<T>* p) {
#if defined(__CUDA_ARCH__)
    DevNode<T> out;
    const uint4* s = reinterpret_cast<const uint4*>(p);
    uint4* d = reinterpret_cast<uint4*>(&out);
    #pragma unroll
    for (int k = 0; k < (int)(sizeof(DevNode<T>) / 16); ++k) d[k] = __ldcg(s + k);
    return out;
#else
    return *p;
#endif
}

// Arrival at a parent: returns how many children arrived before.  On the device the exchange is acquire-release: the
// release half publishes the child record written just before, the acquire half makes the sibling's record visible.
BVH_HD int refit_arrive(int* flag) {
#if defined(__CUDA_ARCH__)
    cuda::atomic_ref<int, cuda::thread_scope_device> f(*flag);
    return f.fetch_add(1, cuda::memory_order_acq_rel);
#else
    return (*flag)++;
#endif
}

// The climb from slot i (nothing when it is an inner node).  On the device the arrival is acquire-release (refit_arrive),
// so the second child's thread sees every global write of the calls below the first child before it calls inner.
template <typename T, typename LeafFn, typename InnerFn>
BVH_HD void climb_from_leaf(const DevNode<T>* nodes, size_t i, const uint32_t* __restrict__ parent, int* __restrict__ flags,
                            LeafFn&& leaf, InnerFn&& inner) {
    const auto index = nodes[i].index;
    const uint32_t count = index_count(index);
    if (count == 0) return;
    const size_t first = (size_t)index_first(index);
    leaf(i - 1, first, first + count);
    size_t node = i;
    while (node != 1) {
        const size_t p = parent[node];
        if (p == 0) return;                                            // dead slot (collapsed subtree)
        if (refit_arrive(flags + p) == 0) return;                      // the sibling will carry on
        inner(p - 1, (size_t)index_first(nodes[p].index));
        node = p;
    }
}

template <typename T, typename BoxOf>
BVH_HD void refit_from_leaf(DevNode<T>* __restrict__ nodes, size_t i, const uint32_t* __restrict__ parent,
                            int* __restrict__ flags, const uint32_t* __restrict__ prim_ids, const BoxOf& box_of) {
    using R = Real<T>;
    climb_from_leaf<T>(nodes, i, parent, flags,
        [&](size_t node, size_t begin, size_t end) {
            T bmin[3] = { R::max(), R::max(), R::max() };
            T bmax[3] = { R::neg(R::max()), R::neg(R::max()), R::neg(R::max()) };
            for (uint32_t k = (uint32_t)begin; k < (uint32_t)end; ++k) {
                T pmin[3], pmax[3];
                box_of(k, prim_ids[k], pmin, pmax);
                for (int a = 0; a < 3; ++a) { bmin[a] = robust_min(bmin[a], pmin[a]); bmax[a] = robust_max(bmax[a], pmax[a]); }
            }
            write_node(nodes + node + 1, bmin, bmax, nodes[node + 1].index);
        },
        [&](size_t node, size_t left) {
            const DevNode<T> l = refit_load_child(nodes + left + 1), r = refit_load_child(nodes + left + 2);
            T pmin[3], pmax[3];
            for (int a = 0; a < 3; ++a) {
                pmin[a] = robust_min(l.bounds[2 * a], r.bounds[2 * a]);
                pmax[a] = robust_max(l.bounds[2 * a + 1], r.bounds[2 * a + 1]);
            }
            write_node(nodes + node + 1, pmin, pmax, nodes[node + 1].index);
        });
}

} // namespace bvhb200
