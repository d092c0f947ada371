// include/bvh/v2/cuda/intersect.cuh — traverse a GPU-built BVH from your own CUDA kernels.
//
// The reference library has one extension point, Bvh::intersect<IsAnyHit, IsRobust>(ray, start, stack, leaf_fn,
// inner_fn) (reference bvh.h:59-73,159-182): the library walks the tree, the caller intersects the primitives of every
// leaf it reaches and shrinks ray.tmax on a hit.  DeviceView::intersect is that call on the device, over the tree a
// handle keeps on its GPU.  It runs the library's own stack machine (bvhb200::traverse_top_down, traverse_core.cuh, the
// one the batched kernels use), so it visits the same leaves in the same order as the reference's Bvh::intersect on the
// same tree.
//
//     bvh3f* bvh = bvh3f_build(nullptr, bboxes, centers, n, nullptr);     // or bvh3f_build_triangles
//     bvh_device_view3f c;
//     bvh3f_get_device_view(bvh, &c);                                       // include/bvh_b200_device.h
//     auto view = bvh::v2::cuda::DeviceView<float>::from(c);               // pass it to the kernel by value
//
//     __global__ void kernel(bvh::v2::cuda::DeviceView<float> view, const MySphere* spheres, bvh_ray3f* rays, ...) {
//         using View = bvh::v2::cuda::DeviceView<float>;
//         bvh_ray3f ray = rays[i];
//         View::SmallStack<64> stack;                                      // capacity >= view.stack_bound()
//         size_t best = SIZE_MAX;
//         view.intersect<false, false>(ray, view.root_index(), stack, [&](size_t begin, size_t end) {
//             for (size_t k = begin; k < end; ++k)                         // BVH-order slots; spheres[view.prim_id(k)]
//                 if (my_test(spheres[view.prim_id(k)], ray)) { ray.tmax = ...; best = k; }
//             return best != SIZE_MAX;
//         });
//     }
//
// Compile with (nvcc 12.x, sm_90a):
//     nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -I <repo>/include -I <repo>/bvh_b200/csrc ...
// The traversal's own arithmetic uses round-to-nearest intrinsics and is exact under any flags.  A leaf function's
// arithmetic is the caller's: to match a host computation bit for bit, compile with --fmad=false (or write it with the
// __fadd_rn / __fmul_rn family), since nvcc otherwise contracts a * b + c into one FMA.  The header also compiles as
// plain host C++ (g++ -std=c++17, same include flags), where the same traversal runs on host-resident copies of the
// arrays.
//
// Rules a leaf function follows (the reference's, bvh.h:124-157):
//   * it receives a BVH-order range [begin, end); view.prim_id(k) is the original primitive id of slot k;
//   * it may shrink (or otherwise change) ray.tmax and ray.tmin: the next box test reads them.  Other ray fields are
//     read once, before the traversal starts;
//   * it returns whether it hit; with IsAnyHit a true return ends the traversal.
// The inner hook, when given, is called once per inner step with the reference index of the left child of the node
// being expanded (the right child is that index + 1), before the step's box tests: the reference's InnerFn, which
// receives those two nodes.
//
// Stacks: anything with push(Index) and try_pop(Index&) (false when empty), empty at the start.  A traversal holds at
// most view.stack_bound() = depth + 1 entries, and no stack checks its capacity on the device: check it on the host
// (DeviceView<T>::from(c, capacity) and bvh::v2::cuda::Accel<T>::device_view(capacity) throw when it is too small).
//   DeviceView<T>::SmallStack<N>   N entries per thread in registers / local memory (the reference's SmallStack);
//   DeviceView<T>::SharedStack     the batched kernels' shared-memory stack: depth + 2 entries per thread, laid out
//                                  [entry][thread] (no bank conflicts); make it with shared_stack(smem, blockDim.x)
//                                  from a dynamic shared array of shared_stack_bytes(blockDim.x) bytes.
#pragma once

#include <bvh_b200_device.h>
#include <cstddef>
#include <cstdint>
#include <stdexcept>
#include <string>

#include "traverse_core.cuh"

namespace bvh::v2::cuda {

namespace detail {
template <typename T> struct ViewTypes;
template <> struct ViewTypes<float>  { using CView = bvh_device_view3f; using Ray = bvh_ray3f; };
template <> struct ViewTypes<double> { using CView = bvh_device_view3d; using Ray = bvh_ray3d; };
struct NoInnerFn { template <typename I> BVH_HD void operator()(I) const {} };
}

// A plain-data view of one device tree (what bvhNN_get_device_view reports), passed to kernels by value.
template <typename T> struct DeviceView {
    using Scalar = T;
    using Index = typename bvhb200::Real<T>::UInt;      // a node's packed index: first id << 4 | primitive count
    using Ray = typename detail::ViewTypes<T>::Ray;     // bvh_ray3f / bvh_ray3d
    using Node = bvhb200::DevNode<T>;                   // { T bounds[6] (minx, maxx, miny, maxy, minz, maxz); Index index; pad }
    using Tri = bvhb200::DevTri<T>;                     // PrecomputedTri: p0, e1 = p0 - p1, e2 = p2 - p0, n = cross(e1, e2)
    template <unsigned Capacity> using SmallStack = bvhb200::ArrayStack<Index, Capacity>;
#if defined(__CUDACC__)
    using SharedStack = bvhb200::SmemStack<Index>;
#endif

    const Node* nodes = nullptr;        // node_count + 1 slots: reference node i at slot i + 1 (slot 0 is padding)
    const uint32_t* prim_ids = nullptr; // prim_ids[k]: original id of BVH-order primitive k
    const Tri* tris = nullptr;          // BVH-order triangles, or nullptr when none are attached
    size_t node_count = 0, prim_count = 0;
    size_t depth = 0;                   // longest chain of inner nodes below the root
    int device = 0;
    void* stream = nullptr;             // the handle's cudaStream_t

    static DeviceView from(const typename detail::ViewTypes<T>::CView& c) {
        DeviceView v;
        v.nodes = static_cast<const Node*>(c.nodes);
        v.prim_ids = c.prim_ids;
        v.tris = static_cast<const Tri*>(c.tris);
        v.node_count = c.node_count; v.prim_count = c.prim_count; v.depth = c.depth;
        v.device = c.device; v.stream = c.stream;
        return v;
    }
    // Same, for kernels whose per-thread stack holds `stack_capacity` entries: throws std::length_error when the tree
    // needs more.
    static DeviceView from(const typename detail::ViewTypes<T>::CView& c, size_t stack_capacity) {
        if (stack_capacity < c.depth + 1)
            throw std::length_error("bvh::v2::cuda::DeviceView: a stack of " + std::to_string(stack_capacity) +
                                    " entries is too small for a tree of depth " + std::to_string(c.depth));
        return from(c);
    }

    // get_root().index (reference bvh.h:54)
    BVH_HD Index root_index() const { return nodes[1].index; }
    // reference node i
    BVH_HD const Node& node(size_t i) const { return nodes[i + 1]; }
    BVH_HD size_t prim_id(size_t i) const { return prim_ids[i]; }
    // entries a traversal's stack can hold at once
    BVH_HD size_t stack_bound() const { return depth + 1; }
    // dynamic shared memory of a block of `threads` threads that each use a SharedStack
    BVH_HD size_t shared_stack_bytes(unsigned threads) const { return (depth + 2) * (size_t)threads * sizeof(Index); }
#if defined(__CUDACC__)
    // this thread's stack in a dynamic shared array of shared_stack_bytes(threads) bytes
    __device__ __forceinline__ static SharedStack shared_stack(void* smem, unsigned threads) {
        return SharedStack(static_cast<Index*>(smem) + threadIdx.x, threads, 0);
    }
#endif

    // Bvh::intersect<IsAnyHit, IsRobust> (reference bvh.h:159-182): see the rules at the top of this file.  `ray` is
    // read again after every leaf call, so the leaf function updates the same object (through its own reference).
    template <bool IsAnyHit, bool IsRobust, typename Stack, typename LeafFn, typename InnerFn = detail::NoInnerFn>
    BVH_HD void intersect(const Ray& ray, Index start, Stack& stack, LeafFn&& leaf_fn, InnerFn&& inner_fn = {}) const {
        bvhb200::RayCtx<T> r;
        load(ray, r);
        bvhb200::ray_prologue<T, IsRobust>(r);
        bvhb200::traverse_top_down<T, IsAnyHit, IsRobust>(
            nodes, r, start, stack,
            [&](Index begin, Index end) {
                const bool hit = static_cast<bool>(leaf_fn(static_cast<size_t>(begin), static_cast<size_t>(end)));
                r.tmin = ray.tmin;
                r.tmax = ray.tmax;
                return hit;
            },
            [&](Index first_child) { inner_fn(static_cast<size_t>(first_child)); });
    }

    // PrecomputedTri::intersect (reference tri.h:55-74) on BVH-order triangle k: true, with the hit's distance and
    // barycentrics, when the ray meets it at a distance in [ray.tmin, ray.tmax].  The batched kernels' own test.
    BVH_HD bool intersect_tri(size_t k, const Ray& ray, T& t, T& u, T& v) const {
        bvhb200::RayCtx<T> r;
        load(ray, r);
        bvhb200::HitState<T> hit { bvhb200::kInvalidId, r.tmax, T(0), T(0) };
        Tri tri;
        bvhb200::load_tri(tris + k, tri);
        if (!bvhb200::tri_test<T>(tri, static_cast<uint32_t>(k), prim_ids, false, r, hit)) return false;
        t = hit.t; u = hit.u; v = hit.v;
        return true;
    }

private:
    BVH_HD static void load(const Ray& ray, bvhb200::RayCtx<T>& r) {
        r.org[0] = ray.org.x; r.org[1] = ray.org.y; r.org[2] = ray.org.z;
        r.dir[0] = ray.dir.x; r.dir[1] = ray.dir.y; r.dir[2] = ray.dir.z;
        r.tmin = ray.tmin; r.tmax = ray.tmax;
    }
};

} // namespace bvh::v2::cuda
