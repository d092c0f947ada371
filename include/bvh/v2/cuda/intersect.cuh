// include/bvh/v2/cuda/intersect.cuh — traverse a GPU-built BVH from your own CUDA kernels.
//
// The reference library's ray extension point is Bvh::intersect<IsAnyHit, IsRobust>(ray, start, stack, leaf_fn,
// inner_fn) (reference bvh.h:59-73,159-182): the library walks the tree, the caller intersects the primitives of every
// leaf it reaches and shrinks ray.tmax on a hit.  DeviceView::intersect is that call on the device, over the tree a
// handle keeps on its GPU.  It runs the library's own stack machine (bvhb200::traverse_top_down, traverse_core.cuh, the
// one the batched kernels use), so it visits the same leaves in the same order as the reference's Bvh::intersect on the
// same tree.  The general form, Bvh::traverse_top_down with the caller's own node test, is
// DeviceView::traverse_top_down ("Queries other than rays", below).
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
// Queries other than rays: view.traverse_top_down<IsAnyHit>(start, stack, leaf_fn, node_fn) is the reference's
// Bvh::traverse_top_down (bvh.h:59-65,124-157), of which intersect is one instance.  It starts at `start`; while the
// current node is an inner node it calls node_fn on its two children and descends to the near one, pushes the far one
// when both are hit, and pops the stack when neither is; at a leaf it calls leaf_fn; it ends when the stack is empty.
//   * node function: called as node_fn(const Node& left, const Node& right) with register copies of the two children
//     (node.bounds[6] as minx, maxx, miny, maxy, minz, maxz, node.index), or as node_fn(left, right, size_t left_index)
//     when it takes a third argument: the reference index of the left child (the right one is left_index + 1), what
//     `&left - bvh.nodes.data()` gives on the host, so that it can read data the caller keeps per node (below, "Data per
//     node").  It returns anything that unpacks with a
//     structured binding into three values convertible to bool, (hit_left, hit_right, should_swap): an aggregate of
//     three bools, cuda::std::tuple on the device or std::tuple on the host (std::tuple is not device code).
//     should_swap (visit the right child first) applies when both children are hit, whatever IsAnyHit is;
//   * leaf function: leaf_fn(size_t begin, size_t end) -> bool with BVH-order slots, as for intersect; with IsAnyHit a
//     true return ends the traversal.  A leaf `start` gets one leaf_fn call and no node_fn call;
//   * shared state: the two functions may share state (a search radius the leaf shrinks, a count); every node_fn call
//     comes after all earlier leaf_fn calls have returned;
//   * stacks: the same as for intersect, with the same bound, stack_bound() = depth + 1.
// Each sibling pair is read as one aligned 64-byte (float) / 128-byte (double) block through the read-only path.  A
// box-overlap query (collision broad phase), counting the primitives whose boxes overlap a query box:
//
//     struct Pick { bool left, right, swap; };
//     __device__ bool overlaps(const float* b, const bvh_bbox3f& q) {        // b: minx, maxx, miny, maxy, minz, maxz
//         return b[0] <= q.max.x && q.min.x <= b[1] && b[2] <= q.max.y && q.min.y <= b[3] &&
//                b[4] <= q.max.z && q.min.z <= b[5];
//     }
//     __global__ void overlap(View view, const bvh_bbox3f* boxes, const bvh_bbox3f* queries, uint32_t* counts, size_t n) {
//         const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
//         if (i >= n) return;
//         const bvh_bbox3f q = queries[i];
//         View::SmallStack<64> stack;
//         uint32_t count = 0;
//         view.traverse_top_down<false>(view.root_index(), stack,
//             [&](size_t begin, size_t end) {
//                 for (size_t k = begin; k < end; ++k) {
//                     const bvh_bbox3f b = boxes[view.prim_id(k)];             // original order
//                     const float f[6] = { b.min.x, b.max.x, b.min.y, b.max.y, b.min.z, b.max.z };
//                     count += overlaps(f, q);
//                 }
//                 return false;
//             },
//             [&](const View::Node& l, const View::Node& r) { return Pick { overlaps(l.bounds, q), overlaps(r.bounds, q), false }; });
//         counts[i] = count;
//     }
//
// Data per node: view.traverse_bottom_up(workspace, workspace_bytes, leaf_fn, inner_fn[, stream]) is the reference's
// Bvh::traverse_bottom_up (bvh.h:184-208), the pass Bvh::refit is built on, for data the caller computes per node: mass
// and centre of mass (Barnes-Hut), summed power and normal cones (light trees), a subtree's largest radius or speed, its
// primitive count.  It runs on the GPU, one thread per leaf climbing towards the root, in two kernels on `stream` (the
// handle's by default) with no host synchronisation: bottom_up_link_kernel, then bottom_up_climb_kernel, over slots
// [1, node_count].
//   * leaf_fn(size_t node, size_t begin, size_t end) is called once per leaf, with its reference index and its BVH-order
//     primitive range [begin, end) (view.prim_id(k) is the original id of slot k, as for intersect);
//   * inner_fn(size_t node, size_t left) is called once per inner node, with its reference index and its left child's
//     (the right one is left + 1);
//   * both are device function objects, copied to the kernel by value: a struct with a __device__ (or
//     __host__ __device__) operator(), or an extended __device__ lambda (nvcc --extended-lambda);
//   * every node of a tree whose nodes are all reachable from the root gets exactly one call; every tree the library
//     builds, and every tree it loads from the reference's format, is such a tree;
//   * an inner node's call comes after both of its children's calls, and their global writes are visible to it (the
//     arrival at a parent is an acquire-release atomic at device scope).  Data the pass writes must not be read through
//     __ldg or a `const __restrict__` pointer inside the pass: the read-only path does not see other threads' writes;
//   * the order is otherwise unspecified, and differs from run to run on the device.  A function that combines only its
//     children's values (and its leaf's primitives) therefore gives a result that does not depend on the order;
//   * workspace: view.bottom_up_workspace_bytes() bytes of device memory, allocated by the caller and not initialised:
//     the pass writes its parent links and clears its arrival flags itself, so the same workspace serves pass after pass
//     on one stream.  Two passes must not share one workspace at the same time.  A smaller workspace throws
//     std::length_error, a failed launch std::runtime_error;
//   * compiled as plain host C++, the pass runs serially on host-resident copies, in the reference's order: leaves in
//     descending index, each climbing while both children of the parent are done, which is the call sequence of
//     Bvh::traverse_bottom_up.
// Subtree mass and centre of mass, then a Barnes-Hut potential that reads them through the three-argument node test
// (compile with --fmad=false to match a host computation bit for bit):
//
//     struct MassCentre {                                                  // one object serves as leaf_fn and inner_fn
//         const uint32_t* prim_ids; const float* pos; const float* mass;  // pos: x, y, z per particle, original order
//         float* node_mass; float* node_centre;                            // node_count and 3 * node_count floats
//         __device__ void operator()(size_t node, size_t begin, size_t end) const {          // leaf
//             float m = 0, c[3] = { 0, 0, 0 };
//             for (size_t k = begin; k < end; ++k) {
//                 const uint32_t id = prim_ids[k];
//                 m += mass[id];
//                 for (int a = 0; a < 3; ++a) c[a] += mass[id] * pos[3 * id + a];
//             }
//             node_mass[node] = m;
//             for (int a = 0; a < 3; ++a) node_centre[3 * node + a] = c[a] / m;
//         }
//         __device__ void operator()(size_t node, size_t left) const {                        // inner: after both children
//             const float ml = node_mass[left], mr = node_mass[left + 1], m = ml + mr;
//             node_mass[node] = m;
//             for (int a = 0; a < 3; ++a)
//                 node_centre[3 * node + a] = (ml * node_centre[3 * left + a] + mr * node_centre[3 * (left + 1) + a]) / m;
//         }
//     };
//     size_t bytes = view.bottom_up_workspace_bytes();                     // on the host
//     void* workspace; cudaMallocAsync(&workspace, bytes, stream);
//     const MassCentre mc { view.prim_ids, d_pos, d_mass, d_node_mass, d_node_centre };
//     view.traverse_bottom_up(workspace, bytes, mc, mc, stream);
//     potential<<<blocks, 128, 0, stream>>>(view, d_node_mass, d_node_centre, d_pos, d_mass, d_points, m, 0.25f, d_phi);
//
//     __global__ void potential(View view, const float* node_mass, const float* node_centre, const float* pos,
//                               const float* mass, const float* points, size_t m, float theta2, float* phi) {
//         const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
//         if (i >= m) return;
//         const float p[3] = { points[3 * i], points[3 * i + 1], points[3 * i + 2] };
//         auto dist2 = [&](const float* c) { float d = 0; for (int a = 0; a < 3; ++a) d += (c[a] - p[a]) * (c[a] - p[a]); return d; };
//         float sum = 0;
//         // far enough (node size < theta * distance): the node's mass at its centre, and no descent
//         auto open = [&](const View::Node& n, size_t k) {
//             const float size = fmaxf(fmaxf(n.bounds[1] - n.bounds[0], n.bounds[3] - n.bounds[2]), n.bounds[5] - n.bounds[4]);
//             const float d2 = dist2(node_centre + 3 * k);
//             if (size * size < theta2 * d2) { sum -= node_mass[k] / sqrtf(d2); return false; }
//             return true;
//         };
//         View::SmallStack<64> stack;
//         view.traverse_top_down<false>(view.root_index(), stack,
//             [&](size_t begin, size_t end) {
//                 for (size_t k = begin; k < end; ++k) {
//                     const uint32_t id = view.prim_id(k);
//                     sum -= mass[id] / sqrtf(dist2(pos + 3 * id));
//                 }
//                 return false;
//             },
//             [&](const View::Node& l, const View::Node& r, size_t left) {
//                 const bool open_left = open(l, left), open_right = open(r, left + 1);
//                 return Pick { open_left, open_right, false };
//             });
//         phi[i] = sum;
//     }
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

#include "refit_core.cuh"
#include "traverse_core.cuh"

namespace bvh::v2::cuda {

namespace detail {
template <typename T> struct ViewTypes;
template <> struct ViewTypes<float>  { using CView = bvh_device_view3f; using Ray = bvh_ray3f; };
template <> struct ViewTypes<double> { using CView = bvh_device_view3d; using Ray = bvh_ray3d; };
struct NoInnerFn { template <typename I> BVH_HD void operator()(I) const {} };
}

#if defined(__CUDACC__)
// The two kernels of DeviceView::traverse_bottom_up, one thread per slot of [1, slots).
template <typename T>
__global__ void bottom_up_link_kernel(const bvhb200::DevNode<T>* __restrict__ nodes, size_t slots, uint32_t* __restrict__ parent,
                                      int* __restrict__ flags) {
    const size_t i = 1 + blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < slots) bvhb200::refit_link(nodes, slots, i, parent, flags);
}
template <typename T, typename LeafFn, typename InnerFn>
__global__ void bottom_up_climb_kernel(const bvhb200::DevNode<T>* nodes, size_t slots, const uint32_t* __restrict__ parent,
                                       int* __restrict__ flags, LeafFn leaf_fn, InnerFn inner_fn) {
    const size_t i = 1 + blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < slots) bvhb200::climb_from_leaf<T>(nodes, i, parent, flags, leaf_fn, inner_fn);
}
#endif

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

    // Bvh::traverse_top_down<IsAnyHit> (reference bvh.h:59-65,124-157) with the caller's node test: see "Queries other
    // than rays" at the top of this file.
    template <bool IsAnyHit, typename Stack, typename LeafFn, typename NodeFn>
    BVH_HD void traverse_top_down(Index start, Stack& stack, LeafFn&& leaf_fn, NodeFn&& node_fn) const {
        bvhb200::traverse_nodes<T, IsAnyHit>(
            nodes, start, stack,
            [&](Index begin, Index end) { return static_cast<bool>(leaf_fn(static_cast<size_t>(begin), static_cast<size_t>(end))); },
            node_fn);
    }

    // Bvh::traverse_bottom_up (reference bvh.h:184-208) with the caller's leaf and inner functions: see "Data per node"
    // at the top of this file.  The workspace is the parent links and the arrival flags, one of each per slot.
    BVH_HD size_t bottom_up_workspace_bytes() const { return 2 * (node_count + 1) * sizeof(uint32_t); }

    template <typename LeafFn, typename InnerFn>
    void traverse_bottom_up(void* workspace, size_t workspace_bytes, LeafFn leaf_fn, InnerFn inner_fn) const {
        traverse_bottom_up(workspace, workspace_bytes, leaf_fn, inner_fn, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <typename LeafFn, typename InnerFn>
    void traverse_bottom_up(void* workspace, size_t workspace_bytes, LeafFn leaf_fn, InnerFn inner_fn, void* on_stream) const {
        const size_t need = bottom_up_workspace_bytes();
        if (workspace_bytes < need || (need && !workspace))
            throw std::length_error("bvh::v2::cuda::DeviceView::traverse_bottom_up: a workspace of " +
                                    std::to_string(workspace ? workspace_bytes : 0) + " bytes is too small for " +
                                    std::to_string(node_count) + " nodes (" + std::to_string(need) + " bytes)");
        if (node_count == 0) return;
        const size_t slots = node_count + 1;
        uint32_t* parent = static_cast<uint32_t*>(workspace);
        int* flags = reinterpret_cast<int*>(parent + slots);
#if defined(__CUDACC__)
        cudaStream_t s = static_cast<cudaStream_t>(on_stream);
        int previous = 0;
        check(cudaGetDevice(&previous), "cudaGetDevice");
        if (previous != device) check(cudaSetDevice(device), "cudaSetDevice");
        // a slot no inner node points to (possible only in a tree with unreachable nodes) stops the climb
        cudaError_t e = cudaMemsetAsync(parent, 0, slots * sizeof(uint32_t), s);
        const unsigned block = 256, grid = (unsigned)((node_count + block - 1) / block);
        if (e == cudaSuccess) {
            bottom_up_link_kernel<T><<<grid, block, 0, s>>>(nodes, slots, parent, flags);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) {
            bottom_up_climb_kernel<T><<<grid, block, 0, s>>>(nodes, slots, parent, flags, leaf_fn, inner_fn);
            e = cudaGetLastError();
        }
        if (previous != device) cudaSetDevice(previous);
        check(e, "launch");
#else
        (void)on_stream;
        for (size_t i = 0; i < slots; ++i) parent[i] = 0;
        for (size_t i = 1; i < slots; ++i) bvhb200::refit_link(nodes, slots, i, parent, flags);
        for (size_t i = slots; i-- > 1;) bvhb200::climb_from_leaf<T>(nodes, i, parent, flags, leaf_fn, inner_fn);
#endif
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
#if defined(__CUDACC__)
    static void check(cudaError_t e, const char* what) {
        if (e != cudaSuccess)
            throw std::runtime_error(std::string("bvh::v2::cuda::DeviceView::traverse_bottom_up: ") + what + ": " +
                                     cudaGetErrorString(e));
    }
#endif
    BVH_HD static void load(const Ray& ray, bvhb200::RayCtx<T>& r) {
        r.org[0] = ray.org.x; r.org[1] = ray.org.y; r.org[2] = ray.org.z;
        r.dir[0] = ray.dir.x; r.dir[1] = ray.dir.y; r.dir[2] = ray.dir.z;
        r.tmin = ray.tmin; r.tmax = ray.tmax;
    }
};

} // namespace bvh::v2::cuda
