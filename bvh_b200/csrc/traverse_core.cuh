// bvh_b200/csrc/traverse_core.cuh — the per-ray stack machine.
//
// A faithful restatement of Bvh::traverse_top_down / Bvh::intersect (reference bvh.h:124-182) for a
// single ray: near/far ordering by entry distance with ties going LEFT first (`>` at bvh.h:180),
// far child pushed, pop on a double miss, any-hit leaves as soon as a leaf reports a hit.  The leaf
// convention is the one every reference caller uses (benchmark.cpp:281-292): test each primitive of
// the leaf in order and shrink tmax on a hit.
//
// The same code runs in four places: the one-thread-per-ray kernel, the persistent kernel (which
// splits it into an inner phase and a leaf phase, traverse.cu), the host emulation compiled by
// g++ for the CPU tests (tests/host_emul.cpp) and, through traverse_top_down with the caller's leaf,
// the device traversal API (include/bvh/v2/cuda/intersect.cuh).  traverse_nodes is the same stack machine with the
// caller's node test instead of the ray's (DeviceView::traverse_top_down); its step, node_step, is also the inner step
// of DeviceView::query's persistent kernel.
#pragma once

#include "core.cuh"

#include <type_traits>

namespace bvhb200 {

// Two adjacent nodes (a sibling pair) in registers.
template <typename T> struct NodePair {
    T lb[6], rb[6];
    typename Real<T>::UInt li, ri;
};

#if defined(__CUDACC__)
// 32 bytes as two 128-bit loads from one 32-byte aligned block: sm_90 has no 256-bit global load, and the widest
// vector load it has (LDG.E.128) keeps both halves in the same L1 sector pair.
__device__ __forceinline__ void ldg256(const void* p, uint32_t (&w)[8]) {
    asm("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%8];\n\t"
        "ld.global.nc.v4.b32 {%4,%5,%6,%7}, [%8+16];"
        : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(p));
}
// Node loads allocate their line in L1 (BVH_NODE_NA=0).  Measured on an H100 80GB HBM3 SXM at a 400 W power limit
// (bench.py, 1M-triangle soup, 10M rays): allocating loads take 4.09 instead of 6.96 ms per step for coherent primary
// rays and 11.0 instead of 23.1 ms for incoherent any-hit rays; BVH_NODE_NA=1 (ld.global.nc.L1::no_allocate) keeps the
// other form selectable.
#ifndef BVH_NODE_NA
#define BVH_NODE_NA 0
#endif
#ifndef BVH_TRI_NA
#define BVH_TRI_NA 0
#endif
__device__ __forceinline__ void ldg256_na(const void* p, uint32_t (&w)[8]) {
    asm("ld.global.nc.L1::no_allocate.v4.b32 {%0,%1,%2,%3}, [%8];\n\t"
        "ld.global.nc.L1::no_allocate.v4.b32 {%4,%5,%6,%7}, [%8+16];"
        : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "l"(p));
}
__device__ __forceinline__ void ldg256_node(const void* p, uint32_t (&w)[8]) {
#if BVH_NODE_NA
    ldg256_na(p, w);
#else
    ldg256(p, w);
#endif
}
__device__ __forceinline__ float4 ldg128_tri(const float4* p) {
#if BVH_TRI_NA
    float4 v;
    asm("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
#else
    return __ldg(p);
#endif
}
__device__ __forceinline__ void ldg256(const void* p, unsigned long long (&w)[4]) {
    asm("ld.global.nc.v2.b64 {%0,%1}, [%4];\n\t"
        "ld.global.nc.v2.b64 {%2,%3}, [%4+16];" : "=l"(w[0]), "=l"(w[1]), "=l"(w[2]), "=l"(w[3]) : "l"(p));
}
__device__ __forceinline__ void ldg256_node(const void* p, unsigned long long (&w)[4]) {
#if BVH_NODE_NA
    asm("ld.global.nc.L1::no_allocate.v2.b64 {%0,%1}, [%4];\n\t"
        "ld.global.nc.L1::no_allocate.v2.b64 {%2,%3}, [%4+16];" : "=l"(w[0]), "=l"(w[1]), "=l"(w[2]), "=l"(w[3]) : "l"(p));
#else
    ldg256(p, w);
#endif
}
#endif

#if defined(__CUDA_ARCH__)
// A sibling pair is one naturally aligned 64-byte (float) / 128-byte (double) block, read through the read-only path:
// on sm_90a a 32-byte float node is two 128-bit loads (LDG.E.128), a pair four.  The number of load instructions
// matters because with divergent rays every load costs one L1 wavefront per distinct piece the warp addresses (the
// traversal is bound by the L1 data pipe, not by DRAM; DESIGN.md §3).
__device__ __forceinline__ void load_pair(const DevNode<float>* __restrict__ p, NodePair<float>& o) {
    uint32_t a[8], b[8];
    ldg256_node(p, a);
    ldg256_node(p + 1, b);
    #pragma unroll
    for (int k = 0; k < 6; ++k) { o.lb[k] = __uint_as_float(a[k]); o.rb[k] = __uint_as_float(b[k]); }
    o.li = a[6]; o.ri = b[6];
}
__device__ __forceinline__ void load_pair(const DevNode<double>* __restrict__ p, NodePair<double>& o) {
    unsigned long long a[4], b[4], c[4], d[4];
    const unsigned char* q = reinterpret_cast<const unsigned char*>(p);
    ldg256_node(q, a); ldg256_node(q + 32, b); ldg256_node(q + 64, c); ldg256_node(q + 96, d);
    #pragma unroll
    for (int k = 0; k < 4; ++k) { o.lb[k] = __longlong_as_double((long long)a[k]); o.rb[k] = __longlong_as_double((long long)c[k]); }
    o.lb[4] = __longlong_as_double((long long)b[0]); o.lb[5] = __longlong_as_double((long long)b[1]); o.li = b[2];
    o.rb[4] = __longlong_as_double((long long)d[0]); o.rb[5] = __longlong_as_double((long long)d[1]); o.ri = d[2];
}
// The two halves of a float node, [minx maxx miny maxy] and [minz maxz index spare], one LDG.E.128 each, for the
// closest-hit step that loads a child's second half only when its first does not reject it (inner_step).
// The first halves of both nodes of the pair at p:
__device__ __forceinline__ void load_first_halves(const DevNode<float>* __restrict__ p, NodePair<float>& o) {
    uint32_t a[4], b[4];
#if BVH_NODE_NA
    asm("ld.global.nc.L1::no_allocate.v4.b32 {%0,%1,%2,%3}, [%8];\n\t"
        "ld.global.nc.L1::no_allocate.v4.b32 {%4,%5,%6,%7}, [%8+32];"
#else
    asm("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%8];\n\t"
        "ld.global.nc.v4.b32 {%4,%5,%6,%7}, [%8+32];"
#endif
        : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3]), "=r"(b[0]), "=r"(b[1]), "=r"(b[2]), "=r"(b[3]) : "l"(p));
    #pragma unroll
    for (int k = 0; k < 4; ++k) { o.lb[k] = __uint_as_float(a[k]); o.rb[k] = __uint_as_float(b[k]); }
}
// The second half of the node at p: b[4], b[5] and its index.
__device__ __forceinline__ void load_second_half(const DevNode<float>* __restrict__ p, float (&b)[6], uint32_t& index) {
    uint32_t w0, w1, w2, w3;
#if BVH_NODE_NA
    asm("ld.global.nc.L1::no_allocate.v4.b32 {%0,%1,%2,%3}, [%4+16];"
#else
    asm("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4+16];"
#endif
        : "=r"(w0), "=r"(w1), "=r"(w2), "=r"(w3) : "l"(p));
    b[4] = __uint_as_float(w0); b[5] = __uint_as_float(w1); index = w2;
}
// One node (for the lane-pair kernel: each lane of a pair fetches one child of the sibling pair).
__device__ __forceinline__ void load_node(const DevNode<float>* __restrict__ p, float (&b)[6], uint32_t& index) {
    uint32_t a[8];
    ldg256(p, a);
    #pragma unroll
    for (int k = 0; k < 6; ++k) b[k] = __uint_as_float(a[k]);
    index = a[6];
}
__device__ __forceinline__ void load_node(const DevNode<double>* __restrict__ p, double (&b)[6], uint64_t& index) {
    unsigned long long a[4], c[4];
    const unsigned char* q = reinterpret_cast<const unsigned char*>(p);
    ldg256(q, a); ldg256(q + 32, c);
    #pragma unroll
    for (int k = 0; k < 4; ++k) b[k] = __longlong_as_double((long long)a[k]);
    b[4] = __longlong_as_double((long long)c[0]); b[5] = __longlong_as_double((long long)c[1]);
    index = c[2];
}
#if BVH_TRI_PAD
__device__ __forceinline__ void load_tri(const DevTri<float>* __restrict__ p, DevTri<float>& o) {
    uint32_t a[8], b[8];
    ldg256(p, a);
    ldg256(reinterpret_cast<const unsigned char*>(p) + 32, b);
    o.p0[0] = __uint_as_float(a[0]); o.p0[1] = __uint_as_float(a[1]); o.p0[2] = __uint_as_float(a[2]);
    o.e1[0] = __uint_as_float(a[3]); o.e1[1] = __uint_as_float(a[4]); o.e1[2] = __uint_as_float(a[5]);
    o.e2[0] = __uint_as_float(a[6]); o.e2[1] = __uint_as_float(a[7]); o.e2[2] = __uint_as_float(b[0]);
    o.n[0] = __uint_as_float(b[1]); o.n[1] = __uint_as_float(b[2]); o.n[2] = __uint_as_float(b[3]);
}
__device__ __forceinline__ void load_tri(const DevTri<double>* __restrict__ p, DevTri<double>& o) {
    unsigned long long a[4], b[4], c[4];
    const unsigned char* q = reinterpret_cast<const unsigned char*>(p);
    ldg256(q, a); ldg256(q + 32, b); ldg256(q + 64, c);
    o.p0[0] = __longlong_as_double((long long)a[0]); o.p0[1] = __longlong_as_double((long long)a[1]);
    o.p0[2] = __longlong_as_double((long long)a[2]); o.e1[0] = __longlong_as_double((long long)a[3]);
    o.e1[1] = __longlong_as_double((long long)b[0]); o.e1[2] = __longlong_as_double((long long)b[1]);
    o.e2[0] = __longlong_as_double((long long)b[2]); o.e2[1] = __longlong_as_double((long long)b[3]);
    o.e2[2] = __longlong_as_double((long long)c[0]); o.n[0] = __longlong_as_double((long long)c[1]);
    o.n[1] = __longlong_as_double((long long)c[2]); o.n[2] = __longlong_as_double((long long)c[3]);
}
#else
__device__ __forceinline__ void load_tri(const DevTri<float>* __restrict__ p, DevTri<float>& o) {
    const float4* q = reinterpret_cast<const float4*>(p);
    const float4 a = ldg128_tri(q), b = ldg128_tri(q + 1), c = ldg128_tri(q + 2);
    o.p0[0] = a.x; o.p0[1] = a.y; o.p0[2] = a.z; o.e1[0] = a.w;
    o.e1[1] = b.x; o.e1[2] = b.y; o.e2[0] = b.z; o.e2[1] = b.w;
    o.e2[2] = c.x; o.n[0] = c.y; o.n[1] = c.z; o.n[2] = c.w;
}
__device__ __forceinline__ void load_tri(const DevTri<double>* __restrict__ p, DevTri<double>& o) {
    const double2* q = reinterpret_cast<const double2*>(p);
    const double2 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2), d = __ldg(q + 3), e = __ldg(q + 4), f = __ldg(q + 5);
    o.p0[0] = a.x; o.p0[1] = a.y; o.p0[2] = b.x; o.e1[0] = b.y; o.e1[1] = c.x; o.e1[2] = c.y;
    o.e2[0] = d.x; o.e2[1] = d.y; o.e2[2] = e.x; o.n[0] = e.y; o.n[1] = f.x; o.n[2] = f.y;
}
#endif
#else
template <typename T> inline void load_pair(const DevNode<T>* p, NodePair<T>& o) {
    for (int k = 0; k < 6; ++k) { o.lb[k] = p[0].bounds[k]; o.rb[k] = p[1].bounds[k]; }
    o.li = p[0].index; o.ri = p[1].index;
}
template <typename T> inline void load_first_halves(const DevNode<T>* p, NodePair<T>& o) {
    for (int k = 0; k < 4; ++k) { o.lb[k] = p[0].bounds[k]; o.rb[k] = p[1].bounds[k]; }
}
template <typename T> inline void load_second_half(const DevNode<T>* p, T (&b)[6], typename Real<T>::UInt& index) {
    b[4] = p->bounds[4]; b[5] = p->bounds[5]; index = p->index;
}
template <typename T> inline void load_tri(const DevTri<T>* p, DevTri<T>& o) { o = *p; }
#endif

// The value `top` takes when a ray's traversal is over: all ones, a leaf of 15 primitives at the last representable
// position, which no tree has.  Its primitive count is not 0, so the inner-node loops stop on it without a test of their
// own, and the ray's end needs no flag beside `top`.
template <typename U> constexpr U kTraversalDone = (U)~(U)0;

// The next entry of the stack, or kTraversalDone when it is empty.  The device stack keeps kTraversalDone in its bottom
// entry (SmemStack, below), so there the result is the loaded value itself (the compare only keeps the stack
// pointer at the bottom).
template <typename U, typename Stack> BVH_HD U pop_or_done(Stack& stack) {
    U v = kTraversalDone<U>;
    return stack.try_pop(v) ? v : kTraversalDone<U>;
}

// The reference's choice after a sibling pair's test (bvh.h:137-149): the near child becomes `top`, the far one is
// pushed when both are hit (swapped when `swap`), and the stack is popped when both are missed.  Same decisions as the
// reference's nested branches, written as selects: on the device the lanes of a warp take all four outcomes at once,
// and one predicated path costs fewer issue slots than four divergent ones.
template <typename U, typename Stack>
BVH_HD void descend(bool hit_left, bool hit_right, bool swap, U left_index, U right_index, U& top, Stack& stack) {
    const bool both = hit_left && hit_right;
    const bool right_first = both && swap;
    const U near_index = (hit_left && !right_first) ? left_index : right_index;
    const U far_index = right_first ? left_index : right_index;
    if (both) stack.push(far_index);
    top = (hit_left || hit_right) ? near_index : pop_or_done<U>(stack);
}

// One inner step (reference bvh.h:132-150 with the lambda of :167-181): `top` (an inner node) becomes the next node to
// visit, or kTraversalDone when both children were missed and the stack is empty.
template <typename T, bool kAny, bool kRobust, typename Stack>
BVH_HD void inner_step(const DevNode<T>* __restrict__ nodes, const RayCtx<T>& r,
                       typename Real<T>::UInt& top, Stack& stack) {
    using U = typename Real<T>::UInt;
    NodePair<T> pair;
    // Device slot = reference index + 1.  An inner node's count bits are 0, so its first child's byte offset is
    // index_first(top) * sizeof(DevNode<T>) = top * (sizeof(DevNode<T>) >> kPrimCountBits): one multiply-add from `top`.
    const DevNode<T>* p = reinterpret_cast<const DevNode<T>*>(reinterpret_cast<const unsigned char*>(nodes + 1) +
                                                              (size_t)top * (sizeof(DevNode<T>) >> kPrimCountBits));
    T l0, l1, r0, r1;
    if constexpr (sizeof(T) == 4 && !kAny) {
        // node_test of both children, split after the x and y axes: a child whose x/y interval is already empty is
        // missed (node_test_axes), so its second half is neither loaded nor tested, and its index is not used below.
        // Same operations in the same order as node_test, so the same intervals.  On the device the two conditional
        // loads become predicated LDGs: a lane that skips one issues nothing for it.  Measured on the H100 (DESIGN.md
        // §3), this is faster for float closest-hit rays only; any-hit and double-precision rays load whole nodes.
        pair.li = pair.ri = 0;       // (defined on every path: an index loaded on some only lengthens its live range)
        load_first_halves(p, pair);
        l0 = r.tmin; l1 = r.tmax; r0 = r.tmin; r1 = r.tmax;
        node_test_axes<T, kRobust, 0, 2>(pair.lb, r, l0, l1);
        node_test_axes<T, kRobust, 0, 2>(pair.rb, r, r0, r1);
        if (l0 <= l1) { load_second_half(p, pair.lb, pair.li); node_test_axes<T, kRobust, 2, 3>(pair.lb, r, l0, l1); }
        if (r0 <= r1) { load_second_half(p + 1, pair.rb, pair.ri); node_test_axes<T, kRobust, 2, 3>(pair.rb, r, r0, r1); }
    } else {
        load_pair(p, pair);
        node_test<T, kRobust>(pair.lb, r, l0, l1);
        node_test<T, kRobust>(pair.rb, r, r0, r1);
    }
    // ties go left first (`>` at bvh.h:180)
    descend<U>(l0 <= l1, r0 <= r1, !kAny && l0 > r0, pair.li, pair.ri, top, stack);
}

// node_fn(left, right, left_index) when it takes the left child's reference index, node_fn(left, right) otherwise.
template <typename NodeFn, typename Node, typename U>
BVH_HD decltype(auto) node_test(NodeFn& node_fn, const Node& left, const Node& right, U left_index) {
    if constexpr (std::is_invocable_v<NodeFn&, const Node&, const Node&, size_t>)
        return node_fn(left, right, static_cast<size_t>(left_index));
    else
        return node_fn(left, right);
}

// One step of traverse_nodes: the sibling pair below `top` (an inner node) in one load_pair, register copies of the two
// children handed to the caller's node test, and the reference's decision (descend): `top` becomes the next node to
// visit, or kTraversalDone when both children were missed and the stack is empty.  DeviceView::query's kernel takes the
// same step.
template <typename T, typename Stack, typename NodeFn>
BVH_HD void node_step(const DevNode<T>* __restrict__ nodes, typename Real<T>::UInt& top, Stack& stack, NodeFn& node_fn) {
    using U = typename Real<T>::UInt;
    // device slot = reference index + 1, the same offset arithmetic as inner_step
    const DevNode<T>* p = reinterpret_cast<const DevNode<T>*>(reinterpret_cast<const unsigned char*>(nodes + 1) +
                                                              (size_t)top * (sizeof(DevNode<T>) >> kPrimCountBits));
    NodePair<T> pair;
    load_pair(p, pair);
    DevNode<T> left, right;
    for (int k = 0; k < 6; ++k) { left.bounds[k] = pair.lb[k]; right.bounds[k] = pair.rb[k]; }
    left.index = pair.li; right.index = pair.ri;
    left.pad = right.pad = 0;
    const auto [hit_left, hit_right, should_swap] = node_test(node_fn, static_cast<const DevNode<T>&>(left),
                                                              static_cast<const DevNode<T>&>(right), index_first(top));
    descend<U>(static_cast<bool>(hit_left), static_cast<bool>(hit_right), static_cast<bool>(should_swap),
               pair.li, pair.ri, top, stack);
}

// Bvh::traverse_top_down with the caller's node test (reference bvh.h:124-157), for queries other than rays: box
// overlap, point location, nearest-neighbour searches.  The traversal starts at the node index `start` with an empty
// stack.
//   node_fn(const DevNode<T>& left, const DevNode<T>& right[, size_t left_index])  called once per inner node reached,
//                                 with register copies of its two children and, when it takes a third argument, the
//                                 reference index of the left child (the right one is left_index + 1); returns anything
//                                 that unpacks with a structured binding into (hit_left, hit_right, should_swap), each
//                                 convertible to bool.  should_swap takes effect when both children are hit, whatever
//                                 kAny is.
//   leaf_fn(begin, end) -> bool   called on every leaf reached, with its BVH-order primitive range; with kAny a true
//                                 return ends the traversal.  A leaf `start` is handed to leaf_fn without a node test.
//   stack                         push(U) and try_pop(U&) (false when empty); it holds at most depth + 1 entries.
// Each sibling pair is one load_pair: the node test is the caller's, so there is no split of the node load here.
template <typename T, bool kAny, typename Stack, typename LeafFn, typename NodeFn>
BVH_HD void traverse_nodes(const DevNode<T>* __restrict__ nodes, typename Real<T>::UInt start, Stack& stack,
                           LeafFn&& leaf_fn, NodeFn&& node_fn) {
    using U = typename Real<T>::UInt;
    U top = start;
    for (;;) {
        while (index_count(top) == 0) node_step<T>(nodes, top, stack, node_fn);
        if (top == kTraversalDone<U>) break;
        const U first = index_first(top);
        const bool was_hit = static_cast<bool>(leaf_fn(first, first + (U)index_count(top)));
        if (kAny && was_hit) break;                             // bvh.h:153-155
        top = pop_or_done<U>(stack);
    }
}

// The triangles [first, first + count) of a leaf (benchmark.cpp:281-292).  stats (nullable): [1] leaves, [2] triangle tests.
// accept: tri_test's filter, called with the slot, t, u and v of every candidate that would become the closest hit.  With a
// filter of the caller's the loop is not unrolled: one copy of the caller's code, and one triangle's registers live at a
// time (DeviceView::trace_triangles' float kernel then fits its 56 registers without spills; DESIGN.md §6).
template <typename T, typename Accept = AcceptAll>
BVH_HD void leaf_range(const DevTri<T>* __restrict__ tris, const uint32_t* __restrict__ prim_ids, bool lowest_id,
                       uint32_t first, uint32_t count, RayCtx<T>& r, HitState<T>& hit, uint32_t* stats, Accept&& accept = {}) {
    if (stats) { stats[1] += 1; stats[2] += count; }
    if constexpr (std::is_same_v<std::decay_t<Accept>, AcceptAll>) {
        for (uint32_t i = first; i < first + count; ++i) {
            DevTri<T> tri;
            load_tri(tris + i, tri);
            tri_test<T>(tri, i, prim_ids, lowest_id, r, hit);
        }
    } else {
#if defined(__CUDA_ARCH__)
        #pragma unroll 1
#endif
        for (uint32_t i = first; i < first + count; ++i) {
            DevTri<T> tri;
            load_tri(tris + i, tri);
            tri_test<T>(tri, i, prim_ids, lowest_id, r, hit, accept);
        }
    }
}

// The hit record of a finished ray (bvh_hit3f / bvh_hit3d): its closest hit's original id, t, u and v; a miss reports
// id = all ones (BVH_INVALID_PRIM_ID), t = the ray's tmax, u = v = 0.
template <typename T>
BVH_HD DevHit<T> make_record(const HitState<T>& h, T tmax, const uint32_t* __restrict__ prim_ids) {
    DevHit<T> rec;
    const bool was_hit = h.slot != kInvalidId;
    rec.prim_id = was_hit ? (decltype(rec.prim_id))prim_ids[h.slot] : (decltype(rec.prim_id))~(decltype(rec.prim_id))0;
    rec.t = was_hit ? h.t : tmax;
    rec.u = was_hit ? h.u : (T)0;
    rec.v = was_hit ? h.v : (T)0;
    return rec;
}

// Leaf processing for the leaf index `top`.
template <typename T>
BVH_HD void leaf_step(const DevTri<T>* __restrict__ tris, const uint32_t* __restrict__ prim_ids, bool lowest_id,
                      typename Real<T>::UInt top, RayCtx<T>& r, HitState<T>& hit, uint32_t* stats) {
    leaf_range<T>(tris, prim_ids, lowest_id, (uint32_t)index_first(top), index_count(top), r, hit, stats);
}

// The reference's Bvh::traverse_top_down with the box test of Bvh::intersect (bvh.h:124-182), generic in the leaf and the
// stack, for one ray whose prologue has been run.  The traversal starts at the node index `start` (a node's packed index:
// first id << 4 | primitive count) with an empty stack.
//   leaf_fn(begin, end) -> bool   called on every leaf reached, with its BVH-order primitive range, in the reference's
//                                 order.  It may shrink r.tmax (or change r.tmin); the next box test reads them.  With kAny
//                                 a true return ends the traversal.
//   inner_fn(first_child)         called once per inner step, before the step's box tests, with the reference index of the
//                                 left child of the inner node being expanded (the right child is first_child + 1).
//   stack                         push(U) and try_pop(U&) (false when empty); it holds at most depth + 1 entries.
// A ray whose interval is a NaN misses every box in the reference (each comparison with tmin / tmax fails, node.h:110-115),
// but traverse_top_down tests no box before its first pop: a leaf `start` is still handed to leaf_fn, and an inner one
// costs one inner step that finds both children missed.  The device's min / max accumulation does not keep a NaN
// accumulator (core.cuh acc_max), so such rays go through the branch below, which draws the stacked entries without box
// tests, exactly what the reference does with them.  The interval is checked again after every leaf call.
template <typename T, bool kAny, bool kRobust, typename Stack, typename LeafFn, typename InnerFn>
BVH_HD void traverse_top_down(const DevNode<T>* __restrict__ nodes, RayCtx<T>& r, typename Real<T>::UInt start,
                              Stack& stack, LeafFn&& leaf_fn, InnerFn&& inner_fn) {
    using U = typename Real<T>::UInt;
    U top = start;
    for (;;) {
        if (!ray_interval_is_nan(r)) {
            while (index_count(top) == 0) {
                inner_fn(index_first(top));
                inner_step<T, kAny, kRobust>(nodes, r, top, stack);
            }
        } else {
            while (index_count(top) == 0) {
                inner_fn(index_first(top));
                top = pop_or_done<U>(stack);                    // both children missed
            }
        }
        if (top == kTraversalDone<U>) break;
        const U first = index_first(top);
        const bool was_hit = leaf_fn(first, first + (U)index_count(top));
        if (kAny && was_hit) break;                             // bvh.h:153-155
        top = pop_or_done<U>(stack);
    }
}

// Whole traversal for one ray with the triangle leaf.  stats (nullable): {inner steps, leaves, triangle tests}, the same
// three counters the reference exposes through its InnerFn hook (bvh.h:168, benchmark.cpp:282-296).
template <typename T, bool kAny, bool kRobust, typename Stack>
BVH_HD void traverse_ray(const DevNode<T>* __restrict__ nodes, const DevTri<T>* __restrict__ tris,
                         const uint32_t* __restrict__ prim_ids, bool lowest_id, typename Real<T>::UInt root_index,
                         RayCtx<T>& r, HitState<T>& hit, Stack& stack, uint32_t* stats) {
    using U = typename Real<T>::UInt;
    if (ray_interval_is_nan(r)) return;                         // no triangle can be hit (tri.h:69); counters stay 0
    traverse_top_down<T, kAny, kRobust>(
        nodes, r, root_index, stack,                            // get_root().index, bvh.h:54
        [&](U begin, U end) {
            leaf_range<T>(tris, prim_ids, lowest_id, (uint32_t)begin, (uint32_t)(end - begin), r, hit, stats);
            return hit.slot != kInvalidId;
        },
        [&](U) { if (stats) stats[0] += 1; });
}

// A per-thread stack of `Capacity` entries in registers / local memory (the reference's SmallStack, stack.h).  It holds
// at most depth + 1 entries during a traversal; nothing checks the capacity on the device.
template <typename U, unsigned Capacity> struct ArrayStack {
    static constexpr unsigned capacity = Capacity;
    U elems[Capacity];
    unsigned size = 0;
    BVH_HD void push(U v) { elems[size++] = v; }
    BVH_HD bool try_pop(U& out) {
        if (size == 0) return false;
        out = elems[--size];
        return true;
    }
    BVH_HD bool empty() const { return size == 0; }
};

#if defined(__CUDACC__)
// Shared-memory stack: entry k of thread t lives at base[k * stride + t] (bank = t mod 32).  The stack pointer is kept
// as ONE 32-bit shared-memory address (a push / pop is a store / load plus one add — indexing base[sp * stride] made the
// compiler re-derive the thread's base address from S2R in every push and pop of the inner loop), and entry 0 holds a
// sentinel no node index can equal (all ones: a leaf of 15 primitives at the last representable position), so that
// try_pop() needs no comparison with the bottom address either.  Callers size the array as depth + 2 entries.
template <typename U> struct SmemStack {
    uint32_t top;                                            // shared-window address of the next free entry
    uint32_t step;                                           // bytes between entries
    U* base;
    static constexpr U kSentinel = kTraversalDone<U>;
    __device__ __forceinline__ SmemStack(U* base_, uint32_t stride, uint32_t) : step(stride * (uint32_t)sizeof(U)), base(base_) {
        clear();
        top -= step;
        push(kSentinel);                                     // (through the same volatile asm as every other access)
    }
    __device__ __forceinline__ void clear() { top = (uint32_t)__cvta_generic_to_shared(base) + step; }
    __device__ __forceinline__ void push(U v) {
        // (volatile keeps the stack's own loads and stores in program order; no "memory" clobber: nothing else aliases the stack)
#ifdef BVH_STACK_CLOBBER             // A/B measurements only
        if constexpr (sizeof(U) == 4) asm volatile("st.shared.b32 [%0], %1;" :: "r"(top), "r"((uint32_t)v) : "memory");
        else asm volatile("st.shared.b64 [%0], %1;" :: "r"(top), "l"((unsigned long long)v) : "memory");
#else
        if constexpr (sizeof(U) == 4) asm volatile("st.shared.b32 [%0], %1;" :: "r"(top), "r"((uint32_t)v));
        else asm volatile("st.shared.b64 [%0], %1;" :: "r"(top), "l"((unsigned long long)v));
#endif
        top += step;
    }
    __device__ __forceinline__ U pop() {
        top -= step;
#ifdef BVH_STACK_CLOBBER
        if constexpr (sizeof(U) == 4) { uint32_t v; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(top) : "memory"); return (U)v; }
        else { unsigned long long v; asm volatile("ld.shared.b64 %0, [%1];" : "=l"(v) : "r"(top) : "memory"); return (U)v; }
#else
        if constexpr (sizeof(U) == 4) { uint32_t v; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(top)); return (U)v; }
        else { unsigned long long v; asm volatile("ld.shared.b64 %0, [%1];" : "=l"(v) : "r"(top)); return (U)v; }
#endif
    }
    // pops into `out`; false (and the stack stays empty) when there was nothing to pop
    __device__ __forceinline__ bool try_pop(U& out) {
        const U v = pop();
        if (v == kSentinel) { top += step; return false; }
        out = v;
        return true;
    }
    __device__ __forceinline__ bool empty() const { return top == (uint32_t)__cvta_generic_to_shared(base) + step; }
};
#endif

} // namespace bvhb200
