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
// the device traversal API (include/bvh/v2/cuda/intersect.cuh).
#pragma once

#include "core.cuh"

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
// sm_100 has 256-bit global loads (SASS LDG.E.256): a node is ONE load, a sibling pair two, from one
// naturally aligned 64-byte (float) / 128-byte (double) block, through the read-only path.  Halving the
// number of load instructions matters because with divergent rays every load costs one L1 tag lookup per
// distinct line touched by the warp (profiles/: the traversal is L1-tag bound, not DRAM bound).
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

// One inner step (reference bvh.h:132-150 with the lambda of :167-181): `top` (an inner node) becomes the next node to
// visit, or kTraversalDone when both children were missed and the stack is empty.
template <typename T, bool kAny, bool kRobust, typename Stack>
BVH_HD void inner_step(const DevNode<T>* __restrict__ nodes, const RayCtx<T>& r,
                       typename Real<T>::UInt& top, Stack& stack) {
    using U = typename Real<T>::UInt;
    NodePair<T> pair;
    // Device slot = reference index + 1.  An inner node's count bits are 0, so its first child's byte offset is
    // index_first(top) * sizeof(DevNode<T>) = top * (sizeof(DevNode<T>) >> kPrimCountBits): one multiply-add from `top`.
    load_pair(reinterpret_cast<const DevNode<T>*>(reinterpret_cast<const unsigned char*>(nodes + 1) +
                                                  (size_t)top * (sizeof(DevNode<T>) >> kPrimCountBits)), pair);
    T l0, l1, r0, r1;
    node_test<T, kRobust>(pair.lb, r, l0, l1);
    node_test<T, kRobust>(pair.rb, r, r0, r1);
    const bool hit_left = l0 <= l1, hit_right = r0 <= r1;
    // Same decisions as the reference's nested branches (bvh.h:167-181), written as selects: on the device the lanes of a
    // warp take all four outcomes at once, and one predicated path costs fewer issue slots than four divergent ones.
    const bool both = hit_left && hit_right;
    const bool right_first = !kAny && both && l0 > r0;            // ties go left first (`>` at bvh.h:180)
    const U near_index = (hit_left && !right_first) ? pair.li : pair.ri;
    const U far_index = right_first ? pair.li : pair.ri;
    if (both) stack.push(far_index);
    top = (hit_left || hit_right) ? near_index : pop_or_done<U>(stack);
}

// The triangles [first, first + count) of a leaf (benchmark.cpp:281-292).  stats (nullable): [1] leaves, [2] triangle tests.
template <typename T>
BVH_HD void leaf_range(const DevTri<T>* __restrict__ tris, const uint32_t* __restrict__ prim_ids, bool lowest_id,
                       uint32_t first, uint32_t count, RayCtx<T>& r, HitState<T>& hit, uint32_t* stats) {
    if (stats) { stats[1] += 1; stats[2] += count; }
    for (uint32_t i = first; i < first + count; ++i) {
        DevTri<T> tri;
        load_tri(tris + i, tri);
        tri_test<T>(tri, i, prim_ids, lowest_id, r, hit);
    }
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
