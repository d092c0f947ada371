// bvh_b200/csrc/treelet_warp.cuh — SAH rebuild of the bottom of the LBVH ("treelets"), one warp per treelet, the
// working set in REGISTERS: the second build pass of DefaultBuilder::Quality Medium and High (Low keeps the LBVH).
//
// Why: measured (DESIGN.md §4), the 11-23 % more traversal steps the LBVH needs compared with the reference's SAH
// trees come from the bottom levels: keeping the LBVH above and rebuilding every maximal subtree of at most 64
// primitives with the reference's sweep-SAH rule recovers most of the reference's step counts.
//
// What: every maximal LBVH subtree of 3..64 primitives (listed by the bottom-up pass itself, build_core.cuh
// merge_into_parent) is rebuilt top-down with the greedy rule of the reference's SweepSahBuilder /
// TopDownSahBuilder (sweep_sah_builder.h:57-139, top_down_sah_builder.h:74-131): primitives sorted once along each
// axis, per node the split minimising area(L)*|L| + area(R)*|R| over the three axes and all positions, leaf when no
// split beats area*(count - 1) and count <= max_leaf_size, median split on the largest axis otherwise, stable
// partition of the other two orders, larger-area child first (SATO).  All nodes of one LEVEL of the treelet are
// processed together: in each of the three orders a node's primitives occupy one contiguous segment of positions
// (the same segment in all three), and prefix / suffix boxes and the cheapest split of every segment are segmented
// scans over the 64 positions.  The subtree is written into the node slots the LBVH subtree owned (pairs l .. r-1
// of the sorted range [l, r]; an inner node takes the pair of its split boundary, as in the LBVH numbering), the
// primitives are re-ordered inside [l, r] only, and the subtree's box is unchanged, so nothing above it moves.
//
// How: a lane owns positions 2*lane and 2*lane+1.  Boxes, costs and segment bounds of its positions live in
// registers; a segmented scan is a combine of the lane's two positions, five Kogge-Stone steps over the lane
// aggregates with warp shuffles, and the carry-in; the stable partition ranks a position with two ballots and
// population counts.  Shared memory (3.3 KB per warp for float) only holds what is indexed by PRIMITIVE or read
// from another lane's position: the primitive boxes, the three orders, per-head decisions.  (The first version of
// this pass kept every per-position array in shared memory and ran ~600 __syncwarp-separated phases per treelet;
// this one needs about a tenth of the instructions.)
//
// The algorithm is written ONCE against a lane-execution policy: on the device a per-lane variable is a register
// and `each` runs the body for the calling lane; in the host emulation (tests/host_emul.cpp) a per-lane variable
// is an array of 32 and `each` loops over the lanes, shuffles copy between array elements — the same source, the
// same arithmetic (Real<T> ops, no contraction) and the same combination order, hence the same tree bit for bit.
// Discipline that makes the two equivalent: shared memory written in one `each` block is only read after sync().
#pragma once

#include "build_core.cuh"

namespace bvhb200 {

constexpr int kTreeletMaxPrims = 64;
template <typename T> struct TreeletCfg { static constexpr int kMaxPrims = kTreeletMaxPrims; };

// A box in registers: [minx,maxx,miny,maxy,minz,maxz].
template <typename T> struct Box6 { T v[6]; };
template <typename T> BVH_HD Box6<T> box_join(const Box6<T>& a, const Box6<T>& b) {      // a.extend(b), bbox.h:23-27
    Box6<T> o;
    for (int k = 0; k < 6; k += 2) { o.v[k] = robust_min(a.v[k], b.v[k]); o.v[k + 1] = robust_max(a.v[k + 1], b.v[k + 1]); }
    return o;
}
template <typename T> BVH_HD T box_half_area(const Box6<T>& b) {
    const T mn[3] = { b.v[0], b.v[2], b.v[4] }, mx[3] = { b.v[1], b.v[3], b.v[5] };
    return half_area(mn, mx);
}

// loops over a lane's two positions / the three axes must be unrolled on the device (their indices select registers)
#if defined(__CUDA_ARCH__)
#define BVH_UNROLL _Pragma("unroll")
#else
#define BVH_UNROLL
#endif

BVH_HD uint32_t treelet_popcount(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return (uint32_t)__popc(x);
#else
    return (uint32_t)__builtin_popcount(x);
#endif
}

// ---- lane-execution policies ------------------------------------------------------------------------------
#if defined(__CUDACC__)
template <typename V> __device__ __forceinline__ V lane_shfl_up(const V& v, unsigned d) { return __shfl_up_sync(0xFFFFFFFFu, v, d); }
template <typename V> __device__ __forceinline__ V lane_shfl_down(const V& v, unsigned d) { return __shfl_down_sync(0xFFFFFFFFu, v, d); }
template <typename V> __device__ __forceinline__ V lane_shfl_idx(const V& v, unsigned i) { return __shfl_sync(0xFFFFFFFFu, v, i); }
template <typename T> __device__ __forceinline__ Box6<T> lane_shfl_up(const Box6<T>& v, unsigned d) {
    Box6<T> o;
    #pragma unroll
    for (int k = 0; k < 6; ++k) o.v[k] = __shfl_up_sync(0xFFFFFFFFu, v.v[k], d);
    return o;
}
template <typename T> __device__ __forceinline__ Box6<T> lane_shfl_down(const Box6<T>& v, unsigned d) {
    Box6<T> o;
    #pragma unroll
    for (int k = 0; k < 6; ++k) o.v[k] = __shfl_down_sync(0xFFFFFFFFu, v.v[k], d);
    return o;
}
struct DeviceLanes {
    template <typename V> using Var = V;
    template <typename F> static __device__ __forceinline__ void each(F f) { f(threadIdx.x & 31u); }
    template <typename V> static __device__ __forceinline__ V& at(V& v, unsigned) { return v; }
    template <typename V> static __device__ __forceinline__ const V& at(const V& v, unsigned) { return v; }
    // dst(lane) = src(lane - d) / src(lane + d); lanes without a source keep their own value
    template <typename V> static __device__ __forceinline__ void from_below(V& dst, const V& src, unsigned d) { dst = lane_shfl_up(src, d); }
    template <typename V> static __device__ __forceinline__ void from_above(V& dst, const V& src, unsigned d) { dst = lane_shfl_down(src, d); }
    template <typename V> static __device__ __forceinline__ void from_lane(V& dst, const V& src, unsigned src_lane) { dst = lane_shfl_idx(src, src_lane); }
    static __device__ __forceinline__ uint32_t ballot(bool pred) { return __ballot_sync(0xFFFFFFFFu, pred); }
    static __device__ __forceinline__ uint32_t max_over_lanes(uint32_t v) { return __reduce_max_sync(0xFFFFFFFFu, v); }
    static __device__ __forceinline__ void sync() { __syncwarp(); }
    static __device__ __forceinline__ void atomic_max(uint32_t* p, uint32_t v) { atomicMax(p, v); }
};
#endif

template <bool kReversed> struct HostLanesT {
    template <typename V> struct Var { V lane[32]; };
    template <typename F> static void each(F f) {
        if (kReversed) for (unsigned l = 32; l-- > 0;) f(l);
        else for (unsigned l = 0; l < 32; ++l) f(l);
    }
    template <typename V> static V& at(Var<V>& v, unsigned l) { return v.lane[l]; }
    template <typename V> static const V& at(const Var<V>& v, unsigned l) { return v.lane[l]; }
    template <typename V> static void from_below(Var<V>& dst, const Var<V>& src, unsigned d) {
        const Var<V> t = src;
        for (unsigned l = 0; l < 32; ++l) dst.lane[l] = t.lane[l >= d ? l - d : l];
    }
    template <typename V> static void from_above(Var<V>& dst, const Var<V>& src, unsigned d) {
        const Var<V> t = src;
        for (unsigned l = 0; l < 32; ++l) dst.lane[l] = t.lane[l + d < 32 ? l + d : l];
    }
    template <typename V> static void from_lane(Var<V>& dst, const Var<V>& src, unsigned src_lane) {
        const V t = src.lane[src_lane & 31u];
        for (unsigned l = 0; l < 32; ++l) dst.lane[l] = t;
    }
    static uint32_t ballot(const Var<bool>& pred) {
        uint32_t m = 0;
        for (unsigned l = 0; l < 32; ++l) m |= pred.lane[l] ? (1u << l) : 0u;
        return m;
    }
    static uint32_t max_over_lanes(const Var<uint32_t>& v) {
        uint32_t m = 0;
        for (unsigned l = 0; l < 32; ++l) m = v.lane[l] > m ? v.lane[l] : m;
        return m;
    }
    static void sync() {}
    static void atomic_max(uint32_t* p, uint32_t v) { if (v > *p) *p = v; }
};
using HostLanes = HostLanesT<false>;
using HostLanesReversed = HostLanesT<true>;          // lanes in descending order: exposes a shared-memory hazard as a different tree

// ---- one warp's shared memory ---------------------------------------------------------------------------------
template <typename T> struct TreeletShared {
    T box[6][kTreeletMaxPrims];                  // per PRIMITIVE (local index): minx,maxx,miny,maxy,minz,maxz
    T area_pre[kTreeletMaxPrims];                // per POSITION, current axis: half area of [segment begin, pos] ...
    T area_suf[kTreeletMaxPrims];                // ... and of [pos, segment end)
    uint32_t old_ids[kTreeletMaxPrims];          // prim_ids[l + i] before the rebuild
    uint32_t dst_slot[kTreeletMaxPrims];         // per HEAD position: device slot the segment's node record goes to
    uint32_t decision[kTreeletMaxPrims];         // per HEAD position, this level: bit 0 split, bits 1-2 axis, bits 8-15 first position of the right part
    uint8_t order[2][3][kTreeletMaxPrims];       // local primitive indices sorted along each axis, segment by segment (ping-pong)
    uint8_t side[kTreeletMaxPrims];              // per PRIMITIVE: 1 = goes to the left part
    uint8_t depth[kTreeletMaxPrims];             // per HEAD position: depth of the segment's node inside the treelet
};
static_assert(sizeof(TreeletShared<float>) <= 4096 && sizeof(TreeletShared<double>) <= 8192, "one warp's slice of shared memory");

// Monotone map of a scalar to an unsigned integer (negative values reversed below the positive ones): a total
// order even when a centre is a NaN, so the rank sort below always yields a permutation.
template <typename T> BVH_HD typename Real<T>::UInt treelet_sort_key(T x) {
    using U = typename Real<T>::UInt;
    const U bits = Real<T>::bits(x), sign = (U)1 << (8 * sizeof(U) - 1);
    return (bits & sign) ? (U)~bits : (U)(bits | sign);
}
template <typename T> BVH_HD T treelet_inf() { return Real<T>::from_bits(sizeof(T) == 4 ? (typename Real<T>::UInt)0x7F800000u : (typename Real<T>::UInt)0x7FF0000000000000ull); }

// Rebuilds one treelet.  `leaf_src`: vertices (n x 9, leaf_mode 0) or boxes (n x 6, leaf_mode 1); `centre_src`:
// vertices or centres (n x 3), indexed by ORIGINAL primitive id.  `tris` (leaf_mode 0 only) receives the
// BVH-order triangle records of the range.  info[2] collects by how much a treelet got deeper than the subtree
// it replaces (the traversal stack is sized from info[0] + info[2]); alive[] (nullable) receives the liveness of
// the pairs l .. r-1 (build_core.cuh BuildParams::alive).
template <typename T, typename X>
BVH_HD void treelet_rebuild(TreeletShared<T>& w, const Treelet& t, DevNode<T>* __restrict__ nodes,
                            uint32_t* __restrict__ prim_ids, DevTri<T>* __restrict__ tris,
                            const T* __restrict__ leaf_src, const T* __restrict__ centre_src, int leaf_mode,
                            uint32_t min_leaf, uint32_t max_leaf, uint32_t* __restrict__ info, uint32_t lbvh_depth,
                            uint32_t* __restrict__ alive) {
    using R = Real<T>;
    using U = typename R::UInt;
    const uint32_t n = t.r - t.l + 1, l = t.l;
    const T inf = treelet_inf<T>();
    // depth of the subtree being replaced (its root record still carries it; the tree's root record does not)
    const uint32_t old_depth = t.slot == 1 ? lbvh_depth : AuxPack<T>::depth(nodes[t.slot].pad);

    // Per-lane state: index j = 0 / 1 is the lane's position 2*lane + j.
    typename X::template Var<uint32_t> seg_b[2], seg_e[2];        // the position's segment [seg_b, seg_e); dead positions: [p, p+1)
    typename X::template Var<bool> live[2];                       // the position belongs to an undecided segment
    typename X::template Var<U> key[3][2];                        // sort keys of PRIMITIVE 2*lane + j (set-up only)

    // ---- load the primitives: boxes into shared memory, sort keys into registers ----
    X::each([&] (unsigned lane) {
        BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
            const uint32_t i = 2 * lane + j;
            for (int a = 0; a < 3; ++a) X::at(key[a][j], lane) = ~(U)0;
            X::at(seg_b[j], lane) = i; X::at(seg_e[j], lane) = i + 1; X::at(live[j], lane) = false;
            if (i >= n) continue;
            const uint32_t id = prim_ids[l + i];
            w.old_ids[i] = id;
            T bmin[3], bmax[3], c[3];
            if (leaf_mode == 0) {
                T v[9];
                for (int k = 0; k < 9; ++k) v[k] = leaf_src[9 * (size_t)id + k];
                tri_bounds_center(v, bmin, bmax, c);
            } else {
                for (int k = 0; k < 3; ++k) {
                    bmin[k] = leaf_src[6 * (size_t)id + k]; bmax[k] = leaf_src[6 * (size_t)id + 3 + k];
                    c[k] = centre_src[3 * (size_t)id + k];
                }
            }
            for (int k = 0; k < 3; ++k) { w.box[2 * k][i] = bmin[k]; w.box[2 * k + 1][i] = bmax[k]; X::at(key[k][j], lane) = treelet_sort_key(c[k]); }
            X::at(seg_b[j], lane) = 0; X::at(seg_e[j], lane) = n; X::at(live[j], lane) = true;
            if (alive && i + 1 < n) alive[l + i] = 0u;           // the subtree's pairs: the splits below mark the ones they use
            if (i == 0) { w.dst_slot[0] = t.slot; w.depth[0] = 0; }
        }
    });
    // ---- sort once along each axis: rank of a primitive = number of primitives before it in (centre, index) order ----
    {
        typename X::template Var<uint32_t> rank[3][2];
        X::each([&] (unsigned lane) { for (int a = 0; a < 3; ++a) for (int j = 0; j < 2; ++j) X::at(rank[a][j], lane) = 0; });
        for (uint32_t other_lane = 0; 2 * other_lane < n; ++other_lane) {
            BVH_UNROLL
            for (int oj = 0; oj < 2; ++oj) {                      // primitive `other` = 2 * other_lane + oj (keys of i >= n are all ones: never smaller)
                const uint32_t other = 2 * other_lane + oj;
                typename X::template Var<U> ko[3];
                BVH_UNROLL
                for (int a = 0; a < 3; ++a) X::from_lane(ko[a], key[a][oj], other_lane);
                X::each([&] (unsigned lane) {
                    BVH_UNROLL
                    for (int a = 0; a < 3; ++a) {
                        BVH_UNROLL
                        BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
                            const U mine = X::at(key[a][j], lane), theirs = X::at(ko[a], lane);
                            X::at(rank[a][j], lane) += (theirs < mine || (theirs == mine && other < 2 * lane + j)) ? 1u : 0u;
                        }
                    }
                });
            }
        }
        X::each([&] (unsigned lane) {
            BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
                const uint32_t i = 2 * lane + j;
                if (i < n) for (int a = 0; a < 3; ++a) w.order[0][a][X::at(rank[a][j], lane)] = (uint8_t)i;
            }
        });
        X::sync();
    }

    uint32_t cur = 0;                                             // which half of the order ping-pong is current (warp-uniform)
    uint32_t treelet_depth = 0;                                   // warp-uniform
    uint32_t reach = n;                                           // warp-uniform: length of the longest live segment
    typename X::template Var<bool> flag;
    X::each([&] (unsigned lane) { X::at(flag, lane) = X::at(live[0], lane) || X::at(live[1], lane); });

    // ---- level by level (a tree over n primitives has fewer than n levels: the bound turns a logic error into a
    //      wrong tree the tests catch instead of a warp that never returns) ----
    for (uint32_t level = 0; level < n && X::ballot(flag) != 0u; ++level) {
        // per HEAD position (meaningful where the position is a live head)
        typename X::template Var<Box6<T>> node_box[2];
        typename X::template Var<T> leaf_cost[2], best_cost[2], best_larea[2], best_rarea[2];
        typename X::template Var<uint32_t> best_pos[2], best_axis[2];

        for (uint32_t a = 0; a < 3; ++a) {
            typename X::template Var<Box6<T>> own[2], pre[2], suf[2], agg, got;
            // ---- the position's primitive box; combine of the lane's two positions ----
            X::each([&] (unsigned lane) {
                BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
                    const uint32_t p = 2 * lane + j;
                    Box6<T> b;
                    if (p < n) { const uint32_t prim = w.order[cur][a][p]; for (int k = 0; k < 6; ++k) b.v[k] = w.box[k][prim]; }
                    else for (int k = 0; k < 6; ++k) b.v[k] = (T)0;
                    X::at(own[j], lane) = b;
                }
                const uint32_t p0 = 2 * lane;
                // forward: does position p1's segment reach back to p0?   backward: does p0's segment reach p1?
                X::at(pre[0], lane) = X::at(own[0], lane);
                X::at(pre[1], lane) = X::at(seg_b[1], lane) <= p0 ? box_join(X::at(own[1], lane), X::at(own[0], lane)) : X::at(own[1], lane);
                X::at(suf[1], lane) = X::at(own[1], lane);
                X::at(suf[0], lane) = X::at(seg_e[0], lane) > p0 + 1 ? box_join(X::at(own[0], lane), X::at(own[1], lane)) : X::at(own[0], lane);
            });
            // ---- forward: Kogge-Stone over the lane aggregates (the box ending at the lane's second position) ----
            X::each([&] (unsigned lane) { X::at(agg, lane) = X::at(pre[1], lane); });
            for (unsigned d = 1; d < 32 && 2 * d < reach; d <<= 1) {     // (a step with 2d >= reach joins nothing)
                X::from_below(got, agg, d);
                X::each([&] (unsigned lane) {
                    // lane - d's second position, 2*(lane-d)+1, lies in my second position's segment
                    if (lane >= d && X::at(seg_b[1], lane) <= 2 * (lane - d) + 1) X::at(agg, lane) = box_join(X::at(agg, lane), X::at(got, lane));
                });
            }
            X::from_below(got, agg, 1);
            X::each([&] (unsigned lane) {
                const uint32_t p0 = 2 * lane;
                if (lane >= 1 && X::at(seg_b[0], lane) <= p0 - 1) {      // the previous lane's positions continue into mine
                    X::at(pre[0], lane) = box_join(X::at(pre[0], lane), X::at(got, lane));
                    if (X::at(seg_b[1], lane) <= p0 - 1) X::at(pre[1], lane) = box_join(X::at(pre[1], lane), X::at(got, lane));
                }
            });
            // ---- backward: aggregates = the box starting at the lane's first position ----
            X::each([&] (unsigned lane) { X::at(agg, lane) = X::at(suf[0], lane); });
            for (unsigned d = 1; d < 32 && 2 * d < reach; d <<= 1) {     // (a step with 2d >= reach joins nothing)
                X::from_above(got, agg, d);
                X::each([&] (unsigned lane) {
                    // lane + d's first position, 2*(lane+d), lies in my first position's segment
                    if (lane + d < 32 && X::at(seg_e[0], lane) > 2 * (lane + d)) X::at(agg, lane) = box_join(X::at(agg, lane), X::at(got, lane));
                });
            }
            X::from_above(got, agg, 1);
            typename X::template Var<T> right_cost[2], next_right_cost, cand_cost[2];
            typename X::template Var<uint32_t> cand_pos[2];
            X::each([&] (unsigned lane) {
                const uint32_t p1 = 2 * lane + 1;
                if (lane + 1 < 32 && X::at(seg_e[1], lane) > p1 + 1) {   // the next lane's positions continue mine
                    X::at(suf[1], lane) = box_join(X::at(suf[1], lane), X::at(got, lane));
                    if (X::at(seg_e[0], lane) > p1 + 1) X::at(suf[0], lane) = box_join(X::at(suf[0], lane), X::at(got, lane));
                }
                BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
                    const uint32_t p = 2 * lane + j;
                    const T as = box_half_area(X::at(suf[j], lane)), ap = box_half_area(X::at(pre[j], lane));
                    if (p < n) { w.area_pre[p] = ap; w.area_suf[p] = as; }
                    // cost of [pos, segment end) as a leaf: get_leaf_cost, split_heuristic.h:30-33
                    X::at(right_cost[j], lane) = R::mul(as, (T)(X::at(seg_e[j], lane) - p));
                    if (a == 0 && X::at(live[j], lane) && X::at(seg_b[j], lane) == p) {      // a live head: the suffix box is the node's box
                        X::at(node_box[j], lane) = X::at(suf[j], lane);
                        const uint32_t se = X::at(seg_e[j], lane);
                        const T lc = R::mul(as, (T)(se - p - 1));        // get_non_split_cost, :35-38 (cost_ratio 1)
                        X::at(leaf_cost[j], lane) = lc; X::at(best_cost[j], lane) = lc;
                        X::at(best_pos[j], lane) = (p + se + 1) / 2; X::at(best_axis[j], lane) = 0;     // sweep_sah_builder.h:111
                        X::at(best_larea[j], lane) = (T)0; X::at(best_rarea[j], lane) = (T)0;
                    }
                }
            });
            // ---- cost of splitting after pos (left = [begin, pos], right = [pos + 1, end)); first minimum per segment ----
            X::from_above(next_right_cost, right_cost[0], 1);
            X::each([&] (unsigned lane) {
                BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
                    const uint32_t p = 2 * lane + j, se = X::at(seg_e[j], lane);
                    T cost = inf;
                    if (X::at(live[j], lane) && p + 1 < se) {
                        const T rc = j == 0 ? X::at(right_cost[1], lane) : X::at(next_right_cost, lane);
                        cost = R::add(R::mul(box_half_area(X::at(pre[j], lane)), (T)(p + 1 - X::at(seg_b[j], lane))), rc);
                    }
                    X::at(cand_cost[j], lane) = cost; X::at(cand_pos[j], lane) = p + 1;
                }
                // suffix minimum inside the lane (ties: the earlier position stays — strict < in the reference's sweep)
                if (X::at(seg_e[0], lane) > 2 * lane + 1 && X::at(cand_cost[1], lane) < X::at(cand_cost[0], lane)) {
                    X::at(cand_cost[0], lane) = X::at(cand_cost[1], lane); X::at(cand_pos[0], lane) = X::at(cand_pos[1], lane);
                }
            });
            {
                typename X::template Var<T> mc, gc;
                typename X::template Var<uint32_t> mp, gp;
                X::each([&] (unsigned lane) { X::at(mc, lane) = X::at(cand_cost[0], lane); X::at(mp, lane) = X::at(cand_pos[0], lane); });
                for (unsigned d = 1; d < 32 && 2 * d < reach; d <<= 1) {     // (a step with 2d >= reach joins nothing)
                    X::from_above(gc, mc, d); X::from_above(gp, mp, d);
                    X::each([&] (unsigned lane) {
                        if (lane + d < 32 && X::at(seg_e[0], lane) > 2 * (lane + d) && X::at(gc, lane) < X::at(mc, lane)) {
                            X::at(mc, lane) = X::at(gc, lane); X::at(mp, lane) = X::at(gp, lane);
                        }
                    });
                }
                X::from_above(gc, mc, 1); X::from_above(gp, mp, 1);
                X::each([&] (unsigned lane) {
                    const uint32_t p1 = 2 * lane + 1;
                    if (lane + 1 < 32 && X::at(seg_e[1], lane) > p1 + 1) {                   // the next lane continues my second position's segment
                        if (X::at(gc, lane) < X::at(cand_cost[1], lane)) { X::at(cand_cost[1], lane) = X::at(gc, lane); X::at(cand_pos[1], lane) = X::at(gp, lane); }
                    }
                    // (the first position's value over its whole segment is the aggregate mc / mp)
                    X::at(cand_cost[0], lane) = X::at(mc, lane); X::at(cand_pos[0], lane) = X::at(mp, lane);
                });
            }
            X::sync();                                                                       // area_pre / area_suf are complete
            X::each([&] (unsigned lane) {                                                    // heads: keep the best axis (first one on ties)
                BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
                    const uint32_t p = 2 * lane + j, se = X::at(seg_e[j], lane);
                    if (!X::at(live[j], lane) || X::at(seg_b[j], lane) != p || se - p < 2) continue;
                    if (X::at(cand_cost[j], lane) < X::at(best_cost[j], lane)) {
                        const uint32_t k = X::at(cand_pos[j], lane);
                        X::at(best_cost[j], lane) = X::at(cand_cost[j], lane); X::at(best_pos[j], lane) = k; X::at(best_axis[j], lane) = a;
                        X::at(best_larea[j], lane) = w.area_pre[k - 1];
                        X::at(best_rarea[j], lane) = w.area_suf[k];
                    }
                }
            });
            X::sync();                                                                       // before the next axis overwrites the areas
        }

        // ---- decide every live segment: leaf, SAH split or median fallback; write the node record ----
        typename X::template Var<uint32_t> leaf_depth;
        X::each([&] (unsigned lane) {
            X::at(leaf_depth, lane) = 0;
            BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
                const uint32_t p = 2 * lane + j, se = X::at(seg_e[j], lane);
                if (!X::at(live[j], lane) || X::at(seg_b[j], lane) != p) continue;
                const uint32_t count = se - p;
                const Box6<T>& nb = X::at(node_box[j], lane);
                bool do_split = false;
                uint32_t k = X::at(best_pos[j], lane), axis = X::at(best_axis[j], lane);
                T larea = X::at(best_larea[j], lane), rarea = X::at(best_rarea[j], lane);
                if (count > min_leaf) {                                                      // top_down_sah_builder.h:89
                    if (X::at(best_cost[j], lane) < X::at(leaf_cost[j], lane)) do_split = true;      // sweep_sah_builder.h:116
                    else if (count > max_leaf) {                                             // :117-123: median on the largest axis
                        const T d0 = R::sub(nb.v[1], nb.v[0]), d1 = R::sub(nb.v[3], nb.v[2]), d2 = R::sub(nb.v[5], nb.v[4]);
                        axis = 0;                                                            // Vec::get_largest_axis
                        if (d0 < d1) axis = 1;
                        if ((axis == 0 ? d0 : d1) < d2) axis = 2;
                        k = (p + se + 1) / 2;
                        larea = (T)0; rarea = (T)0;                                          // (no SATO swap for the fallback)
                        do_split = true;
                    }
                }
                const T bmin[3] = { nb.v[0], nb.v[2], nb.v[4] }, bmax[3] = { nb.v[1], nb.v[3], nb.v[5] };
                const uint32_t slot = w.dst_slot[p], depth = w.depth[p];
                if (do_split) {
                    // one of the pairs l .. r-1 the LBVH subtree owned: the one of the split boundary, as in the LBVH
                    // numbering (every inner node of a tree over a contiguous range splits at a different boundary)
                    const uint32_t pair = l + k - 1u;
                    if (alive) alive[pair] = 1u;
                    const bool swap = larea < rarea;                                         // SATO, top_down_sah_builder.h:101-108
                    write_node(nodes + slot, bmin, bmax, make_index<U>((U)(2 * (size_t)pair + 1), 0));
                    // the children's heads are p (left part) and k (right part); decision is read by every position of the segment
                    w.decision[p] = 1u | (axis << 1) | (k << 8) | (swap ? 1u << 16 : 0u);
                } else {
                    write_node(nodes + slot, bmin, bmax, make_index<U>((U)(l + p), count));
                    if (depth > X::at(leaf_depth, lane)) X::at(leaf_depth, lane) = depth;
                    w.decision[p] = 0u;
                }
            }
        });
        {
            const uint32_t deepest = X::max_over_lanes(leaf_depth);                         // deepest leaf of this level
            if (deepest > treelet_depth) treelet_depth = deepest;
        }
        X::sync();                                                                           // decisions are visible

        // ---- partition: mark sides on the split axis, stable-partition the two other orders ----
        typename X::template Var<uint32_t> dec[2];
        X::each([&] (unsigned lane) {
            BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
                const uint32_t p = 2 * lane + j;
                uint32_t d = 0;
                if (X::at(live[j], lane)) d = w.decision[X::at(seg_b[j], lane)];
                X::at(dec[j], lane) = d;
                if (d & 1u) w.side[w.order[cur][(d >> 1) & 3u][p]] = p < ((d >> 8) & 0xFFu) ? 1 : 0;
            }
        });
        X::sync();
        for (uint32_t b = 0; b < 3; ++b) {
            typename X::template Var<bool> goes_left[2];
            X::each([&] (unsigned lane) {
                BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
                    const uint32_t p = 2 * lane + j, d = X::at(dec[j], lane);
                    const bool moves = (d & 1u) && ((d >> 1) & 3u) != b;
                    X::at(goes_left[j], lane) = moves && w.side[w.order[cur][b][p]] != 0;
                }
            });
            const uint32_t left_even = X::ballot(goes_left[0]), left_odd = X::ballot(goes_left[1]);
            X::each([&] (unsigned lane) {
                BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
                    const uint32_t p = 2 * lane + j;
                    if (p >= n) continue;
                    const uint32_t d = X::at(dec[j], lane), prim = w.order[cur][b][p];
                    uint32_t dst = p;
                    if ((d & 1u) && ((d >> 1) & 3u) != b) {
                        const uint32_t h = X::at(seg_b[j], lane), k = (d >> 8) & 0xFFu;
                        // left-goers at positions [h, p): even positions 2i with (h+1)/2 <= i < (p+1)/2, odd ones with h/2 <= i < p/2
                        auto below = [] (uint32_t i) { return i >= 32 ? 0xFFFFFFFFu : (1u << i) - 1u; };
                        const uint32_t before = treelet_popcount(left_even & below((p + 1) >> 1) & ~below((h + 1) >> 1))
                                              + treelet_popcount(left_odd & below(p >> 1) & ~below(h >> 1));
                        dst = X::at(goes_left[j], lane) ? h + before : k + (p - h - before);
                    }
                    w.order[cur ^ 1u][b][dst] = (uint8_t)prim;
                }
            });
        }
        // ---- the children become the segments of the next level ----
        X::each([&] (unsigned lane) {
            BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
                const uint32_t p = 2 * lane + j, d = X::at(dec[j], lane);
                if (!X::at(live[j], lane)) continue;
                const uint32_t h = X::at(seg_b[j], lane);
                if (!(d & 1u)) {                                                             // its node became a leaf: finished
                    X::at(live[j], lane) = false; X::at(seg_b[j], lane) = p; X::at(seg_e[j], lane) = p + 1;
                    continue;
                }
                const uint32_t k = (d >> 8) & 0xFFu;
                if (p == h) {                                                                // the old head hands slots and depth to both children
                    const uint32_t pair = l + k - 1u, swap = (d >> 16) & 1u;
                    const uint8_t depth = (uint8_t)(w.depth[h] + 1);
                    w.dst_slot[k] = (uint32_t)child_slot(pair, swap ? 0 : 1); w.depth[k] = depth;
                    w.dst_slot[h] = (uint32_t)child_slot(pair, swap ? 1 : 0); w.depth[h] = depth;
                }
                if (p < k) X::at(seg_e[j], lane) = k; else X::at(seg_b[j], lane) = k;
            }
            X::at(flag, lane) = X::at(live[0], lane) || X::at(live[1], lane);
            uint32_t longest = 0;
            BVH_UNROLL
            for (int j = 0; j < 2; ++j)
                if (X::at(live[j], lane) && X::at(seg_e[j], lane) - X::at(seg_b[j], lane) > longest) longest = X::at(seg_e[j], lane) - X::at(seg_b[j], lane);
            X::at(leaf_depth, lane) = longest;                                               // (variable reused for the reduction below)
        });
        reach = X::max_over_lanes(leaf_depth);
        cur ^= 1u;
        X::sync();                                                                           // new orders, slots and depths are visible
    }

    // ---- final primitive order = order along axis 0 (every leaf's primitives are contiguous in all three) ----
    X::each([&] (unsigned lane) {
        BVH_UNROLL
        for (int j = 0; j < 2; ++j) {
            const uint32_t pos = 2 * lane + j;
            if (pos >= n) continue;
            const uint32_t id = w.old_ids[w.order[cur][0][pos]];
            prim_ids[l + pos] = id;
            if (leaf_mode == 0 && tris) {
                T v[9];
                for (int k = 0; k < 9; ++k) v[k] = leaf_src[9 * (size_t)id + k];
                tris[l + pos] = precompute_tri(v);
            }
            if (pos == 0 && treelet_depth > old_depth) X::atomic_max(info + 2, treelet_depth - old_depth);
        }
    });
    X::sync();
}

} // namespace bvhb200
