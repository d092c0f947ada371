// bvh_b200/csrc/trace_plan.h — which traversal kernel a batched call runs, and with which scheduling settings.
//
// Plain C++ with no CUDA in it, so that the choice can be compiled and checked on a host (tests/host_emul.cpp).
#pragma once

#include <cstdint>

namespace bvhb200 {

enum TraceFlags : unsigned {
    kTraceAnyHit      = 1u << 0,
    kTraceRobust      = 1u << 1,
    kTraceLastVisited = 1u << 2,   // reference example tie semantics instead of the canonical lowest id
    kTraceSimple      = 1u << 8,   // one-thread-per-ray kernel instead of the persistent one
    kTraceNoTma       = 1u << 9,   // persistent one-lane-per-ray kernel, rays read with streaming loads
    kTraceTma         = 1u << 10,  // persistent one-lane-per-ray kernel, ray chunks staged by bulk async copy (TMA)
    kTracePair        = 1u << 11,  // persistent lane-pair kernel (two lanes per ray)
    kTraceWide        = 1u << 12,  // persistent kernel over the compressed 4-wide tree
    kTraceSortRays    = 1u << 13,  // traverse the batch in the Morton order of the ray origins (results stay in the caller's order)
};

// The values are reported through BVH_PROP_LAST_KERNEL (include/bvh_b200.h).
enum TraceKernel : int { kKernelNone = 0, kKernelPersistentTma, kKernelPersistent, kKernelSimple, kKernelStats, kKernelPair, kKernelWide };

struct TraceRequest {
    unsigned flags;                 // TraceFlags
    bool stats;                     // per-ray statistics requested
    bool is_float;
    bool wide_tree;                 // the tree has a wide companion, or one can still be derived
    bool gather;                    // fused multi-GPU gather
    unsigned long long n;           // rays in the batch
    // the switches the choice reads (Tunables)
    int variant;
    int use_wide;
    uint32_t refill_min, inner_budget, wide_budget;   // 0: auto (refill_min, inner_budget)
};

struct TracePlan {
    TraceKernel kernel;
    bool sort_rays;                 // traverse the rays in the Morton order of their origins
    uint32_t refill_min;            // persistent kernels: idle lanes a warp waits for before it draws new rays
    uint32_t inner_budget;          // persistent kernels: inner steps per lane and round (0xFFFFFFFF: unbounded)
};

// First match wins:
//   statistics                                                   -> kKernelStats
//   kTraceSimple                                                 -> kKernelSimple
//   float, not order-sensitive (LastVisited, Robust, statistics), and kTraceWide or use_wide > 0 without an explicit
//   binary kernel flag, and a wide tree                          -> kKernelWide
//   kTracePair                                                   -> kKernelPair
//   otherwise the persistent kernel, with bulk-copied ray chunks (TMA) for kTraceTma, or for variant 1 without a
//   TMA / NO_TMA flag, unless the rays are sorted (a sorted run of positions is not a contiguous range of rays).
// Sorting applies to the persistent and wide kernels, outside gather mode (its staging groups are runs of consecutive
// ray indices) and for 2^16 <= n < 2^32 - 1.
inline TracePlan plan_trace(const TraceRequest& q) {
    const unsigned f = q.flags;
    const bool order_sensitive = (f & (kTraceLastVisited | kTraceRobust)) != 0 || q.stats;
    const bool explicit_binary = (f & (kTracePair | kTraceNoTma | kTraceTma | kTraceSimple)) != 0;
    const bool want_wide = q.is_float && !order_sensitive && ((f & kTraceWide) || (!explicit_binary && q.use_wide > 0));
    TracePlan p;
    if (q.stats) p.kernel = kKernelStats;
    else if (f & kTraceSimple) p.kernel = kKernelSimple;
    else if (want_wide && q.wide_tree) p.kernel = kKernelWide;
    else if (f & kTracePair) p.kernel = kKernelPair;
    else p.kernel = ((f & kTraceTma) || (!(f & kTraceNoTma) && q.variant == 1)) ? kKernelPersistentTma : kKernelPersistent;
    p.sort_rays = (f & kTraceSortRays) && !q.gather && q.n >= (1u << 16) && q.n < 0xFFFFFFFFull &&
                  (p.kernel == kKernelPersistent || p.kernel == kKernelPersistentTma || p.kernel == kKernelWide);
    if (p.sort_rays && p.kernel == kKernelPersistentTma) p.kernel = kKernelPersistent;
    // 0 = auto (DESIGN.md §3, measured on the H100): closest-hit rays in the binary persistent kernel run best with 14 / 4;
    // any-hit rays and the lane-pair and wide kernels with 8 / 8.  The wide kernel has a budget of its own.
    const bool closest_binary = !(f & kTraceAnyHit) && (p.kernel == kKernelPersistent || p.kernel == kKernelPersistentTma);
    p.refill_min = q.refill_min ? q.refill_min : closest_binary ? 14u : 8u;
    p.inner_budget = p.kernel == kKernelWide ? q.wide_budget : q.inner_budget ? q.inner_budget : closest_binary ? 4u : 8u;
    return p;
}

// The scheduling of DeviceView::query (include/bvh/v2/cuda/intersect.cuh): node-test queries on the persistent
// scheduler, with the settings every kernel but the binary closest-hit one has (8 / 8).  Untuned: nobody has measured
// node-test queries on the H100 with other values.
struct QueryPlan {
    uint32_t refill_min;            // idle lanes a warp waits for before it draws new queries
    uint32_t inner_budget;          // node steps per lane and round
};
inline QueryPlan plan_query() { return QueryPlan { 8u, 8u }; }

// The default length of a persistent warp's private run of consecutive rays (Tunables::chunk_rays, the switch
// "chunk_rays"), and the default rounding of the traversal stack's entries (Tunables::stack_round).
constexpr uint32_t kDefaultRunRays = 64;
constexpr uint32_t kDefaultStackRound = 2;

// The run a persistent warp claims with one global atomic: `chunk_rays` at most, and shorter for small batches, so that
// every resident warp gets about 8 runs (tail balance), in multiples of 32 rays and never fewer than 32.
inline uint32_t persistent_run_rays(uint32_t chunk_rays, unsigned long long n, int sm_count) {
    uint32_t run = chunk_rays;
    const unsigned long long fair = n / ((unsigned long long)sm_count * 32ull * 8ull);
    if (fair < run) run = (uint32_t)fair;
    run &= ~31u;
    return run < 32u ? 32u : run;
}

// The grid of a persistent launch: one resident wave (SM count x resident blocks per SM, at least one), never more
// blocks than the batch can feed at `rays_per_warp` rays per warp.
inline unsigned long long persistent_grid(int sm_count, int blocks_per_sm, unsigned long long n, unsigned rays_per_warp,
                                          unsigned warps_per_block) {
    if (blocks_per_sm < 1) blocks_per_sm = 1;
    unsigned long long grid = (unsigned long long)sm_count * blocks_per_sm;
    const unsigned long long max_useful = (n + rays_per_warp - 1) / rays_per_warp / warps_per_block + 1;
    return grid > max_useful ? max_useful : grid;
}

// Shared-memory stack entries per thread of a tree of `depth`: depth + 1 pending far children at most and the sentinel,
// rounded up to a multiple of `round`, and at least 16.
inline uint32_t stack_entries(uint32_t depth, uint32_t round) {
    uint32_t entries = depth + 2;
    entries = (entries + round - 1u) / round * round;
    return entries < 16 ? 16 : entries;
}

} // namespace bvhb200
