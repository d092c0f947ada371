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

} // namespace bvhb200
