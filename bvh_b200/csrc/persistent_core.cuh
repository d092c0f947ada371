// bvh_b200/csrc/persistent_core.cuh — the warp scheduler of the persistent traversal kernels.
//
// Persistent warps claim private runs of consecutive rays with one global atomicAdd per run and hand them to their idle
// lanes by ballot + prefix rank (active-mask compaction).  A warp draws new rays only once `refill_min` of its lanes are
// idle: the rays drawn together are neighbours (consecutive positions of one run) and start at the root in the same
// iteration, so they stay in step through the top of the tree and their node fetches — same address in the same
// instruction — cost one L1 wavefront instead of one per lane; the price is idle lanes, which these L1-bound kernels can
// afford.  A round is then a bounded inner-node phase, a reconvergence point and one leaf per lane.
//
// What a ray is, where it comes from, what a leaf does and where a finished ray goes belong to the kernel: the library's
// triangle kernels (traverse.cu), DeviceView::trace over the caller's own leaf and DeviceView::query over the caller's
// own node test (include/bvh/v2/cuda/intersect.cuh) pass them in as callables, so all of them run the same rounds.
#pragma once

#include <cstdint>

namespace bvhb200 {

// Resident blocks per SM the persistent kernel's registers are limited for (float, the variants without hit staging):
// 8 -> 64 registers, 9 -> 56, 10 -> 48.  The kernel is latency-bound, so more resident warps per SM hide more of it; on
// the H100 (bench.py c2 / c3) 12 blocks (40 registers, spills) were measured 1.4x slower than 9.  The variants with
// warp-staged hit stores (kGather) keep 8.
#ifndef BVH_TRACE_BLOCKS
#define BVH_TRACE_BLOCKS 9
#endif
constexpr int kTraceBlock = 128;

#if defined(__CUDACC__)

// A round past the watchdog's limit sets the status word: a hang becomes an error (see trace_rays).
__device__ __forceinline__ bool watchdog_fired(uint32_t& rounds, uint32_t limit, uint32_t* status, unsigned lane) {
    if (++rounds <= limit) return false;
    if (lane == 0) atomicExch(status, 1u);
    return true;
}

// First position of a new run of `run` positions (warp-uniform; it may lie beyond the batch).
__device__ __forceinline__ unsigned long long claim_run(unsigned long long* next_ray, uint32_t run, unsigned lane, unsigned mask) {
    unsigned long long first = 0;
    if (lane == 0) first = atomicAdd(next_ray, (unsigned long long)run);
    return __shfl_sync(mask, first, 0);
}

// The rest of the warp's current run, and whether the batch has no rays left (warp-uniform).
struct RunCursor {
    unsigned long long pos = 0, end = 0;
    bool exhausted = false;
};

// Refills the warp's idle lanes among `lanes`, once refill_min of them are idle, until none is idle or the batch has no
// rays left.  draw(idle, rank) hands out one round of rays (rank: the lane's rank in `idle`, counted over lt_mask); it
// returns false when the batch has none left.  account() runs after every draw that handed out rays (the hit staging of
// the gather mode books the records of rays retired as they were drawn).
template <typename Draw, typename Account>
__device__ __forceinline__ void refill_lanes(const bool& has_ray, const RunCursor& c, unsigned lanes, uint32_t refill_min,
                                             unsigned lt_mask, unsigned mask, Draw&& draw, Account&& account) {
    unsigned idle = __ballot_sync(mask, !has_ray) & lanes;
    if ((uint32_t)__popc(idle) < refill_min) idle = 0u;
    while (idle != 0u && !c.exhausted) {
        if (!draw(idle, (unsigned)__popc(idle & lt_mask))) break;
        account();
        idle = __ballot_sync(mask, !has_ray) & lanes;
    }
}

// The rounds of a persistent kernel, until the batch has no rays left.  A round: the watchdog when kWatchdog (`rounds`:
// the count to start from; `limit` and `status`, see watchdog_fired, are read where the watchdog fires); refill_lanes
// through draw(idle, rank) and account(); the inner phase inner(), which retires the rays it finishes; the leaf phase
// leaf(), one leaf per lane holding one, which retires a ray that ends there; account().  `mask` is the member mask of
// every warp primitive.  finish() runs once the batch is done, not when the watchdog fired.  The lane's ray state
// (has_ray and whatever the callables share) belongs to the kernel.
template <bool kWatchdog, typename Draw, typename Account, typename Inner, typename Leaf, typename Finish>
__device__ __forceinline__ void run_rounds(const RunCursor& run, bool& has_ray, unsigned mask, uint32_t rounds, const uint32_t& limit,
                                           uint32_t* const& status, unsigned lanes, uint32_t refill_min, unsigned lt_mask, unsigned lane,
                                           Draw&& draw, Account&& account, Inner&& inner, Leaf&& leaf, Finish&& finish) {
    for (;;) {
        if (kWatchdog && watchdog_fired(rounds, limit, status, lane)) return;
        refill_lanes(has_ray, run, lanes, refill_min, lt_mask, mask, draw, account);
        if (__ballot_sync(mask, has_ray) == 0u) {
            if (run.exhausted) break;                        // nothing in flight and nothing left
            continue;                                        // (only rays that ended at once were drawn: refill again)
        }
        inner();
        __syncwarp(mask);
        leaf();
        __syncwarp(mask);
        account();
    }
    finish();
}

#endif

} // namespace bvhb200
