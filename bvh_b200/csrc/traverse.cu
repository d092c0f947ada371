// bvh_b200/csrc/traverse.cu — batched closest-hit / any-hit ray traversal kernels (sm_90a).
//
// Replaces the caller-side ray loop around Bvh::intersect (reference bvh.h:159-182 driven by
// test/benchmark.cpp:340-393 / c_api/bvh_impl.h:235-250) with two kernels over a whole ray batch:
//
//   trace_persistent_kernel  persistent warps.  Each warp owns private runs of consecutive rays claimed with one
//                            global atomicAdd per run; idle lanes are refilled from the run by ballot + prefix rank
//                            (active-mask compaction) once `refill_min` of them are idle, so that the rays drawn
//                            together — neighbours — walk the top of the tree in step and share their node fetches.
//                            The body is a while-while loop: an inner-node phase bounded to `inner_budget` steps per
//                            lane and round, a reconvergence point, then a leaf phase (Moeller-Trumbore in
//                            registers).  The traversal stack lives in shared memory, laid out [entry][thread] so that
//                            a warp's accesses never bank-conflict.  kTma: the run's rays staged into shared memory by
//                            bulk async copies instead of streaming loads; kGather: hit records delivered to every
//                            rank's gathered array by warp-staged bulk copies (fused multi-GPU gather).
//   trace_simple_kernel      one thread per ray, same stack machine; also the statistics variant that
//                            counts inner steps / leaves / triangle tests per ray (the reference's
//                            InnerFn hook, bvh.h:168) which defines the algorithmic bytes of DESIGN.md.
//
// Both kernels execute the reference's per-ray algorithm exactly (traverse_core.cuh), so on the same
// tree they visit nodes in the same order as the CPU code and produce bit-identical ids, t, u, v.
#include <cstdio>
#include <cstdlib>
#include <type_traits>

#include "build_core.cuh"
#include "engine.h"
#include "radix_sort.cuh"
#include "traverse_core.cuh"
#include "wide_bvh.cuh"

namespace bvhb200 {

namespace {

// Resident blocks per SM the persistent kernel's registers are limited for (float, the variants without hit staging):
// 8 -> 64 registers, 9 -> 56, 10 -> 48.  The kernel is latency-bound, so more resident warps per SM hide more of it; on
// the H100 (bench.py c2 / c3) 12 blocks (40 registers, spills) were measured 1.4x slower than 9.  The variants with
// warp-staged hit stores (kGather) keep 8.
#ifndef BVH_TRACE_BLOCKS
#define BVH_TRACE_BLOCKS 9
#endif
constexpr int kTraceBlock = 128;
constexpr int kChunkRays = 128;          // rays claimed per global atomic by one warp

__device__ __forceinline__ void load_ray(const DevRay<float>* __restrict__ rays, size_t i, RayCtx<float>& r) {
    const float4* q = reinterpret_cast<const float4*>(rays + i);
    const float4 a = __ldcs(q), b = __ldcs(q + 1);           // streamed once: evict-first
    r.org[0] = a.x; r.org[1] = a.y; r.org[2] = a.z; r.dir[0] = a.w;
    r.dir[1] = b.x; r.dir[2] = b.y; r.tmin = b.z; r.tmax = b.w;
}
__device__ __forceinline__ void load_ray(const DevRay<double>* __restrict__ rays, size_t i, RayCtx<double>& r) {
    const double2* q = reinterpret_cast<const double2*>(rays + i);
    const double2 a = __ldcs(q), b = __ldcs(q + 1), c = __ldcs(q + 2), d = __ldcs(q + 3);
    r.org[0] = a.x; r.org[1] = a.y; r.org[2] = b.x; r.dir[0] = b.y;
    r.dir[1] = c.x; r.dir[2] = c.y; r.tmin = d.x; r.tmax = d.y;
}

// Where a finished ray's hit record goes: the caller's local array and, in the fused multi-GPU mode, the
// gathered array of EVERY rank (peer stores over NVLink, or one multimem store through the NVSwitch
// multicast address).  See trace_rays_gather / DESIGN.md "Multi-GPU".
constexpr int kMaxPeers = 8;
template <typename T> struct HitSinks {
    DevHit<T>* local;                 // may be null in gather mode
    DevHit<T>* peer[kMaxPeers];       // gathered arrays (own rank included), already offset to this shard
    int peer_count;
    DevHit<T>* multicast;             // multicast alias of the gathered array (offset to this shard) or null
};

__device__ __forceinline__ void multimem_store_v4(void* p, uint4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};"
                 :: "l"(p), "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w)) : "memory");
}

// A miss reports id = all ones (BVH_INVALID_PRIM_ID), t = the ray's tmax, u = v = 0.
__device__ __forceinline__ void store_hit(const HitSinks<float>& sinks, size_t i, const HitState<float>& h,
                                          float tmax, const uint32_t* __restrict__ prim_ids) {
    uint4 o;
    const bool was_hit = h.slot != kInvalidId;
    o.x = was_hit ? prim_ids[h.slot] : kInvalidId;
    o.y = __float_as_uint(was_hit ? h.t : tmax);
    o.z = __float_as_uint(was_hit ? h.u : 0.f);
    o.w = __float_as_uint(was_hit ? h.v : 0.f);
    if (sinks.local) __stcs(reinterpret_cast<uint4*>(sinks.local + i), o);
    if (sinks.multicast) multimem_store_v4(sinks.multicast + i, o);
    else for (int p = 0; p < sinks.peer_count; ++p) *reinterpret_cast<uint4*>(sinks.peer[p] + i) = o;
}
__device__ __forceinline__ void store_hit(const HitSinks<double>& sinks, size_t i, const HitState<double>& h,
                                          double tmax, const uint32_t* __restrict__ prim_ids) {
    const bool was_hit = h.slot != kInvalidId;
    ulonglong2 a, b;
    a.x = was_hit ? (unsigned long long)prim_ids[h.slot] : ~0ull;
    a.y = (unsigned long long)__double_as_longlong(was_hit ? h.t : tmax);
    b.x = (unsigned long long)__double_as_longlong(was_hit ? h.u : 0.0);
    b.y = (unsigned long long)__double_as_longlong(was_hit ? h.v : 0.0);
    if (sinks.local) {
        ulonglong2* d = reinterpret_cast<ulonglong2*>(sinks.local + i);
        __stcs(d, a);
        __stcs(d + 1, b);
    }
    for (int p = 0; p < sinks.peer_count; ++p) {
        ulonglong2* d = reinterpret_cast<ulonglong2*>(sinks.peer[p] + i);
        d[0] = a; d[1] = b;
    }
}

template <typename T> struct TraceArgs {
    const DevNode<T>* nodes;
    const DevTri<T>* tris;
    const uint32_t* prim_ids;
    const DevRay<T>* rays;
    HitSinks<T> hits;
    unsigned long long n;
    unsigned long long* next_ray;     // persistent kernel: global ray cursor
    uint32_t* ray_stats;              // statistics variant: n x 3
    uint32_t stack_entries;
    const WideNode* wide;             // compressed 4-wide tree (float only) or nullptr
    uint32_t wide_entries;            // stack entries per thread for the wide kernel
    int variant;                      // 0/1: one lane per ray (direct / TMA-staged rays), 2: lane-pair kernel
    bool use_tma;                     // persistent kernel: stage ray chunks with cp.async.bulk
    uint32_t inner_budget;            // persistent kernel: inner steps per lane per round (0xFFFFFFFF = unbounded)
    uint32_t chunk_rays;              // persistent kernels: consecutive rays a warp claims with one global atomic (multiple of 32)
    uint32_t refill_min;              // persistent kernels: idle lanes a warp waits for before it draws new rays (1: refill at once)
    uint32_t full_mask;               // 0xFFFFFFFF passed at run time (see trace_pair_kernel)
    const uint32_t* order;            // ray reordering: the ray drawn at position p is rays[order[p]] (null: identity)
    bool stage_hits;                  // gather mode: warp-aggregated bulk stores (false: one store per record and rank)
    uint32_t* status;                 // device word set to 1 when a watchdog fired
    uint32_t watchdog;                // persistent kernels: trap after this many rounds of one warp (a hang becomes an error)
    int lowest_id;
};

template <typename T, bool kAny, bool kRobust, bool kStats>
__global__ void __launch_bounds__(kTraceBlock)
trace_simple_kernel(TraceArgs<T> a) {
    using U = typename Real<T>::UInt;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const unsigned long long i = (unsigned long long)blockIdx.x * kTraceBlock + threadIdx.x;
    if (i >= a.n) return;
    SmemStack<U> stack { reinterpret_cast<U*>(smem_raw) + threadIdx.x, kTraceBlock, 0 };
    RayCtx<T> r;
    load_ray(a.rays, i, r);
    ray_prologue<T, kRobust>(r);
    HitState<T> hit { kInvalidId, r.tmax, (T)0, (T)0 };
    const T tmax_in = r.tmax;
    uint32_t stats[3] = { 0, 0, 0 };
    const U root_index = a.nodes[1].index;
    traverse_ray<T, kAny, kRobust>(a.nodes, a.tris, a.prim_ids, a.lowest_id != 0, root_index, r, hit, stack,
                                   kStats ? stats : nullptr);
    store_hit(a.hits, i, hit, tmax_in, a.prim_ids);
    if (kStats) {
        a.ray_stats[3 * i + 0] = stats[0];
        a.ray_stats[3 * i + 1] = stats[1];
        a.ray_stats[3 * i + 2] = stats[2];
    }
}

// ---- TMA (bulk async copy) helpers for the ray-chunk prefetch ------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }


// ---- warp-aggregated hit stores of the fused multi-GPU gather ------------------------------------------
// In gather mode every finished ray's record has to reach the gathered array of EVERY rank.  One 16-byte
// store per rank and ray (round 1) puts world_size extra store instructions per ray on the pipe this kernel
// is bound by (L1 LSU wavefronts).  Instead a warp stages the records of each GROUP of 32 consecutive rays
// (512 contiguous bytes of the output) in shared memory; when the group's last ray retires ONE lane issues one
// bulk asynchronous copy shared -> global per rank (cp.async.bulk, SASS UBLKCP: the copy is done by the TMA
// unit, not by the LSU pipe).  A warp keeps kStageSlots groups open; when a new group needs a slot and all
// are held by stragglers, the oldest is evicted: its finished records go out as plain per-record stores and
// its unfinished rays switch to per-record stores.  Records of rays without a slot are stored directly.
constexpr int kStageSlots = 2;
constexpr uint32_t kNoTag = 0xFFFFFFFFu;

__device__ __forceinline__ void bulk_copy_s2g(void* dst, uint32_t src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// Warp-uniform bookkeeping of a warp's staging slots.  It lives in SHARED memory, not in registers: the traversal loop
// only ever touches the two per-lane words of HitStager (as registers the nine words below cost the gather variants
// eight registers, spills in the inner loop and one resident block per SM: 4.1 instead of 3.2 ms per 10M rays, r02 N=2 run).
struct StagerWarp {
    uint32_t done[kStageSlots];     // bit i: record i of the slot's group is in the buffer
    uint32_t want[kStageSlots];     // the records the group has (all ones, or fewer for the batch's tail)
    uint32_t group[kStageSlots];    // ray index / 32 of the slot's group
    uint32_t used, draining;        // bit s: slot s holds an open group / is being read by a bulk copy
    uint32_t next;                  // slots are opened in cyclic order, so `next` is also the oldest one
    uint32_t cur;                   // slot of the group rays are currently drawn from, kStageSlots: none
};

template <typename T> __host__ __device__ constexpr size_t stage_smem_bytes() {
    return (size_t)(kTraceBlock / 32) * (kStageSlots * 32 * sizeof(DevHit<T>) + sizeof(StagerWarp));
}

template <typename T> struct HitStager {
    DevHit<T>* buf;                 // this warp's kStageSlots x 32 records in shared memory (null: staging off)
    StagerWarp* w;                  // this warp's bookkeeping (shared memory)
    // per lane
    uint32_t tag;                   // slot << 5 | index in the group of the lane's ray, kNoTag: direct stores
    uint32_t pending;               // tag of the record written since the last account(), kNoTag: none

    // stage_base: the block's staging area; records of all warps first, then the StagerWarp structs
    __device__ __forceinline__ void init(unsigned char* stage_base, unsigned warp, unsigned lane, bool on) {
        buf = on ? reinterpret_cast<DevHit<T>*>(stage_base) + (size_t)warp * kStageSlots * 32 : nullptr;
        w = reinterpret_cast<StagerWarp*>(stage_base + (size_t)(kTraceBlock / 32) * kStageSlots * 32 * sizeof(DevHit<T>)) + warp;
        if (lane == 0) {
            #pragma unroll
            for (int s = 0; s < kStageSlots; ++s) { w->done[s] = 0; w->want[s] = 0; w->group[s] = 0; }
            w->used = 0; w->draining = 0; w->next = 0; w->cur = kStageSlots;
        }
        __syncwarp();
        tag = kNoTag; pending = kNoTag;
    }
    // tag of a ray drawn now from the current group (converged callers only)
    __device__ __forceinline__ uint32_t tag_for(unsigned long long ray_index) const {
        const uint32_t cur = w->cur;
        return (buf && cur < (uint32_t)kStageSlots) ? (cur << 5) | (uint32_t)(ray_index & 31ull) : kNoTag;
    }
};

template <typename T>
__device__ __forceinline__ void store_record_direct(const HitSinks<T>& sinks, unsigned long long i, const DevHit<T>& rec) {
    using V = typename std::conditional<sizeof(T) == 4, uint4, ulonglong2>::type;
    constexpr int kParts = (int)(sizeof(DevHit<T>) / 16);
    const V* src = reinterpret_cast<const V*>(&rec);
    if (sinks.local) {
        V* d = reinterpret_cast<V*>(sinks.local + i);
        #pragma unroll
        for (int k = 0; k < kParts; ++k) __stcs(d + k, src[k]);
    }
    if (sizeof(T) == 4 && sinks.multicast) { multimem_store_v4(sinks.multicast + i, *reinterpret_cast<const uint4*>(&rec)); return; }
    for (int p = 0; p < sinks.peer_count; ++p) {
        V* d = reinterpret_cast<V*>(sinks.peer[p] + i);
        #pragma unroll
        for (int k = 0; k < kParts; ++k) d[k] = src[k];
    }
}

// All lanes of the warp call the functions below together (converged code); every lane reads the same shared words,
// lane 0 writes them back, a __syncwarp() separates the two.

// Slot s is complete: one lane sends its 32 records to every rank with bulk copies.
template <typename T>
__device__ __forceinline__ void stager_flush_full(HitStager<T>& st, const HitSinks<T>& sinks, int s, unsigned lane) {
    __syncwarp();                                                   // the lanes' shared-memory records are visible to lane 0
    if (lane == 0) {
        fence_proxy_async_smem();                                   // ... and to the async proxy that reads them
        const uint32_t count = 32u - (uint32_t)__clz(st.w->want[s]);  // want is a low mask
        const uint32_t bytes = count * (uint32_t)sizeof(DevHit<T>);
        const uint32_t src = smem_u32(st.buf + s * 32);
        const unsigned long long first = (unsigned long long)st.w->group[s] * 32ull;
        if (sinks.local) bulk_copy_s2g(sinks.local + first, src, bytes);
        if (sinks.multicast) bulk_copy_s2g(sinks.multicast + first, src, bytes);      // ONE copy, replicated to every rank by the NVSwitch
        else for (int p = 0; p < sinks.peer_count; ++p) bulk_copy_s2g(sinks.peer[p] + first, src, bytes);
        bulk_commit();
        st.w->used &= ~(1u << s);
        st.w->draining |= 1u << s;
    }
    __syncwarp();
}

// Slot s is needed for a new group while stragglers hold it: finished records leave as plain stores, unfinished rays
// switch to plain stores.
template <typename T>
__device__ __forceinline__ void stager_evict(HitStager<T>& st, const HitSinks<T>& sinks, int s, unsigned lane) {
    __syncwarp();
    if ((st.w->done[s] >> lane) & 1u)
        store_record_direct(sinks, (unsigned long long)st.w->group[s] * 32ull + lane, st.buf[s * 32 + lane]);
    if (st.tag != kNoTag && (int)(st.tag >> 5) == s) st.tag = kNoTag;       // the group's unfinished rays store directly
    __syncwarp();                                                   // the buffer is free for the next group
    if (lane == 0) st.w->used &= ~(1u << s);
    __syncwarp();
}

// A new group of `count` rays (ray index = 32 * group_id ...) starts being drawn: give it a slot.
template <typename T>
__device__ __forceinline__ void stager_open(HitStager<T>& st, const HitSinks<T>& sinks, unsigned long long group_id,
                                            uint32_t count, unsigned lane) {
    if (!st.buf) return;
    if (group_id > 0xFFFFFFFFull) { if (lane == 0) st.w->cur = kStageSlots; __syncwarp(); return; }
    constexpr uint32_t kAll = (1u << kStageSlots) - 1u;
    uint32_t used = st.w->used, draining = st.w->draining;
    if (((used | draining) & kAll) == kAll && draining != 0u) {
        if (lane == 0) { bulk_wait_read_all(); st.w->draining = 0; }           // the bulk copies have read their buffers
        __syncwarp();
        draining = 0;
    }
    int s = (int)st.w->next;
    if (((used | draining) >> s) & 1u) {                            // the next slot in cyclic order is not free
        #pragma unroll
        for (int k = 0; k < kStageSlots; ++k) if ((((used | draining) >> k) & 1u) == 0u) s = k;
    }
    if ((used >> s) & 1u) stager_evict(st, sinks, s, lane);        // every slot is held by stragglers: evict the oldest
    if (lane == 0) {
        st.w->done[s] = 0; st.w->want[s] = count >= 32u ? 0xFFFFFFFFu : ((1u << count) - 1u); st.w->group[s] = (uint32_t)group_id;
        st.w->used |= 1u << s;
        st.w->next = (uint32_t)(s + 1 == kStageSlots ? 0 : s + 1);
        st.w->cur = (uint32_t)s;
    }
    __syncwarp();
}

// Books the records written since the last call; flushes groups that became complete.
template <typename T>
__device__ __forceinline__ void stager_account(HitStager<T>& st, const HitSinks<T>& sinks, unsigned lane) {
    if (!st.buf) return;
    if (__ballot_sync(0xFFFFFFFFu, st.pending != kNoTag) == 0u) return;
    #pragma unroll
    for (int s = 0; s < kStageSlots; ++s) {
        const uint32_t mine = (st.pending != kNoTag && (int)(st.pending >> 5) == s) ? (1u << (st.pending & 31u)) : 0u;
        const uint32_t bits = __reduce_or_sync(0xFFFFFFFFu, mine);
        if (bits != 0u) {
            const uint32_t done = st.w->done[s] | bits;
            const bool full = done == st.w->want[s];
            __syncwarp();
            if (lane == 0) st.w->done[s] = done;
            if (full) stager_flush_full(st, sinks, s, lane); else __syncwarp();
        }
    }
    st.pending = kNoTag;
}

// One finished ray (divergent code): into the lane's staging slot, or straight to the sinks.
template <typename T>
__device__ __forceinline__ void stager_retire(HitStager<T>& st, const HitSinks<T>& sinks, unsigned long long i, const DevHit<T>& rec) {
    if (st.tag != kNoTag) {
        st.buf[(st.tag >> 5) * 32 + (st.tag & 31u)] = rec;
        st.pending = st.tag;
        st.tag = kNoTag;
    } else {
        store_record_direct(sinks, i, rec);
    }
}

template <typename T>
__device__ __forceinline__ DevHit<T> make_record(const HitState<T>& h, T tmax, const uint32_t* __restrict__ prim_ids) {
    DevHit<T> rec;
    const bool was_hit = h.slot != kInvalidId;
    rec.prim_id = was_hit ? (decltype(rec.prim_id))prim_ids[h.slot] : (decltype(rec.prim_id))~(decltype(rec.prim_id))0;
    rec.t = was_hit ? h.t : tmax;
    rec.u = was_hit ? h.u : (T)0;
    rec.v = was_hit ? h.v : (T)0;
    return rec;
}

__device__ __forceinline__ void read_ray_smem(const DevRay<float>* p, RayCtx<float>& r) {
    const float4* q = reinterpret_cast<const float4*>(p);
    const float4 a = q[0], b = q[1];
    r.org[0] = a.x; r.org[1] = a.y; r.org[2] = a.z; r.dir[0] = a.w;
    r.dir[1] = b.x; r.dir[2] = b.y; r.tmin = b.z; r.tmax = b.w;
}
__device__ __forceinline__ void read_ray_smem(const DevRay<double>* p, RayCtx<double>& r) {
    const double2* q = reinterpret_cast<const double2*>(p);
    const double2 a = q[0], b = q[1], c = q[2], d = q[3];
    r.org[0] = a.x; r.org[1] = a.y; r.org[2] = b.x; r.dir[0] = b.y;
    r.dir[1] = c.x; r.dir[2] = c.y; r.tmin = d.x; r.tmax = d.y;
}

constexpr int kTmaChunkRays = 32;        // rays per bulk copy (1 KB of float rays), two buffers per warp

template <typename T> __host__ __device__ constexpr size_t tma_smem_bytes() {
    return (size_t)(kTraceBlock / 32) * 2 * kTmaChunkRays * sizeof(DevRay<T>) + (size_t)(kTraceBlock / 32) * 2 * 8;
}

// Persistent kernel.  kTma = true stages the warp's next ray chunk into shared memory with a bulk
// asynchronous copy (cp.async.bulk, SASS UBLKCP) signalled through an mbarrier, double-buffered, so
// that the ray fetch of the refill path never waits on DRAM; kTma = false reads rays with streaming
// 128-bit loads.
template <typename T, bool kAny, bool kRobust, bool kTma, bool kGather>
__global__ void __launch_bounds__(kTraceBlock, sizeof(T) == 4 ? (kGather ? 8 : BVH_TRACE_BLOCKS) : 4)
trace_persistent_kernel(TraceArgs<T> a) {
    using U = typename Real<T>::UInt;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    constexpr unsigned kFull = 0xFFFFFFFFu;
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const unsigned lt_mask = (1u << lane) - 1u;
    SmemStack<U> stack { reinterpret_cast<U*>(smem_raw) + threadIdx.x, kTraceBlock, 0 };
    const bool lowest_id = a.lowest_id != 0;
    const U root_index = a.nodes[1].index;
    const uint32_t inner_budget = a.inner_budget;

    // warp-uniform cursor over the warp's private chunk(s) of rays
    unsigned long long chunk_pos = 0, chunk_end = 0;           // !kTma: global ray indices
    bool exhausted = false;
    // kTma state (warp-uniform)
    // (kept as scalars selected by `cur`, not arrays, so that nothing is spilled to local memory)
    DevRay<T>* ray_buf0 = nullptr; DevRay<T>* ray_buf1 = nullptr;
    uint32_t bar0 = 0, bar1 = 0, phase0 = 0, phase1 = 0, count0 = 0, count1 = 0;
    unsigned long long base0 = 0, base1 = 0;
    uint32_t cur = 0, buf_pos = 0;

    auto prefetch = [&] (uint32_t b) {      // stage the next 32 rays of the warp's private run (claiming a new run when it is used up)
        if (chunk_pos == chunk_end) {
            unsigned long long first = 0;
            if (lane == 0) first = atomicAdd(a.next_ray, (unsigned long long)a.chunk_rays);
            first = __shfl_sync(kFull, first, 0);
            chunk_pos = first;
            chunk_end = first + a.chunk_rays;               // (may lie beyond n: the count below is clipped)
        }
        const unsigned long long base = chunk_pos;
        chunk_pos += kTmaChunkRays;
        uint32_t cnt = 0;
        if (base < a.n) cnt = (uint32_t)(base + kTmaChunkRays < a.n ? kTmaChunkRays : a.n - base);
        if (b == 0) { count0 = cnt; base0 = base; } else { count1 = cnt; base1 = base; }
        if (cnt != 0 && lane == 0) {
            const uint32_t bar = b == 0 ? bar0 : bar1;
            fence_proxy_async_smem();       // earlier generic reads of this buffer happen-before the async write
            mbar_arrive_expect_tx(bar, cnt * (uint32_t)sizeof(DevRay<T>));
            bulk_copy_g2s(smem_u32(b == 0 ? ray_buf0 : ray_buf1), a.rays + base, cnt * (uint32_t)sizeof(DevRay<T>), bar);
        }
    };

    // gather mode: hit records leave through the warp's staging slots (HitStager above)
    HitStager<T> stager;
    if (kGather) {
        unsigned char* stage_base = smem_raw + (size_t)a.stack_entries * kTraceBlock * sizeof(U) + (kTma ? tma_smem_bytes<T>() : 0);
        stager.init(stage_base, warp, lane, a.stage_hits);
    }
    auto retire = [&] (unsigned long long index, const HitState<T>& h, T tmax) {
        if (kGather) stager_retire(stager, a.hits, index, make_record(h, tmax, a.prim_ids));
        else store_hit(a.hits, index, h, tmax, a.prim_ids);
    };

    if (kTma) {
        unsigned char* tma_base = smem_raw + (size_t)a.stack_entries * kTraceBlock * sizeof(U);
        DevRay<T>* bufs = reinterpret_cast<DevRay<T>*>(tma_base);
        uint64_t* bars = reinterpret_cast<uint64_t*>(tma_base + (size_t)(kTraceBlock / 32) * 2 * kTmaChunkRays * sizeof(DevRay<T>));
        ray_buf0 = bufs + ((size_t)warp * 2 + 0) * kTmaChunkRays;
        ray_buf1 = bufs + ((size_t)warp * 2 + 1) * kTmaChunkRays;
        bar0 = smem_u32(bars + warp * 2 + 0);
        bar1 = smem_u32(bars + warp * 2 + 1);
        if (lane == 0) { mbar_init(bar0, 1); mbar_init(bar1, 1); fence_mbar_init(); fence_proxy_async_smem(); }
        __syncwarp();
        prefetch(0);
        prefetch(1);
    }

    bool has_ray = false;
    unsigned long long ray_index = 0;
    RayCtx<T> r;
    HitState<T> hit;
    T tmax_in = (T)0;
    U top = 0;

    uint32_t rounds = 0;
    for (;;) {
        if (++rounds > a.watchdog) {                       // a hang becomes an error (see trace_rays)
            if (lane == 0) atomicExch(a.status, 1u);
            return;
        }
        // ---- refill idle lanes from the private chunk (claiming a new chunk when it runs dry) ----
        // A warp draws new rays only once refill_min of its lanes are idle.  The rays drawn together are neighbours
        // (consecutive indices of one chunk) and start at the root in the same iteration, so they stay in step through
        // the top of the tree and their node fetches — same address in the same instruction — cost one L1 wavefront
        // instead of one per lane; the price is idle lanes, which this L1-bound kernel can afford.
        unsigned idle = __ballot_sync(kFull, !has_ray);
        if ((uint32_t)__popc(idle) < a.refill_min) idle = 0u;
        while (idle != 0u && !exhausted) {
            unsigned take, rank = __popc(idle & lt_mask);
            bool got = false;
            if (kTma) {
                const uint32_t cur_count = cur == 0 ? count0 : count1;
                if (cur_count == 0) { exhausted = true; break; }
                const uint32_t cur_bar = cur == 0 ? bar0 : bar1, cur_phase = cur == 0 ? phase0 : phase1;
                while (!mbar_try_wait(cur_bar, cur_phase)) { }
                if (kGather && buf_pos == 0) stager_open(stager, a.hits, (cur == 0 ? base0 : base1) >> 5, cur_count, lane);
                const unsigned avail = cur_count - buf_pos, want = __popc(idle);
                take = want < avail ? want : avail;
                if (!has_ray && rank < take) {
                    ray_index = (cur == 0 ? base0 : base1) + buf_pos + rank;
                    read_ray_smem((cur == 0 ? ray_buf0 : ray_buf1) + buf_pos + rank, r);
                    got = true;
                }
                buf_pos += take;
                if (buf_pos == cur_count) {                // buffer drained: re-arm it with the next chunk
                    __syncwarp();
                    if (cur == 0) phase0 ^= 1u; else phase1 ^= 1u;
                    prefetch(cur);
                    cur ^= 1u; buf_pos = 0;
                }
            } else {
                if (chunk_pos == chunk_end) {
                    unsigned long long base = 0;
                    if (lane == 0) base = atomicAdd(a.next_ray, (unsigned long long)a.chunk_rays);
                    base = __shfl_sync(kFull, base, 0);
                    if (base >= a.n) { exhausted = true; break; }
                    chunk_pos = base;
                    chunk_end = base + a.chunk_rays < a.n ? base + a.chunk_rays : a.n;
                }
                unsigned avail = (unsigned)(chunk_end - chunk_pos);
                const unsigned want = __popc(idle);
                if (kGather) {                              // one staging group = 32 consecutive rays: never draw across a boundary
                    const unsigned in_group = (unsigned)(chunk_pos & 31ull);
                    if (in_group == 0) stager_open(stager, a.hits, chunk_pos >> 5, avail < 32u ? avail : 32u, lane);
                    if (avail > 32u - in_group) avail = 32u - in_group;
                }
                take = want < avail ? want : avail;
                if (!has_ray && rank < take) {
                    ray_index = chunk_pos + rank;
                    if (a.order) ray_index = a.order[ray_index];
                    load_ray(a.rays, ray_index, r);
                    got = true;
                }
                chunk_pos += take;
            }
            if (got) {
                tmax_in = r.tmax;
                hit.slot = kInvalidId; hit.t = r.tmax; hit.u = (T)0; hit.v = (T)0;
                if (kGather) stager.tag = stager.tag_for(ray_index);
                if (ray_interval_is_nan(r)) {
                    retire(ray_index, hit, tmax_in);                             // can never hit: retire as a miss
                } else {
                    ray_prologue<T, kRobust>(r);
                    top = root_index;
                    stack.clear();
                    has_ray = true;
                }
            }
            if (kGather) stager_account(stager, a.hits, lane);      // (a NaN ray may just have been retired)
            idle = __ballot_sync(kFull, !has_ray);
        }
        if (__ballot_sync(kFull, has_ray) == 0u) {
            if (exhausted) break;                            // nothing in flight and nothing left
            continue;                                        // (only NaN rays were drawn: refill again)
        }

        // ---- inner phase: descend until this lane holds a leaf, its ray is finished, or the step
        //      budget of this round is spent (bounding the wait of lanes that already hold a leaf) ----
        if (has_ray) {
            uint32_t budget = inner_budget;
            while (index_count(top) == 0 && budget != 0) {                     // (kTraversalDone ends it too)
                --budget;
                inner_step<T, kAny, kRobust>(a.nodes, r, top, stack);
            }
            if (top == kTraversalDone<U>) {
                retire(ray_index, hit, tmax_in);
                has_ray = false;
            }
        }
        __syncwarp();

        // ---- leaf phase ---------------------------------------------------------------------------
        if (has_ray && index_count(top) != 0) {
            leaf_step<T>(a.tris, a.prim_ids, lowest_id, top, r, hit, nullptr);
            if ((kAny && hit.slot != kInvalidId) || !stack.try_pop(top)) {
                retire(ray_index, hit, tmax_in);
                has_ray = false;
            }
        }
        __syncwarp();
        if (kGather) stager_account(stager, a.hits, lane);
    }
    if (kGather && stager.buf && lane == 0) bulk_wait_all();         // the last bulk stores have left shared memory and landed
}

// ---- lane-pair kernel ------------------------------------------------------------------------------
// Two adjacent lanes serve ONE ray: in an inner step lane 0 of the pair fetches and tests the left
// child, lane 1 the right child (one 256-bit load each, both from the same 64-byte block), and the two
// exchange (hit, entry distance, index) with pair-masked __ballot_sync / __shfl_xor_sync.  Why: with
// divergent rays the L1 data pipe spends one wavefront per thread per load (profiles/: the one-lane-per-ray
// kernel is bound by l1tex__data_pipe_lsu_wavefronts at ~87 % of peak); the two lanes of a pair hit the same
// line, so a whole sibling pair costs ONE wavefront instead of two.  Control state (top, stack pointer,
// tmax, hit) is replicated in both lanes, which take identical decisions; the leaf phase is executed
// redundantly by both lanes (same addresses, so no extra memory wavefronts).  Per-ray semantics are
// unchanged: same visit order, same results as traverse_ray().
template <typename U> __device__ __forceinline__ U shfl_xor1(unsigned mask, U v);
template <> __device__ __forceinline__ uint32_t shfl_xor1<uint32_t>(unsigned mask, uint32_t v) { return __shfl_xor_sync(mask, v, 1); }
template <> __device__ __forceinline__ uint64_t shfl_xor1<uint64_t>(unsigned mask, uint64_t v) { return __shfl_xor_sync(mask, (unsigned long long)v, 1); }
template <> __device__ __forceinline__ float shfl_xor1<float>(unsigned mask, float v) { return __shfl_xor_sync(mask, v, 1); }
template <> __device__ __forceinline__ double shfl_xor1<double>(unsigned mask, double v) { return __shfl_xor_sync(mask, v, 1); }

template <typename T, bool kAny, bool kRobust>
__global__ void __launch_bounds__(kTraceBlock, sizeof(T) == 4 ? 8 : 4)
trace_pair_kernel(TraceArgs<T> a) {
    using U = typename Real<T>::UInt;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    // The member mask of every warp-synchronous primitive below comes from a kernel argument (always
    // 0xFFFFFFFF).  With a compile-time full mask ptxas elides the hardware warp barrier wherever it
    // believes the warp is already converged and keeps the round counter in a uniform register; on an
    // earlier GPU that produced occasional hangs of this kernel (a warp split in two that never rejoined, found with
    // the watchdog below).  A run-time mask forces a real WARPSYNC in front of each vote / shuffle.
    const unsigned kFull = a.full_mask;
    constexpr unsigned kEven = 0x55555555u;
    const unsigned lane = threadIdx.x & 31u, sub = lane & 1u, pair_shift = lane & ~1u;
    const unsigned lt_mask = (1u << pair_shift) - 1u;                  // pairs before this one
    SmemStack<U> stack { reinterpret_cast<U*>(smem_raw) + (threadIdx.x >> 1), kTraceBlock / 2, 0 };
    const bool lowest_id = a.lowest_id != 0;
    const U root_index = a.nodes[1].index;
    const uint32_t inner_budget = a.inner_budget;

    unsigned long long chunk_pos = 0, chunk_end = 0;                   // warp-uniform
    bool exhausted = false;

    bool has_ray = false;
    unsigned long long ray_index = 0;
    RayCtx<T> r;
    HitState<T> hit;
    T tmax_in = (T)0;
    U top = 0;

    // `lane_zero` is 0 for every thread (blocks have 128 threads) but not provably so: adding it keeps the
    // round counters in ordinary per-lane registers instead of a warp-uniform register shared by the warp.
    const uint32_t lane_zero = threadIdx.x >> 10;
    uint32_t rounds = lane_zero;
    for (;;) {
        if (++rounds > a.watchdog) {                       // a hang becomes an error (see trace_rays)
            if (lane == 0) atomicExch(a.status, 1u);
            return;
        }
        // ---- refill idle pairs -----------------------------------------------------------------------
        unsigned idle = __ballot_sync(kFull, !has_ray) & kEven;
        while (idle != 0u && !exhausted) {
            if (chunk_pos == chunk_end) {
                unsigned long long base = 0;
                if (lane == 0) base = atomicAdd(a.next_ray, (unsigned long long)kChunkRays);
                base = __shfl_sync(kFull, base, 0);
                if (base >= a.n) { exhausted = true; break; }
                chunk_pos = base;
                chunk_end = base + kChunkRays < a.n ? base + kChunkRays : a.n;
            }
            const unsigned avail = (unsigned)(chunk_end - chunk_pos), want = __popc(idle);
            const unsigned take = want < avail ? want : avail;
            const unsigned rank = __popc(idle & lt_mask);
            if (!has_ray && rank < take) {
                ray_index = chunk_pos + rank;
                load_ray(a.rays, ray_index, r);
                tmax_in = r.tmax;
                hit.slot = kInvalidId; hit.t = r.tmax; hit.u = (T)0; hit.v = (T)0;
                if (ray_interval_is_nan(r)) {
                    if (sub == 0) store_hit(a.hits, ray_index, hit, tmax_in, a.prim_ids);
                } else {
                    ray_prologue<T, kRobust>(r);
                    top = root_index;
                    stack.clear();
                    has_ray = true;
                }
            }
            chunk_pos += take;
            idle = __ballot_sync(kFull, !has_ray) & kEven;
        }
        if (__ballot_sync(kFull, has_ray) == 0u) {
            if (exhausted) break;
            continue;
        }

        // ---- inner phase (bounded, WARP-UNIFORM trip count) ----------------------------------------------
        // Every lane runs every round of this loop so that the pair exchange can use full-mask warp
        // primitives (a pair-specific mask would make the hardware execute the shuffle once per pair).
        // The body is written without data-dependent branches: lanes that hold a leaf or no ray fetch the
        // root pair and discard the result, pushes / pops / retirement are predicated.
        {
            bool retired = false;
            for (uint32_t budget = inner_budget + lane_zero; budget != 0; --budget) {
                const bool active = has_ray && index_count(top) == 0;
                if (__ballot_sync(kFull, active) == 0u) break;
                T b[6]; U my_index;
                const size_t pair_slot = active ? (size_t)index_first(top) + 1 : (size_t)1;
                load_node(a.nodes + pair_slot + sub, b, my_index);
                T t0, t1;
                node_test<T, kRobust>(b, r, t0, t1);
                const bool my_hit = active && t0 <= t1;
                const unsigned votes = (__ballot_sync(kFull, my_hit) >> pair_shift) & 3u;
                const T other_t0 = shfl_xor1<T>(kFull, t0);
                const U other_index = shfl_xor1<U>(kFull, my_index);
                const U left_index = sub ? other_index : my_index, right_index = sub ? my_index : other_index;
                const T l0 = sub ? other_t0 : t0, r0 = sub ? t0 : other_t0;
                const bool hit_left = (votes & 1u) != 0, hit_right = (votes & 2u) != 0;
                const bool swap_order = !kAny && l0 > r0;                   // bvh.h:180
                const U near_index = hit_left ? ((hit_right && swap_order) ? right_index : left_index) : right_index;
                const U far_index = swap_order ? left_index : right_index;
                const bool do_push = active && hit_left && hit_right;
                const bool do_pop = active && !hit_left && !hit_right;
                if (do_push) stack.push(far_index);
                U next = near_index;
                const bool finished = do_pop && stack.empty();
                if (do_pop && !finished) next = stack.pop();
                if (active) top = next;
                if (finished) { has_ray = false; retired = true; }
            }
            if (retired && sub == 0) store_hit(a.hits, ray_index, hit, tmax_in, a.prim_ids);
        }
        __syncwarp(kFull);

        // ---- leaf phase (both lanes of the pair run it redundantly) -------------------------------------
        if (has_ray && index_count(top) != 0) {
            leaf_step<T>(a.tris, a.prim_ids, lowest_id, top, r, hit, nullptr);
            if ((kAny && hit.slot != kInvalidId) || stack.empty()) {
                if (sub == 0) store_hit(a.hits, ray_index, hit, tmax_in, a.prim_ids);
                has_ray = false;
            } else {
                top = stack.pop();
            }
        }
        __syncwarp();
    }
}


// ---- wide kernel: persistent traversal of the compressed 4-wide tree (wide_bvh.cuh) -------------------
// One lane per ray, same refill / bounded-round structure as trace_persistent_kernel.  An inner step
// fetches ONE 64-byte node (two 256-bit loads from the same line), dequantises four child boxes straight
// into ray-parameter space (t = q * (cell * inv_dir) + (origin - org) * inv_dir, far planes with the
// padded inverse direction so that rounding can only enlarge a box), visits the hit children nearest
// first and pushes the others far-to-near.  Leaves are the binary tree's leaves: same BVH-order triangle
// array, same exact triangle test and canonical tie-break as every other kernel.
template <bool kAny, bool kGather>
__global__ void __launch_bounds__(kTraceBlock, 8)
trace_wide_kernel(TraceArgs<float> a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    constexpr unsigned kFull = 0xFFFFFFFFu;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned lt_mask = (1u << lane) - 1u;
    SmemStack<uint32_t> stack { reinterpret_cast<uint32_t*>(smem_raw) + threadIdx.x, kTraceBlock, 0 };
    const uint32_t inner_budget = a.inner_budget;
    HitStager<float> stager;
    if (kGather) {
        unsigned char* stage_base = smem_raw + (size_t)a.wide_entries * kTraceBlock * sizeof(uint32_t);
        stager.init(stage_base, threadIdx.x >> 5, lane, a.stage_hits);
    }
    auto retire = [&] (unsigned long long index, const HitState<float>& h, float tmax) {
        if (kGather) stager_retire(stager, a.hits, index, make_record(h, tmax, a.prim_ids));
        else store_hit(a.hits, index, h, tmax, a.prim_ids);
    };

    unsigned long long chunk_pos = 0, chunk_end = 0;
    bool exhausted = false;
    bool has_ray = false;
    unsigned long long ray_index = 0;
    RayCtx<float> r;                   // aux = padded inverse direction (far planes)
    HitState<float> hit;
    float tmax_in = 0.f;
    uint32_t top = 0;

    uint32_t rounds = 0;
    for (;;) {
        if (++rounds > a.watchdog) {
            if (lane == 0) atomicExch(a.status, 1u);
            return;
        }
        unsigned idle = __ballot_sync(kFull, !has_ray);
        if ((uint32_t)__popc(idle) < a.refill_min) idle = 0u;       // (see trace_persistent_kernel)
        while (idle != 0u && !exhausted) {
            if (chunk_pos == chunk_end) {
                unsigned long long base = 0;
                if (lane == 0) base = atomicAdd(a.next_ray, (unsigned long long)a.chunk_rays);
                base = __shfl_sync(kFull, base, 0);
                if (base >= a.n) { exhausted = true; break; }
                chunk_pos = base;
                chunk_end = base + a.chunk_rays < a.n ? base + a.chunk_rays : a.n;
            }
            unsigned avail = (unsigned)(chunk_end - chunk_pos);
            const unsigned want = __popc(idle);
            if (kGather) {                                  // one staging group = 32 consecutive rays
                const unsigned in_group = (unsigned)(chunk_pos & 31ull);
                if (in_group == 0) stager_open(stager, a.hits, chunk_pos >> 5, avail < 32u ? avail : 32u, lane);
                if (avail > 32u - in_group) avail = 32u - in_group;
            }
            const unsigned take = want < avail ? want : avail;
            const unsigned rank = __popc(idle & lt_mask);
            if (!has_ray && rank < take) {
                ray_index = chunk_pos + rank;
                if (a.order) ray_index = a.order[ray_index];
                load_ray(a.rays, ray_index, r);
                tmax_in = r.tmax;
                hit.slot = kInvalidId; hit.t = r.tmax; hit.u = 0.f; hit.v = 0.f;
                if (kGather) stager.tag = stager.tag_for(ray_index);
                if (ray_interval_is_nan(r)) {
                    retire(ray_index, hit, tmax_in);
                } else {
                    wide_ray_setup(r);
                    top = 0;                                    // wide node 0, inner
                    stack.clear();
                    has_ray = true;
                }
            }
            chunk_pos += take;
            if (kGather) stager_account(stager, a.hits, lane);
            idle = __ballot_sync(kFull, !has_ray);
        }
        if (__ballot_sync(kFull, has_ray) == 0u) {
            if (exhausted) break;
            continue;
        }

        // ---- inner phase ----------------------------------------------------------------------------
        // (Speculative descent — a lane that reaches a leaf puts it aside once and keeps descending — was measured
        // slower on an earlier GPU and removed: the steps taken before tmax shrinks cost more than the idle lanes they fill.)
        if (has_ray) {
            uint32_t budget = inner_budget;
            while (index_count(top) == 0 && budget != 0) {
                --budget;
                uint32_t w[16];
                {
                    uint32_t w0[8], w1[8];
                    const WideNode* node = a.wide + (top >> kPrimCountBits);
                    ldg256(node, w0);                       // (allocating: a wide node serves four children)
                    ldg256(reinterpret_cast<const unsigned char*>(node) + 32, w1);
                    #pragma unroll
                    for (int k = 0; k < 8; ++k) { w[k] = w0[k]; w[8 + k] = w1[k]; }
                }
                if (!wide_step<kAny>(w, r, top, stack)) { has_ray = false; break; }
            }
            if (!has_ray) retire(ray_index, hit, tmax_in);
        }
        __syncwarp();

        // ---- leaf phase -----------------------------------------------------------------------------
        if (has_ray && index_count(top) != 0) {
            leaf_step<float>(a.tris, a.prim_ids, true, top, r, hit, nullptr);
            if ((kAny && hit.slot != kInvalidId) || !stack.try_pop(top)) {
                retire(ray_index, hit, tmax_in);
                has_ray = false;
            }
        }
        __syncwarp();
        if (kGather) stager_account(stager, a.hits, lane);
    }
    if (kGather && stager.buf && lane == 0) bulk_wait_all();
}


// ---- ray reordering (BVH_SORT_RAYS) ---------------------------------------------------------------------------
// Incoherent batches (ambient occlusion, diffuse bounces) arrive in an order unrelated to space: the 32 rays of a
// warp start in 32 different places, every node fetch is its own cache line and the lanes never agree on a branch.
// With this flag the batch is traversed in the Morton order of the ray ORIGINS: one kernel computes 30-bit keys
// against the root box (counting the radix digits on the way), the one-sweep radix sort of the build
// (radix_sort.cuh) orders ray indices by key, and the persistent kernels draw ray order[p] at position p.  Rays are
// not moved (a 32-byte ray is one sector wherever it lies) and every hit record goes to its ray's own slot, so the
// caller sees the same result in the same place.
template <typename T>
__global__ void __launch_bounds__(256)
ray_key_kernel(const DevRay<T>* __restrict__ rays, uint32_t n, const DevNode<T>* __restrict__ nodes,
               uint32_t* __restrict__ keys, uint32_t* __restrict__ digit_totals) {
    __shared__ uint32_t digit_hist[4 * 256];
    for (int k = threadIdx.x; k < 4 * 256; k += 256) digit_hist[k] = 0;
    __syncthreads();
    const DevNode<T> root = nodes[1];
    float lo[3], scale[3];
    #pragma unroll
    for (int k = 0; k < 3; ++k) {
        lo[k] = (float)root.bounds[2 * k];
        const float extent = (float)root.bounds[2 * k + 1] - lo[k];
        scale[k] = extent > 0.f ? 1024.f / extent : 0.f;
    }
    for (uint32_t i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
        uint32_t q[3];
        #pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float c = ((float)rays[i].org[k] - lo[k]) * scale[k];
            q[k] = c > 0.f ? (c < 1023.f ? (uint32_t)c : 1023u) : 0u;           // (a NaN origin lands in cell 0)
        }
        const uint32_t key = MortonTraits<uint32_t>::encode(q[0], q[1], q[2]);
        keys[i] = key;
        #pragma unroll
        for (int pass = 0; pass < 4; ++pass) atomicAdd(&digit_hist[pass * 256 + ((key >> (8 * pass)) & 255u)], 1u);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < 4 * 256; k += 256) { const uint32_t c = digit_hist[k]; if (c) atomicAdd(digit_totals + k, c); }
}

// Scratch of one reordered call (freed, stream-ordered, when the call has been enqueued).
struct RayOrderScratch {
    cudaStream_t stream;
    void* ptrs[5] = { nullptr, nullptr, nullptr, nullptr, nullptr };
    explicit RayOrderScratch(cudaStream_t s) : stream(s) {}
    ~RayOrderScratch() { for (void* p : ptrs) device_free(p, stream); }
};

template <typename T>
int make_ray_order(const DeviceBvh<T>& bvh, const DevRay<T>* d_rays, uint32_t n, RayOrderScratch& scratch, const uint32_t** order, cudaStream_t stream) {
    const size_t words = onesweep_state_words(n, 4);
    for (int k = 0; k < 4; ++k) if (device_alloc(&scratch.ptrs[k], (size_t)n * sizeof(uint32_t), stream)) return -1;
    if (device_alloc(&scratch.ptrs[4], words * sizeof(uint32_t), stream)) return -1;
    uint32_t* keys_a = static_cast<uint32_t*>(scratch.ptrs[0]); uint32_t* keys_b = static_cast<uint32_t*>(scratch.ptrs[1]);
    uint32_t* vals_a = static_cast<uint32_t*>(scratch.ptrs[2]); uint32_t* vals_b = static_cast<uint32_t*>(scratch.ptrs[3]);
    uint32_t* state = static_cast<uint32_t*>(scratch.ptrs[4]);
    BVH_CUDA_TRY(cudaMemsetAsync(state, 0, words * sizeof(uint32_t), stream));
    int sm_count = 132;
    BVH_CUDA_TRY(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, bvh.device));
    const uint32_t want = (n + 255) / 256, cap = (uint32_t)sm_count * 4;
    ray_key_kernel<T><<<want < cap ? want : cap, 256, 0, stream>>>(d_rays, n, bvh.nodes, keys_a, state + 64);
    BVH_CUDA_TRY(radix_sort_onesweep<uint32_t>(keys_a, vals_a, keys_b, vals_b, state, n, 30, stream));
    *order = vals_a;                                          // four passes: the result is back in buffer A
    // (a timed-out look-back leaves a wrong but in-range order only if it also leaves duplicates; the kernels index
    // rays[order[p]] with order values < n in either case because vals start as the identity permutation)
    return 0;
}

template <typename KernelT>
int configure_smem(KernelT kernel, size_t smem_bytes) {
    if (smem_bytes > 48 * 1024)
        BVH_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    return 0;
}

// One resident wave of persistent CTAs (SM count x occupancy), never more than the batch can feed.
template <typename KernelT, typename T>
int launch_persistent(KernelT kernel, const TraceArgs<T>& args, size_t smem, unsigned rays_per_warp, int device, cudaStream_t stream) {
    if (smem > 200 * 1024) { set_error("trace: tree too deep for the shared-memory stack"); return -1; }
    if (configure_smem(kernel, smem)) return -1;
    if (const int carve = tunables().smem_carveout.load(); carve >= 0)
        BVH_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
    int sm_count = 132, per_sm = 1;
    BVH_CUDA_TRY(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device));
    BVH_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kTraceBlock, smem));
    if (per_sm < 1) per_sm = 1;
    unsigned long long grid = (unsigned long long)sm_count * per_sm;
    const unsigned long long max_useful = (args.n + rays_per_warp - 1) / rays_per_warp / (kTraceBlock / 32) + 1;
    if (grid > max_useful) grid = max_useful;
    BVH_CUDA_TRY(cudaMemsetAsync(args.next_ray, 0, sizeof(unsigned long long), stream));
    kernel<<<(unsigned)grid, kTraceBlock, smem, stream>>>(args);
    return 0;
}

template <typename T, bool kAny>
int launch_wide(const TraceArgs<T>& args, bool gather, int device, cudaStream_t stream) {
    if constexpr (sizeof(T) == 4) {
        const size_t smem = (size_t)args.wide_entries * kTraceBlock * sizeof(uint32_t);
        if (gather) return launch_persistent(trace_wide_kernel<kAny, true>, args, smem + stage_smem_bytes<T>(), 32, device, stream);
        return launch_persistent(trace_wide_kernel<kAny, false>, args, smem, 32, device, stream);
    } else {
        set_error("trace: the wide kernel is float-only");
        return -1;
    }
}

template <typename T, bool kAny, bool kRobust>
int launch(const TraceArgs<T>& args, bool simple, bool stats, bool gather, int device, cudaStream_t stream) {
    using U = typename Real<T>::UInt;
    const size_t smem = (size_t)args.stack_entries * kTraceBlock * sizeof(U);
    if (smem > 200 * 1024) { set_error("trace: tree too deep for the shared-memory stack"); return -1; }
    if (stats || simple) {
        const unsigned long long blocks = (args.n + kTraceBlock - 1) / kTraceBlock;
        if (blocks > 0x7FFFFFFFull) { set_error("trace: batch too large for one launch"); return -1; }
        if (stats) {
            if (configure_smem(trace_simple_kernel<T, kAny, kRobust, true>, smem)) return -1;
            trace_simple_kernel<T, kAny, kRobust, true><<<(unsigned)blocks, kTraceBlock, smem, stream>>>(args);
        } else {
            if (configure_smem(trace_simple_kernel<T, kAny, kRobust, false>, smem)) return -1;
            trace_simple_kernel<T, kAny, kRobust, false><<<(unsigned)blocks, kTraceBlock, smem, stream>>>(args);
        }
    } else if (args.variant == 3) {
        if (launch_wide<T, kAny>(args, gather, device, stream)) return -1;
    } else if (args.variant == 2) {
        if (launch_persistent(trace_pair_kernel<T, kAny, kRobust>, args, smem / 2, 16, device, stream)) return -1;   // one stack per lane pair
    } else {
        const size_t tma = args.use_tma ? tma_smem_bytes<T>() : 0, stage = gather ? stage_smem_bytes<T>() : 0;
        int rc;
        if (args.use_tma) rc = gather ? launch_persistent(trace_persistent_kernel<T, kAny, kRobust, true, true>, args, smem + tma + stage, 32, device, stream)
                                      : launch_persistent(trace_persistent_kernel<T, kAny, kRobust, true, false>, args, smem + tma, 32, device, stream);
        else              rc = gather ? launch_persistent(trace_persistent_kernel<T, kAny, kRobust, false, true>, args, smem + stage, 32, device, stream)
                                      : launch_persistent(trace_persistent_kernel<T, kAny, kRobust, false, false>, args, smem, 32, device, stream);
        if (rc) return -1;
    }
    BVH_CUDA_TRY(cudaGetLastError());
    return 0;
}

} // namespace

template <typename T>
int trace_rays(const DeviceBvh<T>& bvh, const DevRay<T>* d_rays, DevHit<T>* d_hits, size_t n,
               unsigned flags, uint32_t* d_ray_stats, cudaStream_t stream, const GatherTargets* gather) {
    if (n == 0) return 0;
    if (!bvh.nodes || !bvh.tris) { set_error("trace: the BVH has no triangles attached (bvhNN_set_triangles)"); return -1; }
    TraceArgs<T> args;
    args.nodes = bvh.nodes; args.tris = bvh.tris; args.prim_ids = bvh.prim_ids;
    args.rays = d_rays; args.n = n;
    args.hits.local = d_hits; args.hits.peer_count = 0; args.hits.multicast = nullptr;
    for (int p = 0; p < kMaxPeers; ++p) args.hits.peer[p] = nullptr;
    if (gather) {
        if (gather->count < 0 || gather->count > kMaxPeers) { set_error("trace: at most 8 gather targets"); return -1; }
        for (int p = 0; p < gather->count; ++p) args.hits.peer[p] = static_cast<DevHit<T>*>(gather->peer[p]) + gather->offset;
        args.hits.peer_count = gather->count;
        if (gather->multicast) {
            if (sizeof(T) != 4) { set_error("trace: multicast gather is float-only"); return -1; }
            args.hits.multicast = static_cast<DevHit<T>*>(gather->multicast) + gather->offset;
        }
    } else if (!d_hits) { set_error("trace: no hit array"); return -1; }
    args.ray_stats = d_ray_stats;
    args.lowest_id = (flags & kTraceLastVisited) ? 0 : 1;
    uint32_t entries = bvh.depth + 2;                           // depth + 1 pending far children at most, + the sentinel
    {                                                           // (an entry is one 512-byte row of the block: any count keeps the alignment)
        const uint32_t r = (uint32_t)tunables().stack_round.load();
        entries = (entries + r - 1u) / r * r;
    }
    if (entries < 16) entries = 16;
    args.stack_entries = entries;
    args.next_ray = nullptr;
    args.inner_budget = tunables().inner_budget.load();
    args.refill_min = tunables().refill_min.load();
    {   // a warp's private run of consecutive rays: as long as the batch allows with ~8 runs per resident warp (tail balance)
        uint32_t run = tunables().chunk_rays.load();
        int sm_count = 132;
        BVH_CUDA_TRY(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, bvh.device));
        const unsigned long long fair = n / ((unsigned long long)sm_count * 32ull * 8ull);
        if (fair < run) run = (uint32_t)fair;
        run &= ~31u;
        args.chunk_rays = run < 32u ? 32u : run;
    }
    args.watchdog = tunables().watchdog.load();
    args.full_mask = 0xFFFFFFFFu;
    args.stage_hits = tunables().gather_staging.load() != 0;
    args.variant = (flags & kTracePair) ? 2 : ((flags & (kTraceNoTma | kTraceTma)) ? 0 : tunables().variant.load());
    // the wide (compressed 4-wide) path: float, canonical tie-break, fast slab test, no statistics
    args.wide = nullptr; args.wide_entries = 0;
    if constexpr (sizeof(T) == 4) {
        const bool explicit_binary = (flags & (kTracePair | kTraceNoTma | kTraceTma | kTraceSimple)) != 0;
        const bool order_sensitive = (flags & (kTraceLastVisited | kTraceRobust)) != 0 || d_ray_stats != nullptr;
        const bool want_wide = !order_sensitive && ((flags & kTraceWide) || (!explicit_binary && (tunables().use_wide.load() > 0)));
        if (want_wide && !bvh.wide && !bvh.wide_unavailable) {      // derived on first use
            if (rebuild_wide(const_cast<DeviceBvh<T>&>(bvh), stream, true)) return -1;
        }
        if (bvh.wide && want_wide) {
            args.wide = bvh.wide;
            uint32_t e = 3 * bvh.wide_depth + 3;                // (+ the sentinel entry)
            args.wide_entries = (e + 1u) & ~1u;
            args.variant = 3;
        }
    }
    args.use_tma = (flags & kTraceTma) ? true : ((flags & kTraceNoTma) ? false : tunables().variant.load() == 1);
    const bool simple = (flags & kTraceSimple) != 0, stats = d_ray_stats != nullptr;
    if (!bvh.scratch) {
        void* p = nullptr;
        if (device_alloc(&p, 2 * sizeof(unsigned long long), stream)) return -1;
        bvh.scratch = static_cast<unsigned long long*>(p);
        BVH_CUDA_TRY(cudaMemsetAsync(bvh.scratch, 0, 2 * sizeof(unsigned long long), stream));
    }
    args.next_ray = bvh.scratch;
    args.status = reinterpret_cast<uint32_t*>(bvh.scratch + 1);
    // ray reordering: persistent kernels without bulk-copied ray chunks (a chunk is no longer contiguous); not in
    // gather mode (its staging groups are runs of consecutive ray indices), not for the diagnostic kernels
    RayOrderScratch order_scratch(stream);
    args.order = nullptr;
    if ((flags & kTraceSortRays) && !gather && !simple && !stats && args.variant != 2 && n >= (1u << 16) && n < 0xFFFFFFFFull) {
        if (make_ray_order(bvh, d_rays, (uint32_t)n, order_scratch, &args.order, stream)) return -1;
        args.use_tma = false;
    }
    int rc;
    const bool any = (flags & kTraceAnyHit) != 0, robust = (flags & kTraceRobust) != 0;
    // gather mode: the kernel variants with warp-aggregated hit stores when staging is on (one bulk copy per 32 records and
    // rank, or ONE bulk copy to the multicast address); otherwise the plain variants deliver the records with store_hit()
    // (one store per record and rank / one multimem store) and carry none of the staging code
    const bool staged = gather != nullptr && args.stage_hits;
    // refill threshold and inner budget, 0 = auto (DESIGN.md §3, measured on the H100): closest-hit rays in the binary
    // persistent kernel run best with 14 / 4; any-hit rays and the lane-pair and wide kernels with 8 / 8
    const bool closest_binary = !any && (args.variant == 0 || args.variant == 1);
    if (args.refill_min == 0) args.refill_min = closest_binary ? 14u : 8u;
    if (args.inner_budget == 0) args.inner_budget = closest_binary ? 4u : 8u;
    if (args.variant == 3) args.inner_budget = tunables().wide_budget.load();
    bvh.last_kernel = stats ? kKernelStats : simple ? kKernelSimple : args.variant == 3 ? kKernelWide : args.variant == 2 ? kKernelPair
                    : args.use_tma ? kKernelPersistentTma : kKernelPersistent;
    if (any) rc = robust ? launch<T, true, true>(args, simple, stats, staged, bvh.device, stream)
                         : launch<T, true, false>(args, simple, stats, staged, bvh.device, stream);
    else     rc = robust ? launch<T, false, true>(args, simple, stats, staged, bvh.device, stream)
                         : launch<T, false, false>(args, simple, stats, staged, bvh.device, stream);
    return rc;
}

template <typename T> int check_trace_status(const DeviceBvh<T>& bvh, cudaStream_t stream) {
    if (!bvh.scratch) { BVH_CUDA_TRY(cudaStreamSynchronize(stream)); return 0; }
    unsigned long long status = 0;
    BVH_CUDA_TRY(cudaMemcpyAsync(&status, bvh.scratch + 1, sizeof status, cudaMemcpyDeviceToHost, stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(stream));
    if (status != 0) {
        BVH_CUDA_TRY(cudaMemsetAsync(bvh.scratch + 1, 0, sizeof status, stream));
        set_error("trace: the traversal kernel's watchdog fired (a warp exceeded its round limit); results are incomplete");
        return -1;
    }
    return 0;
}
template int check_trace_status<float>(const DeviceBvh<float>&, cudaStream_t);
template int check_trace_status<double>(const DeviceBvh<double>&, cudaStream_t);

template int trace_rays<float>(const DeviceBvh<float>&, const DevRay<float>*, DevHit<float>*, size_t, unsigned, uint32_t*, cudaStream_t, const GatherTargets*);
template int trace_rays<double>(const DeviceBvh<double>&, const DevRay<double>*, DevHit<double>*, size_t, unsigned, uint32_t*, cudaStream_t, const GatherTargets*);

} // namespace bvhb200
