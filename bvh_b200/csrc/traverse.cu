// bvh_b200/csrc/traverse.cu — batched closest-hit / any-hit ray traversal kernels (sm_90a).
//
// Replaces the caller-side ray loop around Bvh::intersect (reference bvh.h:159-182 driven by
// test/benchmark.cpp:340-393 / c_api/bvh_impl.h:235-250) with kernels over a whole ray batch:
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
//   trace_wide_kernel        the same rounds (run_rounds, shared with trace_persistent_kernel) over the compressed
//                            4-wide tree of wide_bvh.cuh.
//   trace_pair_kernel        two lanes per ray, one child box each; the same ray feed, its own round loop.
//   trace_simple_kernel      one thread per ray, same stack machine; also the statistics variant that
//                            counts inner steps / leaves / triangle tests per ray (the reference's
//                            InnerFn hook, bvh.h:168) which defines the algorithmic bytes of DESIGN.md.
//
// The binary-tree kernels execute the reference's per-ray algorithm exactly (traverse_core.cuh), so on the same
// tree they visit nodes in the same order as the CPU code and produce bit-identical ids, t, u, v.
#include <cstdio>
#include <cstdlib>
#include <type_traits>

#include "build_core.cuh"
#include "engine.h"
#include "persistent_core.cuh"
#include "radix_sort.cuh"
#include "traverse_core.cuh"
#include "wide_bvh.cuh"

namespace bvhb200 {

namespace {

// (kTraceBlock, BVH_TRACE_BLOCKS and the persistent kernels' warp scheduler: persistent_core.cuh)
constexpr uint32_t kPairRunRays = 128;   // the lane-pair kernel's runs: fixed, the chunk_rays switch does not apply to it

// One ray record into registers.  kStreamed: from global memory, read once (ld.global.cs, evict-first); otherwise a plain
// load (the TMA kernel's shared-memory copy of the rays).
template <bool kStreamed, typename V> __device__ __forceinline__ V load_ray_piece(const V* p) { return kStreamed ? __ldcs(p) : *p; }
template <bool kStreamed = true>
__device__ __forceinline__ void load_ray(const DevRay<float>* p, RayCtx<float>& r) {
    const float4* q = reinterpret_cast<const float4*>(p);
    const float4 a = load_ray_piece<kStreamed>(q), b = load_ray_piece<kStreamed>(q + 1);
    r.org[0] = a.x; r.org[1] = a.y; r.org[2] = a.z; r.dir[0] = a.w;
    r.dir[1] = b.x; r.dir[2] = b.y; r.tmin = b.z; r.tmax = b.w;
}
template <bool kStreamed = true>
__device__ __forceinline__ void load_ray(const DevRay<double>* p, RayCtx<double>& r) {
    const double2* q = reinterpret_cast<const double2*>(p);
    const double2 a = load_ray_piece<kStreamed>(q), b = load_ray_piece<kStreamed>(q + 1);
    const double2 c = load_ray_piece<kStreamed>(q + 2), d = load_ray_piece<kStreamed>(q + 3);
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

// (a finished ray's record: make_record, traverse_core.cuh)

// One record to every sink with one store per sink (16-byte pieces).
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
    uint32_t inner_budget;           // persistent kernel: inner steps per lane per round (0xFFFFFFFF = unbounded)
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
    load_ray(a.rays + i, r);
    ray_prologue<T, kRobust>(r);
    HitState<T> hit { kInvalidId, r.tmax, (T)0, (T)0 };
    const T tmax_in = r.tmax;
    uint32_t stats[3] = { 0, 0, 0 };
    const U root_index = a.nodes[1].index;
    traverse_ray<T, kAny, kRobust>(a.nodes, a.tris, a.prim_ids, a.lowest_id != 0, root_index, r, hit, stack,
                                   kStats ? stats : nullptr);
    store_record_direct(a.hits, i, make_record(hit, tmax_in, a.prim_ids));
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

// One finished ray: through the warp's staging slots in gather mode, else straight to the sinks.
template <typename T, bool kGather>
__device__ __forceinline__ void retire_ray(HitStager<T>& st, const HitSinks<T>& sinks, unsigned long long i, const HitState<T>& h,
                                           T tmax, const uint32_t* __restrict__ prim_ids) {
    if (kGather) stager_retire(st, sinks, i, make_record(h, tmax, prim_ids));
    else store_record_direct(sinks, i, make_record(h, tmax, prim_ids));
}

// ---- the ray feed of the persistent kernels ------------------------------------------------------------------
// (the scheduler — claim_run, RunCursor, refill_lanes, run_rounds — is persistent_core.cuh's; the draws below add the
// TMA staging, the gather mode's staging groups and the ray reordering of the library's triangle kernels)

// One draw: the lanes of `idle` (`rank`: this lane's rank among them) take the next popc(idle) positions of the run at
// most, clipped to the batch and, in gather mode, to the staging group of 32 consecutive rays the run is in.  Claims a new
// run when the current one is used up; returns false, with `exhausted` set, when the batch has none left.  `got` is set
// when this lane drew a ray; its index (through the `order` indirection when there is one) goes to `index`, the ray to `r`.
template <typename T, bool kGather>
__device__ __forceinline__ bool draw_from_run(RunCursor& c, const TraceArgs<T>& a, uint32_t run, unsigned idle, unsigned rank,
                                              bool lane_idle, HitStager<T>& stager, unsigned lane, unsigned mask,
                                              unsigned long long& index, RayCtx<T>& r, bool& got) {
    if (c.pos == c.end) {
        const unsigned long long first = claim_run(a.next_ray, run, lane, mask);
        if (first >= a.n) { c.exhausted = true; return false; }
        c.pos = first;
        c.end = first + run < a.n ? first + run : a.n;
    }
    unsigned avail = (unsigned)(c.end - c.pos);
    const unsigned want = __popc(idle);
    if (kGather) {                                  // never draw across a staging group's boundary
        const unsigned in_group = (unsigned)(c.pos & 31ull);
        if (in_group == 0) stager_open(stager, a.hits, c.pos >> 5, avail < 32u ? avail : 32u, lane);
        if (avail > 32u - in_group) avail = 32u - in_group;
    }
    const unsigned take = want < avail ? want : avail;
    if (lane_idle && rank < take) {
        index = c.pos + rank;
        if (a.order) index = a.order[index];
        load_ray(a.rays + index, r);
        got = true;
    }
    c.pos += take;
    return true;
}

// Starts a ray a lane has just drawn: a miss at its tmax so far and, in gather mode, its staging slot.  A ray whose
// interval is a NaN can hit nothing: it retires at once as a miss and false is returned.
template <typename T, bool kGather, typename Retire>
__device__ __forceinline__ bool start_ray(const RayCtx<T>& r, HitState<T>& hit, T& tmax_in, HitStager<T>& stager,
                                          unsigned long long index, Retire&& retire) {
    tmax_in = r.tmax;
    hit.slot = kInvalidId; hit.t = r.tmax; hit.u = (T)0; hit.v = (T)0;
    if (kGather) stager.tag = stager.tag_for(index);
    if (ray_interval_is_nan(r)) { retire(); return false; }
    return true;
}

constexpr int kTmaChunkRays = 32;        // rays per bulk copy (1 KB of float rays), two buffers per warp

template <typename T> __host__ __device__ constexpr size_t tma_smem_bytes() {
    return (size_t)(kTraceBlock / 32) * 2 * kTmaChunkRays * sizeof(DevRay<T>) + (size_t)(kTraceBlock / 32) * 2 * 8;
}

// The leaf phase of the triangle kernels: the lane's leaf, then its ray retires on an any-hit hit or an empty stack.
template <typename T, bool kAny, typename U, typename Stack, typename Retire>
__device__ __forceinline__ void triangle_leaf_phase(const TraceArgs<T>& a, bool lowest_id, bool& has_ray, U& top, RayCtx<T>& r,
                                                    HitState<T>& hit, Stack& stack, Retire&& retire) {
    if (has_ray && index_count(top) != 0) {
        leaf_step<T>(a.tris, a.prim_ids, lowest_id, top, r, hit, nullptr);
        if ((kAny && hit.slot != kInvalidId) || !stack.try_pop(top)) {
            retire();
            has_ray = false;
        }
    }
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

    RunCursor run;                  // (kTma: its end is not clipped to the batch; the count of each staged chunk is)
    // kTma state (warp-uniform)
    // (kept as scalars selected by `cur`, not arrays, so that nothing is spilled to local memory)
    DevRay<T>* ray_buf0 = nullptr; DevRay<T>* ray_buf1 = nullptr;
    uint32_t bar0 = 0, bar1 = 0, phase0 = 0, phase1 = 0, count0 = 0, count1 = 0;
    unsigned long long base0 = 0, base1 = 0;
    uint32_t cur = 0, buf_pos = 0;

    auto prefetch = [&] (uint32_t b) {      // stage the next 32 rays of the warp's private run (claiming a new run when it is used up)
        if (run.pos == run.end) {
            run.pos = claim_run(a.next_ray, a.chunk_rays, lane, kFull);
            run.end = run.pos + a.chunk_rays;
        }
        const unsigned long long base = run.pos;
        run.pos += kTmaChunkRays;
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
    auto retire = [&] { retire_ray<T, kGather>(stager, a.hits, ray_index, hit, tmax_in, a.prim_ids); };

    // one draw: from the staged chunk (kTma) or straight from the run
    auto draw = [&] (unsigned idle, unsigned rank) {
        bool got = false;
        if (kTma) {
            const uint32_t cur_count = cur == 0 ? count0 : count1;
            if (cur_count == 0) { run.exhausted = true; return false; }
            const uint32_t cur_bar = cur == 0 ? bar0 : bar1, cur_phase = cur == 0 ? phase0 : phase1;
            while (!mbar_try_wait(cur_bar, cur_phase)) { }
            if (kGather && buf_pos == 0) stager_open(stager, a.hits, (cur == 0 ? base0 : base1) >> 5, cur_count, lane);
            const unsigned avail = cur_count - buf_pos, want = __popc(idle);
            const unsigned take = want < avail ? want : avail;
            if (!has_ray && rank < take) {
                ray_index = (cur == 0 ? base0 : base1) + buf_pos + rank;
                load_ray<false>((cur == 0 ? ray_buf0 : ray_buf1) + buf_pos + rank, r);
                got = true;
            }
            buf_pos += take;
            if (buf_pos == cur_count) {                    // buffer drained: re-arm it with the next chunk
                __syncwarp();
                if (cur == 0) phase0 ^= 1u; else phase1 ^= 1u;
                prefetch(cur);
                cur ^= 1u; buf_pos = 0;
            }
        } else {
            if (!draw_from_run<T, kGather>(run, a, a.chunk_rays, idle, rank, !has_ray, stager, lane, kFull, ray_index, r, got)) return false;
        }
        if (got && start_ray<T, kGather>(r, hit, tmax_in, stager, ray_index, retire)) {
            ray_prologue<T, kRobust>(r);
            top = root_index;
            stack.clear();
            has_ray = true;
        }
        return true;
    };

    // inner phase: descend until this lane holds a leaf, its ray is finished, or the step budget of this round is spent
    // (bounding the wait of lanes that already hold a leaf)
    auto inner = [&] {
        if (has_ray) {
            uint32_t budget = inner_budget;
            while (index_count(top) == 0 && budget != 0) {                     // (kTraversalDone ends it too)
                --budget;
                inner_step<T, kAny, kRobust>(a.nodes, r, top, stack);
            }
            if (top == kTraversalDone<U>) {
                retire();
                has_ray = false;
            }
        }
    };
    auto account = [&] { if (kGather) stager_account(stager, a.hits, lane); };
    auto leaf = [&] { triangle_leaf_phase<T, kAny>(a, lowest_id, has_ray, top, r, hit, stack, retire); };
    // (finish: the last bulk stores have left shared memory and landed)
    auto finish = [&] { if (kGather && stager.buf && lane == 0) bulk_wait_all(); };
    run_rounds<true>(run, has_ray, kFull, 0u, a.watchdog, a.status, kFull, a.refill_min, lt_mask, lane, draw, account, inner, leaf, finish);
}

// ---- lane-pair kernel ------------------------------------------------------------------------------
// Two adjacent lanes serve ONE ray: in an inner step lane 0 of the pair fetches and tests the left
// child, lane 1 the right child (each a 32-byte node, two 128-bit loads, both nodes from the same 64-byte block), and
// the two exchange (hit, entry distance, index) with pair-masked __ballot_sync / __shfl_xor_sync.  Why: with
// divergent rays the L1 data pipe spends one wavefront per thread per load (the one-lane-per-ray kernel was
// measured bound by l1tex__data_pipe_lsu_wavefronts at ~87 % of peak on an earlier GPU); the two lanes of a pair hit the same
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

    RunCursor run;
    HitStager<T> stager;                                               // (no gather mode: unused)

    bool has_ray = false;
    unsigned long long ray_index = 0;
    RayCtx<T> r;
    HitState<T> hit;
    T tmax_in = (T)0;
    U top = 0;
    // both lanes of a pair hold the ray; the even one stores its record
    auto retire = [&] { if (sub == 0) store_record_direct(a.hits, ray_index, make_record(hit, tmax_in, a.prim_ids)); };

    // Pairs are drawn like lanes, through the even lanes (the odd lane of a pair has its partner's rank), with no
    // refill threshold: every idle pair is refilled at once.  (Rays are never sorted for this kernel: `order` is null.)
    auto draw = [&] (unsigned idle, unsigned rank) {
        bool got = false;
        if (!draw_from_run<T, false>(run, a, kPairRunRays, idle, rank, !has_ray, stager, lane, kFull, ray_index, r, got)) return false;
        if (got && start_ray<T, false>(r, hit, tmax_in, stager, ray_index, retire)) {
            ray_prologue<T, kRobust>(r);
            top = root_index;
            stack.clear();
            has_ray = true;
        }
        return true;
    };

    // `lane_zero` is 0 for every thread (blocks have 128 threads) but not provably so: adding it keeps the
    // round counters in ordinary per-lane registers instead of a warp-uniform register shared by the warp.
    const uint32_t lane_zero = threadIdx.x >> 10;
    uint32_t rounds = lane_zero;
    for (;;) {
        if (watchdog_fired(rounds, a.watchdog, a.status, lane)) return;
        refill_lanes(has_ray, run, kEven, 0u, lt_mask, kFull, draw, [] {});
        if (__ballot_sync(kFull, has_ray) == 0u) {
            if (run.exhausted) break;
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
            if (retired) retire();
        }
        __syncwarp(kFull);

        // ---- leaf phase (both lanes of the pair run it redundantly) -------------------------------------
        if (has_ray && index_count(top) != 0) {
            leaf_step<T>(a.tris, a.prim_ids, lowest_id, top, r, hit, nullptr);
            if ((kAny && hit.slot != kInvalidId) || stack.empty()) {
                retire();
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
// fetches ONE 64-byte node (four 128-bit loads from the same line), dequantises four child boxes straight
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

    RunCursor run;
    bool has_ray = false;
    unsigned long long ray_index = 0;
    RayCtx<float> r;                   // aux = padded inverse direction (far planes)
    HitState<float> hit;
    float tmax_in = 0.f;
    uint32_t top = 0;
    auto retire = [&] { retire_ray<float, kGather>(stager, a.hits, ray_index, hit, tmax_in, a.prim_ids); };

    auto draw = [&] (unsigned idle, unsigned rank) {
        bool got = false;
        if (!draw_from_run<float, kGather>(run, a, a.chunk_rays, idle, rank, !has_ray, stager, lane, kFull, ray_index, r, got)) return false;
        if (got && start_ray<float, kGather>(r, hit, tmax_in, stager, ray_index, retire)) {
            wide_ray_setup(r);
            top = 0;                                        // wide node 0, inner
            stack.clear();
            has_ray = true;
        }
        return true;
    };

    // inner phase
    // (Speculative descent — a lane that reaches a leaf puts it aside once and keeps descending — was measured
    // slower on an earlier GPU and removed: the steps taken before tmax shrinks cost more than the idle lanes they fill.)
    auto inner = [&] {
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
            if (!has_ray) retire();
        }
    };
    // (plan_trace never chooses this kernel for BVH_TIE_LAST_VISITED: the lowest id wins ties)
    auto account = [&] { if (kGather) stager_account(stager, a.hits, lane); };
    auto leaf = [&] { triangle_leaf_phase<float, kAny>(a, true, has_ray, top, r, hit, stack, retire); };
    // (finish: the last bulk stores have left shared memory and landed)
    auto finish = [&] { if (kGather && stager.buf && lane == 0) bulk_wait_all(); };
    run_rounds<true>(run, has_ray, kFull, 0u, a.watchdog, a.status, kFull, a.refill_min, lt_mask, lane, draw, account, inner, leaf, finish);
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

// The most dynamic shared memory a trace launch may ask for (stack, TMA and staging areas together).
constexpr size_t kMaxTraceSmem = 200 * 1024;

// The kernel's dynamic shared-memory limit is a process-wide attribute of the function, not of the call: it is always
// raised to kMaxTraceSmem, never to this call's size, so that a concurrent call on a shallower tree cannot lower it
// between another thread's setting and launch.
template <typename KernelT>
int configure_smem(KernelT kernel, size_t smem_bytes) {
    if (smem_bytes > 48 * 1024)
        BVH_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxTraceSmem));
    return 0;
}

// One resident wave of persistent CTAs (SM count x occupancy), never more than the batch can feed.
template <typename KernelT, typename T>
int launch_persistent(KernelT kernel, const TraceArgs<T>& args, size_t smem, unsigned rays_per_warp, int device, cudaStream_t stream) {
    if (smem > kMaxTraceSmem) { set_error("trace: tree too deep for the shared-memory stack"); return -1; }
    if (configure_smem(kernel, smem)) return -1;
    if (const int carve = tunables().smem_carveout.load(); carve >= 0)
        BVH_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
    int sm_count = 132, per_sm = 1;
    BVH_CUDA_TRY(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device));
    BVH_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kTraceBlock, smem));
    const unsigned long long grid = persistent_grid(sm_count, per_sm, args.n, rays_per_warp, kTraceBlock / 32);
    BVH_CUDA_TRY(cudaMemsetAsync(args.next_ray, 0, sizeof(unsigned long long), stream));
    kernel<<<(unsigned)grid, kTraceBlock, smem, stream>>>(args);
    return 0;
}

// One switch over the kernel the plan chose.  staged: gather mode with warp-aggregated hit stores (one bulk copy per 32
// records and rank, or ONE to the multicast address); otherwise records leave with one store per record and sink.
template <typename T, bool kAny, bool kRobust>
int launch(TraceKernel kernel, const TraceArgs<T>& args, bool staged, int device, cudaStream_t stream) {
    using U = typename Real<T>::UInt;
    size_t smem = (size_t)args.stack_entries * kTraceBlock * sizeof(U);
    if (smem > kMaxTraceSmem) { set_error("trace: tree too deep for the shared-memory stack"); return -1; }
    const size_t stage = staged ? stage_smem_bytes<T>() : 0;
    void (*persistent)(TraceArgs<T>) = nullptr;
    unsigned rays_per_warp = 32;
    switch (kernel) {
    case kKernelSimple:
    case kKernelStats: {
        const unsigned long long blocks = (args.n + kTraceBlock - 1) / kTraceBlock;
        if (blocks > 0x7FFFFFFFull) { set_error("trace: batch too large for one launch"); return -1; }
        void (*simple)(TraceArgs<T>) = kernel == kKernelStats ? trace_simple_kernel<T, kAny, kRobust, true>
                                                              : trace_simple_kernel<T, kAny, kRobust, false>;
        if (configure_smem(simple, smem)) return -1;
        simple<<<(unsigned)blocks, kTraceBlock, smem, stream>>>(args);
        break;
    }
    case kKernelPersistent:
        persistent = staged ? trace_persistent_kernel<T, kAny, kRobust, false, true> : trace_persistent_kernel<T, kAny, kRobust, false, false>;
        smem += stage;
        break;
    case kKernelPersistentTma:
        persistent = staged ? trace_persistent_kernel<T, kAny, kRobust, true, true> : trace_persistent_kernel<T, kAny, kRobust, true, false>;
        smem += tma_smem_bytes<T>() + stage;
        break;
    case kKernelPair:
        persistent = trace_pair_kernel<T, kAny, kRobust>;
        smem /= 2;                                          // one stack per lane pair
        rays_per_warp = 16;
        break;
    case kKernelWide:
        if constexpr (sizeof(T) == 4) {
            persistent = staged ? trace_wide_kernel<kAny, true> : trace_wide_kernel<kAny, false>;
            smem = (size_t)args.wide_entries * kTraceBlock * sizeof(uint32_t) + stage;
            break;
        }
        [[fallthrough]];
    default:
        set_error("trace: no such kernel for this precision");
        return -1;
    }
    if (persistent && launch_persistent(persistent, args, smem, rays_per_warp, device, stream)) return -1;
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
    const Tunables& tun = tunables();
    TraceRequest request { flags, d_ray_stats != nullptr, sizeof(T) == 4, bvh.wide != nullptr || !bvh.wide_unavailable,
                           gather != nullptr, (unsigned long long)n, tun.variant.load(), tun.use_wide.load(),
                           tun.refill_min.load(), tun.inner_budget.load(), tun.wide_budget.load() };
    TracePlan plan = plan_trace(request);
    if (plan.kernel == kKernelWide && !bvh.wide) {              // the wide tree is derived on first use
        if (rebuild_wide(const_cast<DeviceBvh<T>&>(bvh), stream, true)) return -1;
        request.wide_tree = bvh.wide != nullptr;
        plan = plan_trace(request);
    }
    bvh.last_kernel = plan.kernel;
    args.ray_stats = d_ray_stats;
    args.lowest_id = (flags & kTraceLastVisited) ? 0 : 1;
    // (an entry is one 512-byte row of the block: any count keeps the alignment)
    args.stack_entries = stack_entries(bvh.depth, (uint32_t)tun.stack_round.load());
    args.wide = nullptr; args.wide_entries = 0;
    if (plan.kernel == kKernelWide) {
        args.wide = bvh.wide;
        const uint32_t e = 3 * bvh.wide_depth + 3;              // (+ the sentinel entry)
        args.wide_entries = (e + 1u) & ~1u;
    }
    args.inner_budget = plan.inner_budget;
    args.refill_min = plan.refill_min;
    {   // a warp's private run of consecutive rays
        int sm_count = 132;
        BVH_CUDA_TRY(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, bvh.device));
        args.chunk_rays = persistent_run_rays(tun.chunk_rays.load(), n, sm_count);
    }
    args.watchdog = tun.watchdog.load();
    args.full_mask = 0xFFFFFFFFu;
    args.stage_hits = tun.gather_staging.load() != 0;
    if (!bvh.scratch) {
        void* p = nullptr;
        if (device_alloc(&p, 2 * sizeof(unsigned long long), stream)) return -1;
        bvh.scratch = static_cast<unsigned long long*>(p);
        BVH_CUDA_TRY(cudaMemsetAsync(bvh.scratch, 0, 2 * sizeof(unsigned long long), stream));
    }
    args.next_ray = bvh.scratch;
    args.status = reinterpret_cast<uint32_t*>(bvh.scratch + 1);
    RayOrderScratch order_scratch(stream);
    args.order = nullptr;
    if (plan.sort_rays && make_ray_order(bvh, d_rays, (uint32_t)n, order_scratch, &args.order, stream)) return -1;
    const bool staged = gather != nullptr && args.stage_hits;
    if (flags & kTraceAnyHit) return (flags & kTraceRobust) ? launch<T, true, true>(plan.kernel, args, staged, bvh.device, stream)
                                                            : launch<T, true, false>(plan.kernel, args, staged, bvh.device, stream);
    return (flags & kTraceRobust) ? launch<T, false, true>(plan.kernel, args, staged, bvh.device, stream)
                                  : launch<T, false, false>(plan.kernel, args, staged, bvh.device, stream);
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
