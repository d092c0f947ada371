// bvh_b200/csrc/lbvh_build.cu — the CUDA LBVH construction pipeline (sm_90a).
//
// Replaces DefaultBuilder<Node>::build (reference default_builder.h:33-62) and everything under it.
// Kernels, in launch order (DESIGN.md has the byte accounting):
//   K1 centre_bounds_kernel   per-primitive centre (tri.h:25) -> per-block min/max partials
//   K2 morton_kernel          final bounds reduce, grid quantisation (mini_tree_builder.h:170-183),
//                             Morton interleave (utils.h:103-120), clears the arrival flags
//   K3 radix sort             radix_sort.cuh, 3 kernels x 4 (30-bit keys) or x 8 (63-bit keys) passes
//   K4 hierarchy_thread_kernel  one thread per sorted primitive: leaf box (tri.h:24), BVH-order
//                             PrecomputedTri (tri.h:35-37), then the bottom-up pass of build_core.cuh
//                             that links parents, unions boxes (bvh.h:213-217), collapses subtrees into
//                             leaves by SAH (split_heuristic.h:30-38) and stores each node once, in its
//                             final reference-layout slot; merges inside a block's 128 leaves meet in
//                             shared memory, the rest through global arrival flags.
#include <cstdlib>
#include <string>

#include <cuda/atomic>

#include "build_core.cuh"
#include "engine.h"
#include "radix_sort.cuh"
#include "treelet_warp.cuh"
#include "wide_bvh.cuh"

namespace bvhb200 {

namespace {

constexpr int kBlock = 256;

// ---- device-side memory ordering for the bottom-up pass ---------------------------------------
// The arrival flag is exchanged with acquire-release semantics at device scope: the release half
// publishes the node record written just before, the acquire half makes the sibling's record visible
// to the second arrival.  One acq_rel atomic replaces the two __threadfence() calls of the classic
// formulation (ncu: membar was the top stall reason of this kernel).
struct DeviceSync {
    static __device__ __forceinline__ void fence() {}
    static __device__ __forceinline__ int exchange(int* p, int v) {
        cuda::atomic_ref<int, cuda::thread_scope_device> flag(*p);
        return flag.exchange(v, cuda::memory_order_acq_rel);
    }
    // read through L2 (the sibling's record was written by another SM)
    template <typename X> static __device__ __forceinline__ X load(const X* p) {
        static_assert(sizeof(X) % 16 == 0, "load granularity");
        X out;
        const uint4* s = reinterpret_cast<const uint4*>(p);
        uint4* d = reinterpret_cast<uint4*>(&out);
        #pragma unroll
        for (int k = 0; k < (int)(sizeof(X) / 16); ++k) d[k] = __ldcg(s + k);
        return out;
    }
};

template <typename T> struct MinMax3 { T mn[3], mx[3]; };

template <typename T> __device__ __forceinline__ T shfl_down(T v, int o) { return __shfl_down_sync(0xFFFFFFFFu, v, o); }

// K1.  mode 0: verts (n x 9) -> centre of each triangle; mode 1: centres given (n x 3).
template <typename T>
__global__ void __launch_bounds__(kBlock)
centre_bounds_kernel(const T* __restrict__ src, uint32_t n, int mode, MinMax3<T>* __restrict__ partials) {
    using R = Real<T>;
    T mn[3] = { R::max(), R::max(), R::max() };
    T mx[3] = { R::neg(R::max()), R::neg(R::max()), R::neg(R::max()) };       // BBox::make_empty, bbox.h:40-44
    for (uint32_t i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        T c[3];
        if (mode == 0) {
            T v[9];
            #pragma unroll
            for (int k = 0; k < 9; ++k) v[k] = __ldg(src + 9 * (size_t)i + k);
            T bmin[3], bmax[3];
            tri_bounds_center(v, bmin, bmax, c);
        } else {
            #pragma unroll
            for (int k = 0; k < 3; ++k) c[k] = __ldg(src + 3 * (size_t)i + k);
        }
        #pragma unroll
        for (int k = 0; k < 3; ++k) { mn[k] = robust_min(mn[k], c[k]); mx[k] = robust_max(mx[k], c[k]); }
    }
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        #pragma unroll
        for (int k = 0; k < 3; ++k) {
            mn[k] = robust_min(mn[k], shfl_down(mn[k], o));
            mx[k] = robust_max(mx[k], shfl_down(mx[k], o));
        }
    }
    __shared__ MinMax3<T> warp_part[kBlock / 32];
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { for (int k = 0; k < 3; ++k) { warp_part[warp].mn[k] = mn[k]; warp_part[warp].mx[k] = mx[k]; } }
    __syncthreads();
    if (threadIdx.x == 0) {
        MinMax3<T> acc = warp_part[0];
        for (int w = 1; w < kBlock / 32; ++w)
            for (int k = 0; k < 3; ++k) {
                acc.mn[k] = robust_min(acc.mn[k], warp_part[w].mn[k]);
                acc.mx[k] = robust_max(acc.mx[k], warp_part[w].mx[k]);
            }
        partials[blockIdx.x] = acc;
    }
}

// K2.
template <typename T, typename K>
__global__ void __launch_bounds__(kBlock)
morton_kernel(const T* __restrict__ src, uint32_t n, int mode, const MinMax3<T>* __restrict__ partials,
              uint32_t num_partials, K* __restrict__ keys, int* __restrict__ flags, uint32_t* __restrict__ alive,
              uint32_t* __restrict__ digit_totals, int passes) {
    using R = Real<T>;
    __shared__ MinMax3<T> warp_part[kBlock / 32];
    __shared__ GridXform<T> xform;
    // digit histograms of every radix pass, counted while the keys are produced (radix_sort.cuh, one-sweep variant)
    __shared__ uint32_t digit_hist[8 * 256];
    if (digit_totals) for (int k = threadIdx.x; k < passes * 256; k += kBlock) digit_hist[k] = 0;
    {
        T mn[3] = { R::max(), R::max(), R::max() };
        T mx[3] = { R::neg(R::max()), R::neg(R::max()), R::neg(R::max()) };
        for (uint32_t i = threadIdx.x; i < num_partials; i += kBlock) {
            const MinMax3<T> p = partials[i];
            #pragma unroll
            for (int k = 0; k < 3; ++k) { mn[k] = robust_min(mn[k], p.mn[k]); mx[k] = robust_max(mx[k], p.mx[k]); }
        }
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            #pragma unroll
            for (int k = 0; k < 3; ++k) {
                mn[k] = robust_min(mn[k], shfl_down(mn[k], o));
                mx[k] = robust_max(mx[k], shfl_down(mx[k], o));
            }
        }
        const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        if (lane == 0) { for (int k = 0; k < 3; ++k) { warp_part[warp].mn[k] = mn[k]; warp_part[warp].mx[k] = mx[k]; } }
        __syncthreads();
        if (threadIdx.x == 0) {
            MinMax3<T> acc = warp_part[0];
            for (int w = 1; w < kBlock / 32; ++w)
                for (int k = 0; k < 3; ++k) {
                    acc.mn[k] = robust_min(acc.mn[k], warp_part[w].mn[k]);
                    acc.mx[k] = robust_max(acc.mx[k], warp_part[w].mx[k]);
                }
            xform = make_grid_xform(acc.mn, acc.mx, MortonTraits<K>::bits_per_axis);
        }
        __syncthreads();
    }
    const GridXform<T> g = xform;
    for (uint32_t i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        T c[3];
        if (mode == 0) {
            T v[9];
            #pragma unroll
            for (int k = 0; k < 9; ++k) v[k] = __ldg(src + 9 * (size_t)i + k);
            T bmin[3], bmax[3];
            tri_bounds_center(v, bmin, bmax, c);
        } else {
            #pragma unroll
            for (int k = 0; k < 3; ++k) c[k] = __ldg(src + 3 * (size_t)i + k);
        }
        const K key = morton_key<T, K>(c, g);
        keys[i] = key;
        if (i + 1 < n) { flags[i] = -1; alive[i] = 1u; }
        if (digit_totals) for (int pass = 0; pass < passes; ++pass) atomicAdd(&digit_hist[pass * 256 + ((uint32_t)(key >> (8 * pass)) & 255u)], 1u);
    }
    if (digit_totals) {
        __syncthreads();
        for (int k = threadIdx.x; k < passes * 256; k += kBlock) { const uint32_t c = digit_hist[k]; if (c) atomicAdd(digit_totals + k, c); }
    }
}

// Shared-memory meeting point of the block-local phase: plain shared accesses ordered by block-scope fences
// around a shared-memory exchange (nobody ever waits, so divergent lanes of one warp cannot deadlock).
struct BlockSync {
    static __device__ __forceinline__ void fence() { __threadfence_block(); }
    static __device__ __forceinline__ int exchange(int* p, int v) { return atomicExch(p, v); }
};

// K4.  leaf_mode 0: verts (n x 9), also writes BVH-order triangles; 1: bboxes (n x 6, min3 max3).
// Leaf stage shared by the hierarchy kernel variants: the leaf's box (and its BVH-order triangle record).
template <typename T>
__device__ __forceinline__ void hierarchy_leaf(uint32_t i, const uint32_t* __restrict__ vals, const T* __restrict__ leaf_src,
                                               int leaf_mode, DevTri<T>* __restrict__ tris, T bmin[3], T bmax[3]) {
    const uint32_t id = vals[i];
    if (leaf_mode == 0) {
        T v[9];
        #pragma unroll
        for (int k = 0; k < 9; ++k) v[k] = __ldg(leaf_src + 9 * (size_t)id + k);
        T c[3];
        tri_bounds_center(v, bmin, bmax, c);
        const DevTri<T> tri = precompute_tri(v);
        const uint4* s = reinterpret_cast<const uint4*>(&tri);
        uint4* d = reinterpret_cast<uint4*>(tris + i);
        #pragma unroll
        for (int k = 0; k < (int)(sizeof(DevTri<T>) / 16); ++k) d[k] = s[k];
    } else {
        #pragma unroll
        for (int k = 0; k < 3; ++k) {
            bmin[k] = __ldg(leaf_src + 6 * (size_t)id + k);
            bmax[k] = __ldg(leaf_src + 6 * (size_t)id + 3 + k);
        }
    }
}

// Variant G: one thread per leaf, every merge through the global arrival flags.
template <typename T, typename K>
__global__ void __launch_bounds__(kBlock)
hierarchy_global_kernel(BuildParams<T> p, const K* __restrict__ keys, const uint32_t* __restrict__ vals,
                        const T* __restrict__ leaf_src, int leaf_mode, DevTri<T>* __restrict__ tris) {
    const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
    if (i >= p.n) return;
    T bmin[3], bmax[3];
    hierarchy_leaf(i, vals, leaf_src, leaf_mode, tris, bmin, bmax);
    build_bottom_up<T, K, DeviceSync>(p, keys, i, bmin, bmax);
}

// Variant T: one thread per leaf; merges whose two children lie inside the block's B consecutive leaves meet
// in shared memory; after one block barrier, whatever reached a block wall or was not matched locally carries
// on through the global arrival flags.
template <typename T, typename K, int B>
__global__ void __launch_bounds__(B)
hierarchy_thread_kernel(BuildParams<T> p, const K* __restrict__ keys, const uint32_t* __restrict__ vals,
                        const T* __restrict__ leaf_src, int leaf_mode, DevTri<T>* __restrict__ tris) {
    __shared__ DevNode<T> s_nodes[2 * B];
    __shared__ int s_flags[B];
    __shared__ int s_info[B];
    const uint32_t t = threadIdx.x;
    const uint32_t i0 = blockIdx.x * B;
    const uint32_t iend = min(i0 + (uint32_t)B, p.n);
    const uint32_t i = i0 + t;
    const bool active = i < p.n;
    s_flags[t] = -1;
    s_info[t] = 0;
    T bmin[3], bmax[3];
    if (active) hierarchy_leaf(i, vals, leaf_src, leaf_mode, tris, bmin, bmax);
    if (p.n == 1) {
        if (active) build_bottom_up<T, K, DeviceSync>(p, keys, i, bmin, bmax);
        return;
    }
    __syncthreads();
    const LocalSlots<T> loc { s_nodes, s_flags, s_info };
    ClimbState<T> st;
    uint32_t parent = 0, side = 0;
    int outcome = kStepRetired;
    if (active) {
        climb_init(st, i, bmin, bmax);
        do outcome = local_step<T, K, BlockSync>(p, keys, st, loc, i0, iend, parent, side); while (outcome == kStepCarry);
    }
    __syncthreads();
    if (!active) return;
    if (outcome == kStepRetired && (parent < i0 || s_info[parent - i0] != 0)) return;     // matched, or the root
    climb_global<T, K, DeviceSync>(p, keys, st, parent, side, published_record(st));
}

// Variant selection.  The pass is bound by the dependent chain of the top levels and the vertex gather of the leaf
// stage, which all variants share, so they differ little; thread128 is the default (not re-measured on the H100).
// BVH_B200_HIERARCHY=global|thread64|thread128|thread256 overrides the default for experiments; all variants
// build the same tree (tests/test_host_emulation.py::test_block_local_phase_builds_the_same_tree).
template <typename T, typename K>
void launch_hierarchy(const BuildParams<T>& p, const K* keys, const uint32_t* vals, const T* leaf_src, int mode,
                      DevTri<T>* tris, cudaStream_t stream) {
    const int v = tunables().hierarchy.load();
    const uint32_t n = p.n;
#define BVH_LAUNCH_H(B) hierarchy_thread_kernel<T, K, B><<<(n + B - 1) / B, B, 0, stream>>>(p, keys, vals, leaf_src, mode, tris)
    if (v == 0) hierarchy_global_kernel<T, K><<<(n + kBlock - 1) / kBlock, kBlock, 0, stream>>>(p, keys, vals, leaf_src, mode, tris);
    else if (v == 64) BVH_LAUNCH_H(64);
    else if (v == 256 && sizeof(T) == 4) BVH_LAUNCH_H((sizeof(T) == 4 ? 256 : 128));
    else BVH_LAUNCH_H(128);
#undef BVH_LAUNCH_H
}

// ---- second pass of Quality Medium / High: SAH rebuild of the bottom subtrees (treelet_warp.cuh) ------------
// The treelets were listed by the hierarchy kernel (build_core.cuh merge_into_parent).  One WARP per treelet:
// warps claim list entries from a global cursor (treelets differ in size); the working set of a treelet is in the
// warp's registers plus a 3.3 KB (float) slice of the block's shared memory.
constexpr int kTreeletWarps = 8;

// kMinBlocks: resident blocks per SM the register allocation is held to (float: 2 -> 109 registers, 3 -> 77, 4 -> 64
// with a 32-byte spill; ncu of the 2-block build: 24 % of the warp slots active, stalls dominated by fixed-latency
// dependencies, i.e. too few warps to hide them).
template <typename T, int kMinBlocks>
__global__ void __launch_bounds__(kTreeletWarps * 32, kMinBlocks)
treelet_kernel(const Treelet* __restrict__ list, const uint32_t* __restrict__ list_count, uint32_t* __restrict__ cursor,
               DevNode<T>* __restrict__ nodes, uint32_t* __restrict__ prim_ids, DevTri<T>* __restrict__ tris,
               const T* __restrict__ leaf_src, const T* __restrict__ centre_src, int leaf_mode, uint32_t min_leaf,
               uint32_t max_leaf, uint32_t* __restrict__ info, uint32_t* __restrict__ alive) {
    __shared__ TreeletShared<T> shared[kTreeletWarps];
    TreeletShared<T>& mine = shared[threadIdx.x >> 5];
    const uint32_t count = *list_count, lbvh_depth = info[0];
    for (;;) {
        uint32_t i = 0;
        if ((threadIdx.x & 31u) == 0) i = atomicAdd(cursor, 1u);
        i = __shfl_sync(0xFFFFFFFFu, i, 0);
        if (i >= count) break;
        treelet_rebuild<T, DeviceLanes>(mine, list[i], nodes, prim_ids, tris, leaf_src, centre_src, leaf_mode, min_leaf, max_leaf, info, lbvh_depth, alive);
    }
}

// ---- compaction of the node array ---------------------------------------------------------------------------
// The bottom-up pass numbers the sibling pairs by split position (pair p at reference indices 2p+1, 2p+2) and
// leaves dead pairs behind: the descendants of every subtree the SAH rule collapsed into a leaf, and the pairs a
// rebuilt treelet no longer uses.  This pass keeps the live pairs, in the same (Morton) order: pair p moves to
// pair rank(p) = number of live pairs before it, child references are renumbered, the spare word is cleared.
// The result is the reference's dense array (every node reachable, bvh.h:17-23) shifted by one slot: what the
// traversal reads (half the footprint, neighbouring lines hold neighbouring subtrees), what refit walks and what
// the host mirror receives with one copy.  Three small kernels: live pairs per tile, scan of the tile counts,
// ranks + scatter.
constexpr int kCompactItems = 8;
constexpr int kCompactTile = kBlock * kCompactItems;                // 2048 pairs per block

__global__ void __launch_bounds__(kBlock)
compact_count_kernel(const uint32_t* __restrict__ alive, uint32_t pairs, uint32_t* __restrict__ tile_counts) {
    __shared__ uint32_t warp_sums[kBlock / 32];
    uint32_t local = 0;
    const uint32_t base = blockIdx.x * (uint32_t)kCompactTile;
    #pragma unroll
    for (int k = 0; k < kCompactItems; ++k) {
        const uint32_t i = base + k * kBlock + threadIdx.x;
        if (i < pairs) local += alive[i];
    }
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_down_sync(0xFFFFFFFFu, local, o);
    if ((threadIdx.x & 31u) == 0) warp_sums[threadIdx.x >> 5] = local;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t total = 0;
        for (int w = 0; w < kBlock / 32; ++w) total += warp_sums[w];
        tile_counts[blockIdx.x] = total;
    }
}

// One block: exclusive scan of the tile counts in place; the total goes to info[3].
__global__ void __launch_bounds__(1024)
compact_scan_kernel(uint32_t* __restrict__ tile_counts, uint32_t tiles, uint32_t* __restrict__ info) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    for (uint32_t base = 0; base < tiles; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < tiles ? tile_counts[i] : 0u;
        uint32_t incl = v;
        #pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= (unsigned)o) incl += x; }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const uint32_t w = warp_sums[lane];
            uint32_t wi = w;
            #pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, wi, o); if (lane >= (unsigned)o) wi += x; }
            warp_sums[lane] = wi - w;                                // exclusive over the warps
        }
        __syncthreads();
        const uint32_t before = carry + warp_sums[warp] + incl - v;
        if (i < tiles) tile_counts[i] = before;
        __syncthreads();
        if (threadIdx.x == 1023) carry = before + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) info[3] = carry;
}

// rank[p] = number of live pairs before p (written for every p: the scatter below looks up its children's).
__global__ void __launch_bounds__(kBlock)
compact_rank_kernel(const uint32_t* __restrict__ alive, uint32_t pairs, const uint32_t* __restrict__ tile_offsets,
                    uint32_t* __restrict__ rank) {
    __shared__ uint32_t warp_sums[kBlock / 32];
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    // thread t owns kCompactItems CONSECUTIVE pairs, so that its local prefix is a plain running sum
    const uint32_t first = blockIdx.x * (uint32_t)kCompactTile + threadIdx.x * kCompactItems;
    uint32_t a[kCompactItems], local = 0;
    #pragma unroll
    for (int k = 0; k < kCompactItems; ++k) { a[k] = first + k < pairs ? alive[first + k] : 0u; local += a[k]; }
    uint32_t incl = local;
    #pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= (unsigned)o) incl += x; }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    uint32_t before = tile_offsets[blockIdx.x] + incl - local;
    for (unsigned w = 0; w < warp; ++w) before += warp_sums[w];
    #pragma unroll
    for (int k = 0; k < kCompactItems; ++k) { if (first + k < pairs) rank[first + k] = before; before += a[k]; }
}

template <typename T>
__global__ void __launch_bounds__(kBlock)
compact_scatter_kernel(const DevNode<T>* __restrict__ src, DevNode<T>* __restrict__ dst, const uint32_t* __restrict__ alive,
                       const uint32_t* __restrict__ rank, uint32_t pairs) {
    const uint32_t p = blockIdx.x * kBlock + threadIdx.x;
    if (p == 0) {                                                    // slot 0 is padding, slot 1 the root
        DevNode<T> zero;
        for (int k = 0; k < 6; ++k) zero.bounds[k] = (T)0;
        zero.index = 0; zero.pad = 0;
        dst[0] = zero;
        dst[1] = compact_remap(src[1], rank);
    }
    if (p >= pairs || alive[p] == 0u) return;
    const size_t from = child_slot(p, 0), to = child_slot(rank[p], 0);
    const DevNode<T> left = compact_remap(src[from], rank), right = compact_remap(src[from + 1], rank);
    const uint4* l4 = reinterpret_cast<const uint4*>(&left);
    const uint4* r4 = reinterpret_cast<const uint4*>(&right);
    uint4* d = reinterpret_cast<uint4*>(dst + to);
    constexpr int kParts = (int)(sizeof(DevNode<T>) / 16);
    #pragma unroll
    for (int k = 0; k < kParts; ++k) { d[k] = l4[k]; d[kParts + k] = r4[k]; }
}

// ---- export to the reference's layout (host mirror) ---------------------------------------------------------
// The dense device array is the reference's node array shifted by one slot and padded by one word per node; this
// writes the reference's own records (Node<T,3>: six bounds + index, 7 words of 4 / 8 bytes, node.h:31-37) and
// size_t primitive ids (bvh.h:22), one word per thread (coalesced), ready for ONE device-to-host copy each.
template <typename T>
__global__ void __launch_bounds__(kBlock)
export_nodes_kernel(const DevNode<T>* __restrict__ nodes, size_t node_count, typename Real<T>::UInt* __restrict__ out) {
    using U = typename Real<T>::UInt;
    const size_t w = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (w >= node_count * 7) return;
    const size_t node = w / 7, k = w - node * 7;
    out[w] = reinterpret_cast<const U*>(nodes + node + 1)[k];
}
__global__ void __launch_bounds__(kBlock)
export_ids_kernel(const uint32_t* __restrict__ ids, size_t n, unsigned long long* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (i < n) out[i] = ids[i];
}

template <typename T>
__global__ void __launch_bounds__(kBlock)
permute_tris_kernel(const T* __restrict__ verts, const uint32_t* __restrict__ prim_ids, uint32_t n,
                    DevTri<T>* __restrict__ tris) {
    const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
    if (i >= n) return;
    const uint32_t id = prim_ids[i];
    T v[9];
    #pragma unroll
    for (int k = 0; k < 9; ++k) v[k] = __ldg(verts + 9 * (size_t)id + k);
    const DevTri<T> t = precompute_tri(v);
    const uint4* s = reinterpret_cast<const uint4*>(&t);
    uint4* d = reinterpret_cast<uint4*>(tris + i);
    #pragma unroll
    for (int k = 0; k < (int)(sizeof(DevTri<T>) / 16); ++k) d[k] = s[k];
}

// ---- GPU refit (reference Bvh::refit, bvh.h:184-218, with the leaf function recomputing the leaf
// boxes from moved vertices — what an animation loop does every frame) ----------------------------------
// K_r1: parent[child slot] = parent slot, for every inner node.
template <typename T>
__global__ void __launch_bounds__(kBlock)
refit_parents_kernel(const DevNode<T>* __restrict__ nodes, size_t slots, uint32_t* __restrict__ parent, int* __restrict__ flags) {
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x + 1;
    if (i >= slots) return;
    flags[i] = 0;
    const auto index = nodes[i].index;
    if (index_count(index) == 0) {
        const size_t first = (size_t)index_first(index) + 1;          // device slot of the left child
        if (first + 1 < slots) { parent[first] = (uint32_t)i; parent[first + 1] = (uint32_t)i; }
    }
    if (i == 1) parent[1] = 0;
}

// K_r2: one thread per leaf slot: box of its triangles (tri.h:24, in BVH order), BVH-order PrecomputedTri
// (tri.h:35-37), then climb; the second child to arrive unions the two boxes in the reference's order
// (left.get_bbox().extend(right.get_bbox()), bvh.h:213-217).
template <typename T>
__global__ void __launch_bounds__(kBlock)
refit_leaves_kernel(DevNode<T>* __restrict__ nodes, size_t slots, const uint32_t* __restrict__ parent, int* __restrict__ flags,
                    const T* __restrict__ verts, const uint32_t* __restrict__ prim_ids, DevTri<T>* __restrict__ tris) {
    using R = Real<T>;
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x + 1;
    if (i >= slots) return;
    const auto index = nodes[i].index;
    const uint32_t count = index_count(index);
    if (count == 0) return;
    const uint32_t first = (uint32_t)index_first(index);
    T bmin[3] = { R::max(), R::max(), R::max() };
    T bmax[3] = { R::neg(R::max()), R::neg(R::max()), R::neg(R::max()) };
    for (uint32_t k = first; k < first + count; ++k) {
        const uint32_t id = prim_ids[k];
        T v[9];
        #pragma unroll
        for (int j = 0; j < 9; ++j) v[j] = __ldg(verts + 9 * (size_t)id + j);
        T tmin[3], tmax[3], c[3];
        tri_bounds_center(v, tmin, tmax, c);
        #pragma unroll
        for (int a = 0; a < 3; ++a) { bmin[a] = robust_min(bmin[a], tmin[a]); bmax[a] = robust_max(bmax[a], tmax[a]); }
        const DevTri<T> t = precompute_tri(v);
        const uint4* s = reinterpret_cast<const uint4*>(&t);
        uint4* d = reinterpret_cast<uint4*>(tris + k);
        #pragma unroll
        for (int j = 0; j < (int)(sizeof(DevTri<T>) / 16); ++j) d[j] = s[j];
    }
    write_node(nodes + i, bmin, bmax, index);
    size_t node = i;
    while (node != 1) {
        const size_t p = parent[node];
        if (p == 0) return;                                            // dead slot (collapsed subtree)
        cuda::atomic_ref<int, cuda::thread_scope_device> flag(flags[p]);
        if (flag.fetch_add(1, cuda::memory_order_acq_rel) == 0) return; // the sibling will carry on
        const size_t left = (size_t)index_first(nodes[p].index) + 1;
        const DevNode<T> l = DeviceSync::load(nodes + left), r = DeviceSync::load(nodes + left + 1);
        T pmin[3], pmax[3];
        #pragma unroll
        for (int a = 0; a < 3; ++a) {
            pmin[a] = robust_min(l.bounds[2 * a], r.bounds[2 * a]);
            pmax[a] = robust_max(l.bounds[2 * a + 1], r.bounds[2 * a + 1]);
        }
        write_node(nodes + p, pmin, pmax, nodes[p].index);
        node = p;
    }
}

// ---- collapse of the binary tree into the compressed 4-wide tree (wide_bvh.cuh) ------------------------
// Level-synchronous: the frontier of level L holds (device slot of a binary inner node, index of the wide
// node that represents it).  Each item gathers the node's two children, replaces the larger-area inner
// ones by their own children until four slots are filled, quantises the slot boxes against their union
// and appends the inner slots to the frontier of level L+1.  counters[0] = next free wide node,
// counters[1 + L] = size of frontier L, counters[63] = number of non-empty levels.
constexpr int kWideMaxLevels = 60;

__global__ void __launch_bounds__(kBlock)
wide_collapse_kernel(const DevNode<float>* __restrict__ nodes, WideNode* __restrict__ wide,
                     const uint2* __restrict__ frontier_in, uint2* __restrict__ frontier_out,
                     uint32_t* __restrict__ counters, int level) {
    const uint32_t count = counters[1 + level];
    const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
    if (i >= count) return;
    if (i == 0) atomicMax(&counters[63], (uint32_t)level + 1);
    const uint2 item = frontier_in[i];
    uint32_t slot[4];
    const int used = wide_gather_children(nodes, item.x, slot);
    WideNode w;
    bool is_inner[4];
    wide_encode(nodes, slot, used, w, is_inner);
    for (int c = 0; c < used; ++c) {
        if (!is_inner[c]) continue;
        const uint32_t wide_index = atomicAdd(&counters[0], 1u);
        w.child[c] = wide_index << kPrimCountBits;
        frontier_out[atomicAdd(&counters[2 + level], 1u)] = make_uint2(slot[c], wide_index);
    }
    const uint4* src = reinterpret_cast<const uint4*>(&w);
    uint4* dst = reinterpret_cast<uint4*>(wide + item.y);
    #pragma unroll
    for (int k = 0; k < 4; ++k) dst[k] = src[k];
}

__global__ void wide_init_kernel(uint2* frontier, uint32_t* counters) {
    for (int k = threadIdx.x; k < 64; k += blockDim.x) counters[k] = 0;
    __syncthreads();
    if (threadIdx.x == 0) { frontier[0] = make_uint2(1u, 0u); counters[0] = 1; counters[1] = 1; }
}

// Builds (or rebuilds, after a refit) bvh.wide from the binary tree.  `levels` bounds the number of
// collapse rounds (binary depth + 1 is always enough).  Leaves the number of wide levels in counters[63]
// of the returned scratch, which the caller reads back together with its other results.
int build_wide(DeviceBvh<float>& bvh, uint32_t levels, uint32_t* d_counters, uint2* d_frontier_a, uint2* d_frontier_b,
               cudaStream_t stream) {
    const uint32_t n = bvh.prim_count;
    if (!bvh.wide && device_alloc(reinterpret_cast<void**>(&bvh.wide), (size_t)(n ? n : 1) * sizeof(WideNode), stream)) return -1;
    wide_init_kernel<<<1, 64, 0, stream>>>(d_frontier_a, d_counters);
    if (levels > (uint32_t)kWideMaxLevels) levels = kWideMaxLevels;
    // One launch per level.  (All levels in one cooperative launch with a grid-wide barrier per level was slower than
    // these ~25 small launches on an earlier GPU and was removed.)
    uint64_t bound = 1;
    for (uint32_t level = 0; level < levels; ++level) {
        const uint64_t items = bound < n ? bound : n;                     // frontier L has at most min(4^L, n) items
        const unsigned blocks = (unsigned)((items + kBlock - 1) / kBlock);
        wide_collapse_kernel<<<blocks, kBlock, 0, stream>>>(bvh.nodes, bvh.wide, (level & 1) ? d_frontier_b : d_frontier_a,
                                                            (level & 1) ? d_frontier_a : d_frontier_b, d_counters, (int)level);
        if (bound < n) bound *= 4;
    }
    BVH_CUDA_TRY(cudaGetLastError());
    return 0;
}
inline int build_wide(DeviceBvh<double>&, uint32_t, uint32_t*, uint2*, uint2*, cudaStream_t) { return 0; }

// The wide tree is derived lazily, the first time a trace asks for it (trace_rays), unless the
// environment asks for it at build time (experiments: BVH_B200_USE_WIDE=1 makes it the default path).
bool wide_enabled() {
    return tunables().use_wide.load() > 0;                   // 1: derive the wide tree with the build; otherwise on first use
}

struct Scratch {
    cudaStream_t stream;
    void* ptrs[16];
    int count = 0;
    explicit Scratch(cudaStream_t s) : stream(s) {}
    ~Scratch() { for (int i = 0; i < count; ++i) device_free(ptrs[i], stream); }
    template <typename X> int alloc(X** out, size_t elems) {
        void* p = nullptr;
        if (device_alloc(&p, elems * sizeof(X), stream)) return -1;
        ptrs[count++] = p;
        *out = static_cast<X*>(p);
        return 0;
    }
};

// Collapses the binary tree of `bvh` into its wide companion (float trees only) and records the wide
// depth.  Synchronises the stream.
// After the counters of a wide collapse limited to `rounds` levels came back: depth and size, or the fallback.
template <typename T> void finish_wide_tree(DeviceBvh<T>& bvh, const uint32_t (&host_counters)[64], uint32_t rounds, cudaStream_t stream) {
    bvh.wide_depth = host_counters[63];
    bvh.wide_count = host_counters[0];
    if (host_counters[1 + rounds] != 0) {
        // the collapse stopped at its level limit with nodes still waiting: their wide records were never written.
        // Such a (degenerate, very deep) tree is traced with the binary kernels only.
        device_free(bvh.wide, stream);
        bvh.wide = nullptr; bvh.wide_depth = 0; bvh.wide_count = 0;
        bvh.wide_unavailable = true;
    }
}

template <typename T> int make_wide_tree(DeviceBvh<T>& bvh, cudaStream_t stream, bool force = false) {
    if (sizeof(T) != 4 || bvh.wide_unavailable) return 0;
    if (!force && !wide_enabled() && !bvh.wide) return 0;        // not wanted yet (a stale one is always refreshed)
    Scratch scratch(stream);
    uint32_t* counters; uint2* fa; uint2* fb;
    const size_t cap = bvh.prim_count ? bvh.prim_count : 1;
    if (scratch.alloc(&counters, 64) || scratch.alloc(&fa, cap) || scratch.alloc(&fb, cap)) return -1;
    const uint32_t rounds = bvh.depth + 1 < (uint32_t)kWideMaxLevels ? bvh.depth + 1 : (uint32_t)kWideMaxLevels;
    if (build_wide(bvh, rounds, counters, fa, fb, stream)) return -1;
    uint32_t host_counters[64];
    BVH_CUDA_TRY(cudaMemcpyAsync(host_counters, counters, sizeof(host_counters), cudaMemcpyDeviceToHost, stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(stream));
    finish_wide_tree(bvh, host_counters, rounds, stream);
    return 0;
}

template <typename T, typename K>
int build_with_key(DeviceBvh<T>& out, const T* d_verts, const T* d_bboxes, const T* d_centers,
                   uint32_t n, const BuildOptions& options, int key_bits, cudaStream_t stream) {
    Scratch scratch(stream);
    const int mode = d_verts ? 0 : 1;
    const T* centre_src = d_verts ? d_verts : d_centers;
    const T* leaf_src = d_verts ? d_verts : d_bboxes;

    int sm_count = 132;
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, out.device);
    const uint32_t blocks_needed = (n + kBlock - 1) / kBlock;
    const uint32_t grid = blocks_needed < (uint32_t)(sm_count * 4) ? blocks_needed : (uint32_t)(sm_count * 4);
    const uint32_t num_tiles = (n + kRsTile - 1) / kRsTile;

    MinMax3<T>* partials; K* keys_a; K* keys_b; uint32_t* vals_b; uint32_t* tile_hist; int* flags;
    uint32_t* info; uint32_t* alive; DevNode<T>* sparse;
    if (scratch.alloc(&partials, grid) || scratch.alloc(&keys_a, n) || scratch.alloc(&keys_b, n) ||
        scratch.alloc(&vals_b, n) || scratch.alloc(&tile_hist, (size_t)num_tiles * kRsBins + kRsBins) ||
        scratch.alloc(&flags, n) || scratch.alloc(&info, 4) || scratch.alloc(&alive, n) ||
        scratch.alloc(&sparse, 2 * (size_t)n))          // slot 0 padding + 2n-1 nodes numbered by split position
        return -1;

    out.prim_count = n;
    if (device_alloc(reinterpret_cast<void**>(&out.prim_ids), (size_t)n * sizeof(uint32_t), stream)) return -1;
    if (d_verts && device_alloc(reinterpret_cast<void**>(&out.tris), (size_t)n * sizeof(DevTri<T>), stream)) return -1;

    centre_bounds_kernel<T><<<grid, kBlock, 0, stream>>>(centre_src, n, mode, partials);
    uint32_t* sort_status = nullptr;
    if (tunables().sort_onesweep.load() != 0) {
        const int passes = radix_passes(key_bits);
        uint32_t* state;
        const size_t words = onesweep_state_words(n, passes);
        if (scratch.alloc(&state, words)) return -1;
        BVH_CUDA_TRY(cudaMemsetAsync(state, 0, words * sizeof(uint32_t), stream));
        morton_kernel<T, K><<<grid, kBlock, 0, stream>>>(centre_src, n, mode, partials, grid, keys_a, flags, alive, state + 64, passes);
        BVH_CUDA_TRY(radix_sort_onesweep<K>(keys_a, out.prim_ids, keys_b, vals_b, state, n, key_bits, stream));
        sort_status = state + kOsStatusWord;
    } else {
        morton_kernel<T, K><<<grid, kBlock, 0, stream>>>(centre_src, n, mode, partials, grid, keys_a, flags, alive, nullptr, 0);
        BVH_CUDA_TRY(radix_sort_pairs<K>(keys_a, out.prim_ids, keys_b, vals_b, tile_hist, n, key_bits, stream));
    }

    BuildParams<T> p;
    p.nodes = sparse; p.flags = flags; p.info = info; p.n = n; p.alive = alive;
    p.min_leaf = options.min_leaf < 1 ? 1 : options.min_leaf;
    p.max_leaf = options.max_leaf > kMaxLeafPrims ? kMaxLeafPrims : (options.max_leaf < 1 ? 1 : options.max_leaf);
    if (p.min_leaf > p.max_leaf) p.min_leaf = p.max_leaf;
    // Quality Low: the plain LBVH (+ SAH leaf collapse); Medium / High: + SAH treelet pass
    const bool treelets = options.sah_treelets && n > 2;
    uint32_t* treelet_words = nullptr;                       // [0] list length, [1] the warps' cursor
    if (treelets) {
        Treelet* list;
        if (scratch.alloc(&list, (size_t)n / 3 + 1) || scratch.alloc(&treelet_words, 2)) return -1;
        BVH_CUDA_TRY(cudaMemsetAsync(treelet_words, 0, 2 * sizeof(uint32_t), stream));
        p.treelets = list; p.treelet_count = treelet_words; p.treelet_max = (uint32_t)TreeletCfg<T>::kMaxPrims;
    }
    BVH_CUDA_TRY(cudaMemsetAsync(info, 0, 4 * sizeof(uint32_t), stream));
    launch_hierarchy<T, K>(p, keys_a, out.prim_ids, leaf_src, mode, out.tris, stream);
    BVH_CUDA_TRY(cudaGetLastError());

    if (treelets) {
        const int blocks_wanted = sizeof(T) == 4 ? tunables().treelet_blocks.load() : 1;
        auto kernel = blocks_wanted >= 4 ? treelet_kernel<T, sizeof(T) == 4 ? 4 : 1>
                    : blocks_wanted == 3 ? treelet_kernel<T, sizeof(T) == 4 ? 3 : 1> : treelet_kernel<T, sizeof(T) == 4 ? 2 : 1>;
        int per_sm = 1;
        BVH_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kTreeletWarps * 32, 0));
        if (per_sm < 1) per_sm = 1;
        const uint32_t max_blocks = (uint32_t)(sm_count * per_sm), want = (n / 3 + kTreeletWarps) / kTreeletWarps;
        kernel<<<want < max_blocks ? want : max_blocks, kTreeletWarps * 32, 0, stream>>>(
            p.treelets, treelet_words, treelet_words + 1, sparse, out.prim_ids, out.tris, leaf_src, centre_src, mode,
            p.min_leaf, p.max_leaf, info, alive);
        BVH_CUDA_TRY(cudaGetLastError());
    }

    // compaction: live pairs only, renumbered in order (the radix sort's buffers are free again: ranks and tile
    // counts live in them)
    const uint32_t pairs = n - 1;
    uint32_t* rank = reinterpret_cast<uint32_t*>(keys_b);
    uint32_t* tile_counts = vals_b;
    if (pairs > 0) {
        const uint32_t tiles = (pairs + kCompactTile - 1) / kCompactTile;
        compact_count_kernel<<<tiles, kBlock, 0, stream>>>(alive, pairs, tile_counts);
        compact_scan_kernel<<<1, 1024, 0, stream>>>(tile_counts, tiles, info);
        compact_rank_kernel<<<tiles, kBlock, 0, stream>>>(alive, pairs, tile_counts, rank);
        BVH_CUDA_TRY(cudaGetLastError());
    }
    // The dense array is allocated for the worst case (2n slots; the live part sits at its front, so the traversal's
    // footprint is the dense one): its exact size is only known on the device, and waiting for it would put a host
    // round trip into the middle of the build.
    if (device_alloc(reinterpret_cast<void**>(&out.nodes), 2 * (size_t)n * sizeof(DevNode<T>), stream)) return -1;
    compact_scatter_kernel<T><<<(pairs + kBlock) / kBlock, kBlock, 0, stream>>>(sparse, out.nodes, alive, rank, pairs);
    BVH_CUDA_TRY(cudaGetLastError());

    // use_wide 1: the compressed 4-wide companion tree is derived in the same stream before the one host round trip
    // of the build (float trees; the level limit replaces the depth, which is still on the device)
    const bool with_wide = sizeof(T) == 4 && wide_enabled();
    uint32_t* wide_counters = nullptr;
    uint32_t host_wide[64] = {};
    if (with_wide) {
        uint2* fa; uint2* fb;
        if (scratch.alloc(&wide_counters, 64) || scratch.alloc(&fa, n) || scratch.alloc(&fb, n)) return -1;
        if (build_wide(out, (uint32_t)kWideMaxLevels, wide_counters, fa, fb, stream)) return -1;
    }

    uint32_t host_info[4] = { 0, 0, 0, 0 }, host_treelets = 0;
    BVH_CUDA_TRY(cudaMemcpyAsync(host_info, info, sizeof(host_info), cudaMemcpyDeviceToHost, stream));
    if (with_wide) BVH_CUDA_TRY(cudaMemcpyAsync(host_wide, wide_counters, sizeof(host_wide), cudaMemcpyDeviceToHost, stream));
    uint32_t host_sort_status = 0;
    if (sort_status) BVH_CUDA_TRY(cudaMemcpyAsync(&host_sort_status, sort_status, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    if (treelets) BVH_CUDA_TRY(cudaMemcpyAsync(&host_treelets, treelet_words, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(stream));
    // The depth travels through the hierarchy pass in 7 bits of the node's spare word (AuxPack).  It cannot get
    // there: distinct keys split within 63 levels, a run of equal keys is balanced by the index tie-break
    // (<= 28 more levels for 2^27 primitives).  A saturated value would under-size the traversal stacks: refuse.
    if (host_sort_status != 0) { set_error("build: the radix sort's look-back timed out (a tile never published its counts)"); return -1; }
    if (host_info[0] >= 127u) { set_error("build: tree depth exceeds what the build pass can track (127 levels)"); return -1; }
    out.depth = host_info[0] + (treelets ? host_info[2] : 0u);
    out.treelets = host_treelets;
    out.morton_bits = key_bits;
    out.quality = options.quality;
    out.node_slots = 2 * (size_t)(pairs > 0 ? host_info[3] : 0u) + 2;      // slot 0, the root, 2 x live pairs
    out.compact = true;
    if (with_wide) finish_wide_tree(out, host_wide, (uint32_t)kWideMaxLevels, stream);
    return 0;
}

} // namespace

template <typename T>
int build_lbvh(DeviceBvh<T>& out, const T* d_verts, const T* d_bboxes, const T* d_centers,
               uint32_t n, const BuildOptions& options, cudaStream_t stream) {
    if (n == 0) { set_error("build: prim_count == 0 (undefined in the reference, index.h:53)"); return -1; }
    if (!d_verts && (!d_bboxes || !d_centers)) { set_error("build: need vertices or boxes+centres"); return -1; }
    // first_id must fit Index<32,4>: 2n-1 <= 2^28-1 for float (index.h:39)
    if (sizeof(T) == 4 && 2 * (uint64_t)n > ((uint64_t)1 << 28)) { set_error("build: too many primitives for a 32-bit index"); return -1; }
    BuildOptions opts = options;
    opts.sah_treelets = options.quality >= 1;               // DefaultBuilder::Quality Medium / High (default_builder.h:21)
    const int forced_treelets = tunables().sah_treelets.load(), forced_bits = tunables().morton_bits.load();
    if (forced_treelets >= 0) opts.sah_treelets = forced_treelets != 0;                 // A/B experiments only
    int bits = options.morton_bits;
    if (forced_bits != 0) bits = forced_bits;                                           // test hook: 30 or 63
    if (bits == 0) bits = n >= (1u << 22) ? 63 : 30;
    int rc;
    if (bits <= 30) rc = build_with_key<T, uint32_t>(out, d_verts, d_bboxes, d_centers, n, opts, 30, stream);
    else            rc = build_with_key<T, uint64_t>(out, d_verts, d_bboxes, d_centers, n, opts, 63, stream);
    if (rc) release(out, stream);
    return rc;
}

template <typename T>
int attach_triangles(DeviceBvh<T>& bvh, const T* d_verts, cudaStream_t stream) {
    if (!bvh.tris && device_alloc(reinterpret_cast<void**>(&bvh.tris), (size_t)bvh.prim_count * sizeof(DevTri<T>), stream)) return -1;
    const uint32_t blocks = (bvh.prim_count + kBlock - 1) / kBlock;
    permute_tris_kernel<T><<<blocks, kBlock, 0, stream>>>(d_verts, bvh.prim_ids, bvh.prim_count, bvh.tris);
    BVH_CUDA_TRY(cudaGetLastError());
    return 0;
}

template <typename T>
int refit_triangles(DeviceBvh<T>& bvh, const T* d_verts, cudaStream_t stream) {
    if (!bvh.nodes) { set_error("refit: no BVH"); return -1; }
    if (!bvh.tris && device_alloc(reinterpret_cast<void**>(&bvh.tris), (size_t)bvh.prim_count * sizeof(DevTri<T>), stream)) return -1;
    Scratch scratch(stream);
    uint32_t* parent; int* flags;
    if (scratch.alloc(&parent, bvh.node_slots) || scratch.alloc(&flags, bvh.node_slots)) return -1;
    BVH_CUDA_TRY(cudaMemsetAsync(parent, 0, bvh.node_slots * sizeof(uint32_t), stream));
    const unsigned blocks = (unsigned)((bvh.node_slots + kBlock - 1) / kBlock);
    refit_parents_kernel<T><<<blocks, kBlock, 0, stream>>>(bvh.nodes, bvh.node_slots, parent, flags);
    refit_leaves_kernel<T><<<blocks, kBlock, 0, stream>>>(bvh.nodes, bvh.node_slots, parent, flags, d_verts, bvh.prim_ids, bvh.tris);
    BVH_CUDA_TRY(cudaGetLastError());
    return make_wide_tree(bvh, stream);
}

template <typename T>
int export_reference_arrays(const DeviceBvh<T>& bvh, void* d_nodes_out, unsigned long long* d_ids_out, cudaStream_t stream) {
    using U = typename Real<T>::UInt;
    if (!bvh.compact) { set_error("export: the device tree is not dense"); return -1; }
    const size_t node_count = bvh.node_slots - 1, words = node_count * 7;
    export_nodes_kernel<T><<<(unsigned)((words + kBlock - 1) / kBlock), kBlock, 0, stream>>>(bvh.nodes, node_count, static_cast<U*>(d_nodes_out));
    export_ids_kernel<<<(unsigned)((bvh.prim_count + kBlock - 1) / kBlock), kBlock, 0, stream>>>(bvh.prim_ids, bvh.prim_count, d_ids_out);
    BVH_CUDA_TRY(cudaGetLastError());
    return 0;
}

template <typename T> void release(DeviceBvh<T>& bvh, cudaStream_t stream) {
    device_free(bvh.nodes, stream); bvh.nodes = nullptr;
    device_free(bvh.prim_ids, stream); bvh.prim_ids = nullptr;
    device_free(bvh.tris, stream); bvh.tris = nullptr;
    device_free(bvh.scratch, stream); bvh.scratch = nullptr;
    device_free(bvh.wide, stream); bvh.wide = nullptr; bvh.wide_unavailable = false;
    bvh.prim_count = 0; bvh.node_slots = 0;
}

template int build_lbvh<float>(DeviceBvh<float>&, const float*, const float*, const float*, uint32_t, const BuildOptions&, cudaStream_t);
template int build_lbvh<double>(DeviceBvh<double>&, const double*, const double*, const double*, uint32_t, const BuildOptions&, cudaStream_t);
template int attach_triangles<float>(DeviceBvh<float>&, const float*, cudaStream_t);
template int attach_triangles<double>(DeviceBvh<double>&, const double*, cudaStream_t);
template <typename T> int rebuild_wide(DeviceBvh<T>& bvh, cudaStream_t stream, bool force) { return make_wide_tree(bvh, stream, force); }
template int rebuild_wide<float>(DeviceBvh<float>&, cudaStream_t, bool);
template int rebuild_wide<double>(DeviceBvh<double>&, cudaStream_t, bool);
template int refit_triangles<float>(DeviceBvh<float>&, const float*, cudaStream_t);
template int refit_triangles<double>(DeviceBvh<double>&, const double*, cudaStream_t);
template int export_reference_arrays<float>(const DeviceBvh<float>&, void*, unsigned long long*, cudaStream_t);
template int export_reference_arrays<double>(const DeviceBvh<double>&, void*, unsigned long long*, cudaStream_t);
template void release<float>(DeviceBvh<float>&, cudaStream_t);
template void release<double>(DeviceBvh<double>&, cudaStream_t);

} // namespace bvhb200
