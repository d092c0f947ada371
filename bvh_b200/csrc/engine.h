// bvh_b200/csrc/engine.h — internal host-side interface between the C ABI (c_api.cu) and the CUDA
// pipelines (lbvh_build.cu, traverse.cu).  Nothing here is exported.
#pragma once

#include <atomic>
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>
#include <string>

#include "core.cuh"

namespace bvhb200 {

struct WideNode;

// Error plumbing: every engine call returns 0 on success; the message of the last failure on the
// calling thread is kept for bvh_last_error().
void set_error(const std::string& msg);
const char* last_error();

#define BVH_CUDA_TRY(expr)                                                                   \
    do {                                                                                     \
        cudaError_t err__ = (expr);                                                          \
        if (err__ != cudaSuccess) {                                                          \
            ::bvhb200::set_error(std::string(#expr) + ": " + cudaGetErrorString(err__));     \
            return -1;                                                                       \
        }                                                                                    \
    } while (0)

// Stream-ordered allocation from the device's default memory pool (release threshold raised once
// per device so that rebuilds do not go back to the driver).
int device_alloc(void** ptr, size_t bytes, cudaStream_t stream);
void device_free(void* ptr, cudaStream_t stream);
int prepare_device(int device);

// Process-wide switches for experiments and tests; the defaults are the tuned values.  Initialised once from
// the BVH_B200_* environment variables (DESIGN.md), changed at run time with bvh_set_option — nothing on a
// call path reads the environment.
struct Tunables {
    std::atomic<int> morton_bits { 0 };         // 0: auto (63 from 2^22 primitives), 30, 63
    std::atomic<int> sah_treelets { -1 };       // -1: by quality (Medium / High), 0 / 1: forced off / on
    std::atomic<int> hierarchy { 128 };         // leaves per block of the hierarchy kernel (64 / 128 / 256), 0: global flags only
    std::atomic<int> e2e_chunks { 0 };          // chunks of the host-buffer pipeline, 0: auto
    std::atomic<int> variant { 0 };             // persistent kernel: 0 streaming ray loads, 1 ray chunks staged by bulk async copies (TMA)
    std::atomic<int> use_wide { 0 };            // 1: derive the compressed wide tree with the build and trace with it where its semantics allow
    std::atomic<uint32_t> inner_budget { 8 };   // inner steps per lane per round
    std::atomic<uint32_t> refill_min { 8 };     // persistent kernels: idle lanes a warp waits for before it draws new rays (1: at once)
    std::atomic<uint32_t> wide_budget { 4 };    // same for the wide kernel
    std::atomic<uint32_t> watchdog { 1u << 26 };
    std::atomic<uint32_t> chunk_rays { 64 };    // persistent kernels: consecutive rays a warp claims at a time (its cohorts are drawn from them)
    std::atomic<int> stack_round { 2 };         // traversal stack entries are rounded up to a multiple of this (A/B: 8)
    std::atomic<int> smem_carveout { -1 };      // persistent kernels: preferred shared-memory carve-out in percent, -1: the driver's choice
    std::atomic<int> treelet_blocks { 3 };      // treelet kernel: resident blocks per SM its registers are limited for (2 / 3 / 4)
    std::atomic<int> sort_onesweep { 1 };       // build: 1 one-sweep radix sort (one kernel per pass), 0 histogram / scan / scatter per pass
    std::atomic<int> gather_staging { 1 };      // fused gather: 1 warp-aggregated bulk stores, 0 one store per record and rank
};
Tunables& tunables();

struct BuildOptions {
    uint32_t min_leaf = 1;          // TopDownSahBuilder::Config (top_down_sah_builder.h:27-40)
    uint32_t max_leaf = 8;
    int quality = 2;                // DefaultBuilder::Quality (default_builder.h:21); see DESIGN.md
    int morton_bits = 0;            // 0 = auto, 30 or 63
    bool sah_treelets = false;      // treelet_warp.cuh: SAH rebuild of the bottom subtrees (Quality Medium / High)
};

// The device-resident BVH: reference-layout nodes (shifted by one slot, padded), BVH-order
// primitive ids and, when triangles were supplied, BVH-order precomputed triangles.
template <typename T> struct DeviceBvh {
    int device = 0;
    uint32_t prim_count = 0;
    size_t node_slots = 0;              // allocated device slots (slot 0 is padding, slot 1 the root)
    DevNode<T>* nodes = nullptr;
    uint32_t* prim_ids = nullptr;       // prim_ids[i] = original id of BVH-order primitive i
    DevTri<T>* tris = nullptr;          // nullptr until triangles are attached
    uint32_t depth = 0;                 // longest chain of inner nodes below the root (stack bound)
    bool compact = false;               // every slot 1..node_slots-1 is a live node (always true once a build / upload returned)
    // two device words owned by the traversal: [0] the persistent kernels' ray cursor, [1] a sticky status
    // word set by their watchdog (allocated on first use)
    mutable unsigned long long* scratch = nullptr;
    // compressed 4-wide companion tree for the fast traversal path (wide_bvh.cuh); float trees only
    WideNode* wide = nullptr;
    uint32_t wide_depth = 0;            // number of wide levels (bounds the fast path's stack)
    uint32_t wide_count = 0;
    bool wide_unavailable = false;      // the binary tree is too deep for the wide collapse: binary kernels only
    // provenance, reported through bvhNN_get_property
    int morton_bits = 0;                // 30 / 63; 0 when the tree was uploaded from a host mirror
    int quality = -1;                   // DefaultBuilder::Quality the build ran with (-1: not built here)
    uint32_t treelets = 0;              // subtrees rebuilt by the SAH treelet pass
    mutable int last_kernel = 0;        // TraceKernel of the most recent trace_rays call
};

enum TraceKernel : int { kKernelNone = 0, kKernelPersistentTma, kKernelPersistent, kKernelSimple, kKernelStats, kKernelPair, kKernelWide };

// (Re)derives the wide tree from the binary one, e.g. after an upload from the host mirror.
// force = false: only if the tree already has one (refresh) or the environment asks for it at build time;
// force = true: always (first use by a trace).
template <typename T> int rebuild_wide(DeviceBvh<T>& bvh, cudaStream_t stream, bool force = false);

// Reads and clears the traversal status word; returns -1 (with an error message) if a watchdog fired.
// Synchronises the stream.
template <typename T> int check_trace_status(const DeviceBvh<T>& bvh, cudaStream_t stream);

// LBVH build.  Exactly one of d_verts (n x 9) or d_bboxes (n x 6 as min3,max3) + d_centers (n x 3)
// is given; all pointers are device pointers.  With d_verts the BVH-order PrecomputedTri array is
// produced in the same pass.
template <typename T>
int build_lbvh(DeviceBvh<T>& out, const T* d_verts, const T* d_bboxes, const T* d_centers,
               uint32_t n, const BuildOptions& options, cudaStream_t stream);

// Attach triangles to a BVH that was built from boxes/centres or uploaded from a host mirror.
template <typename T>
int attach_triangles(DeviceBvh<T>& bvh, const T* d_verts, cudaStream_t stream);

// GPU refit from moved vertices (same topology, same primitive order): new leaf boxes, new BVH-order
// triangles, inner boxes recomputed bottom-up (reference Bvh::refit, bvh.h:184-218).
template <typename T>
int refit_triangles(DeviceBvh<T>& bvh, const T* d_verts, cudaStream_t stream);

// Writes the tree in the reference's own layout into device buffers the caller copies to the host: node_slots - 1
// records of Node<T,3> (7 words each) and prim_count 64-bit primitive ids.  The device tree must be dense.
template <typename T>
int export_reference_arrays(const DeviceBvh<T>& bvh, void* d_nodes_out, unsigned long long* d_ids_out, cudaStream_t stream);

template <typename T> void release(DeviceBvh<T>& bvh, cudaStream_t stream);

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

// Fused multi-GPU gather: besides (or instead of) the local hit array, every finished ray's record is
// stored at element `offset + i` of the gathered hit array of each rank — peer[] holds that array's address
// on every rank (peer-mapped device pointers, own rank included); multicast, when non-null, is the NVSwitch
// multicast alias of the same array and replaces the per-peer stores by one multimem store.
struct GatherTargets {
    void* peer[8];
    int count;
    void* multicast;
    size_t offset;
};

// Batched traversal; all pointers are device pointers.  ray_stats (nullable): n x 3 uint32
// {inner steps, leaves, triangle tests}; it selects the statistics variant of the kernel.
template <typename T>
int trace_rays(const DeviceBvh<T>& bvh, const DevRay<T>* d_rays, DevHit<T>* d_hits, size_t n,
               unsigned flags, uint32_t* d_ray_stats, cudaStream_t stream, const GatherTargets* gather = nullptr);

} // namespace bvhb200
