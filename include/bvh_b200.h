/* include/bvh_b200.h — C ABI of the H100-native BVH engine (libbvh_c.so).
 *
 * Two groups of entry points, all `extern "C"`, plain pointers and sizes:
 *
 * 1. The reference's own C API, unchanged in name, signature and POD layout — declared in
 *    <bvh/v2/c_api/bvh.h> of this repository, which mirrors reference src/bvh/v2/c_api/bvh.h:90-295
 *    (94 symbols).  bvhNN_build runs the CUDA LBVH pipeline instead of DefaultBuilder
 *    (reference c_api/bvh_impl.h:82-116 -> default_builder.h:33-62); the thread-pool argument is
 *    accepted and ignored (CUDA streams replace ThreadPool, reference thread_pool.h:13-100).
 *
 * 2. Batched extensions (this file).  The reference traverses ONE ray per call and intersects
 *    leaf primitives through a host callback (reference c_api/bvh.h:233-295, bvh_impl.h:235-250);
 *    a device kernel cannot call a host function, so the GPU hot path needs entry points that own
 *    the triangle test.  They replace, for whole batches:
 *       caller-side Tri::get_bbox/get_center loop   reference test/benchmark.cpp:205-212, tri.h:24-25
 *       DefaultBuilder<Node>::build                 reference default_builder.h:33-62
 *       PrecomputedTri permutation                  reference test/benchmark.cpp:221-225, tri.h:35-37
 *       the per-ray loop around Bvh::intersect      reference test/benchmark.cpp:277-298,351-377,
 *                                                   bvh.h:159-182, tri.h:55-74
 *
 * Conventions: functions returning int give 0 on success and non-zero on failure, with a
 * human-readable message available from bvh_last_error() on the same thread.  There is NO CPU
 * fallback: without a CUDA device every batched entry point fails.  Pointers are host pointers
 * unless BVH_DEVICE_POINTERS is passed, in which case they are device pointers on the handle's GPU
 * and the call is asynchronous on the handle's stream (bvhNN_sync waits for it).
 */
#ifndef BVH_B200_H
#define BVH_B200_H

#include <bvh/v2/c_api/bvh.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Hit record of the batched traversal.  A miss has prim_id = all ones (BVH_INVALID_PRIM_ID
 * truncated to the field width), t = the ray's tmax and u = v = 0.  prim_id is an ORIGINAL
 * primitive index (what the reference's callers obtain through bvh.prim_ids[i],
 * test/benchmark.cpp:285); u, v are the barycentrics of PrecomputedTri::intersect (tri.h:55-74). */
struct bvh_hit3f { uint32_t prim_id; float  t, u, v; };   /* 16 bytes */
struct bvh_hit3d { uint64_t prim_id; double t, u, v; };   /* 32 bytes */

/* Per-ray traversal counters (the reference's InnerFn hook, bvh.h:168; test/benchmark.cpp:282-296) */
struct bvh_ray_stats { uint32_t inner_steps, leaves, prim_tests; };

enum bvh_intersect_flags {
    BVH_ANY_HIT          = 1u << 0,  /* Bvh::intersect<IsAnyHit = true>: stop at the first leaf that reports a hit */
    BVH_ROBUST           = 1u << 1,  /* Node::intersect_robust (node.h:68-77) instead of intersect_fast */
    BVH_TIE_LAST_VISITED = 1u << 2,  /* equal-t hits: the last one visited wins, as in the reference's example
                                        leaf loops (tri.h:69 `t <= tmax`); default is the tree-independent
                                        rule "lowest original primitive id wins" */
    BVH_DEVICE_POINTERS  = 1u << 3,  /* rays/hits/vertices are device pointers; the call is stream-ordered */
    BVH_KERNEL_SIMPLE    = 1u << 8,  /* one-thread-per-ray kernel instead of the persistent one (diagnostics) */
    /* kernel selection, for diagnostics and A/B measurements; default = the fastest measured variant */
    BVH_KERNEL_NO_TMA    = 1u << 9,  /* persistent, one lane per ray, rays read with streaming loads (the default form) */
    BVH_KERNEL_TMA       = 1u << 10, /* persistent, one lane per ray, ray chunks staged with cp.async.bulk (TMA) */
    BVH_KERNEL_PAIR      = 1u << 11, /* persistent, two lanes per ray (one child box each) */
    BVH_KERNEL_WIDE      = 1u << 12, /* persistent, compressed 4-wide tree derived from the binary one (float; canonical
                                        tie-break and fast slab test only — otherwise the binary kernels are used) */
    BVH_SORT_RAYS        = 1u << 13  /* incoherent batches: traverse the rays in the Morton order of their origins (device
                                        radix sort of ray indices, ~1 ms per 10M rays); hits[i] still answers rays[i] */
};

/* What bvhNN_get_property reports about a handle. */
enum bvh_property {
    BVH_PROP_DEPTH        = 0,  /* longest chain of inner nodes below the root (traversal stack bound) */
    BVH_PROP_NODE_SLOTS   = 1,  /* device node slots allocated (slot 0 is padding) */
    BVH_PROP_MORTON_BITS  = 2,  /* 30 or 63; 0 for a tree uploaded from the host mirror */
    BVH_PROP_QUALITY      = 3,  /* bvh_build_quality the GPU build ran with */
    BVH_PROP_TREELETS     = 4,  /* bottom subtrees rebuilt by the SAH treelet pass */
    BVH_PROP_WIDE_NODES   = 5,  /* nodes of the compressed 4-wide companion tree (0: not derived) */
    BVH_PROP_LAST_KERNEL  = 6,  /* traversal kernel of the last batched call: 1 persistent+TMA, 2 persistent,
                                   3 simple, 4 statistics, 5 lane-pair, 6 wide */
    BVH_PROP_STREAM       = 7   /* the cudaStream_t the handle's work is ordered on */
};

/* ---- runtime ------------------------------------------------------------------------------- */
BVH_API const char* bvh_last_error(void);
BVH_API int bvh_cuda_device_count(void);
/* Device used by subsequent bvhNN_build* calls on this thread (default 0). */
BVH_API int bvh_cuda_set_device(int device);
/* By default every handle owns a private non-blocking stream.  bvh_cuda_set_stream makes handles
 * created afterwards on this thread use the caller's stream instead (a cudaStream_t; NULL is the legacy
 * default stream), which lets a host framework keep all work ordered on its current stream;
 * bvh_cuda_reset_stream goes back to private streams. */
BVH_API void bvh_cuda_set_stream(void* cuda_stream);
BVH_API void bvh_cuda_reset_stream(void);
/* Pinned host memory for ray / hit buffers (so that host<->device copies run at PCIe speed). */
BVH_API void* bvh_host_alloc(size_t bytes);
BVH_API void bvh_host_free(void* ptr);
/* The library allocates device memory from a private stream-ordered pool per GPU and keeps freed blocks cached
 * in it (rebuilds never go back to the driver); this hands the cached blocks of `device` back. */
BVH_API int bvh_cuda_trim(int device);
/* Process-wide switches for experiments, A/B measurements and tests (the defaults are the measured best):
 * "morton_bits" 0|30|63, "sah_treelets" -1|0|1, "hierarchy" 0|64|128|256, "e2e_chunks", "variant" 0|1,
 * "use_wide" 0|1, "inner_budget" (unset: auto, <= 0: unbounded), "refill_min" 1..32 (idle lanes a warp waits for
 * before it draws new rays; 0: auto — 14 with inner budget 4 for closest-hit rays, 8 / 8 for any-hit rays and the wide kernel),
 * "chunk_rays" (consecutive rays a warp claims at a time), "wide_budget", "watchdog", "gather_staging" 0|1,
 * "sort_onesweep" 0|1, "treelet_blocks" 2|3|4, "stack_round", "smem_carveout" -1|0..100.  Initial values come from
 * the BVH_B200_<NAME> environment variables, read once when the library is first used; unknown names are an error. */
BVH_API int bvh_set_option(const char* name, long value);
/* Subtree reinsertion (reference ReinsertionOptimizer::optimize, reinsertion_optimizer.h:27-30,218-267) on a
 * caller-owned node array in the reference layout: node_count nodes of Node<float|double, dim> (2*dim bounds as
 * [min0,max0,...] + packed index; 20 / 28 / 40 / 56 bytes), root at 0.  This is what bvhNN_optimize runs on the
 * handle's host mirror and what bvh::v2::ReinsertionOptimizer of <bvh/v2/reinsertion_optimizer.h> calls; it is
 * host work by contract (the tree is host data) and needs no GPU.  threads = 0: all hardware threads, 1: serial. */
BVH_API int bvh_optimize_nodes(void* nodes, size_t node_count, int dim, int is_double,
                               double batch_size_ratio, size_t max_iter_count, size_t threads);

#define BVH_B200_DECLARE(T, S)                                                                          \
    /* Fused prep + build + triangle permutation from raw vertices (prim_count x 9: p0 p1 p2). */        \
    BVH_API struct bvh##S* bvh##S##_build_triangles(const T* vertices, size_t prim_count,               \
                                                    const struct bvh_build_config* config, unsigned flags); \
    /* Attach triangles (original order) to a BVH made by bvhNN_build / bvhNN_load so that it can be   \
       traced in batches; precomputes and permutes them into BVH order on the device. */                \
    BVH_API int bvh##S##_set_triangles(struct bvh##S* bvh, const T* vertices, size_t prim_count, unsigned flags); \
    /* Refit on the GPU after the vertices moved (same triangle count and order): recomputes leaf boxes,    \
       inner boxes (reference Bvh::refit, bvh.h:184-218) and the BVH-order triangles; topology unchanged. */ \
    BVH_API int bvh##S##_refit_triangles(struct bvh##S* bvh, const T* vertices, size_t prim_count, unsigned flags); \
    /* Intersect ray_count rays; hits[i] answers rays[i]. */                                            \
    BVH_API int bvh##S##_intersect_rays(struct bvh##S* bvh, const struct bvh_ray##S* rays, size_t ray_count, \
                                        struct bvh_hit##S* hits, unsigned flags);                       \
    /* Fused traversal + all-gather for a ray batch sharded over several GPUs (device pointers only, stream-  \
       ordered).  This rank traces its shard and the kernel itself stores every hit record at element         \
       `shard_offset + i` of the gathered hit array of EVERY rank: gathered_hits[r] is that array's address on  \
       rank r as mapped into this process (peer / symmetric memory, own rank included); multicast_hits, when    \
       non-NULL, is the NVSwitch multicast alias of the same array (one multimem store instead of world_size   \
       stores; float only).  hits may be NULL.  The caller orders a cross-rank barrier after the call before    \
       anyone reads the gathered arrays. */                                                                   \
    BVH_API int bvh##S##_intersect_rays_gather(struct bvh##S* bvh, const struct bvh_ray##S* rays, size_t ray_count, \
                                               struct bvh_hit##S* hits, void* const* gathered_hits, int world_size, \
                                               size_t shard_offset, void* multicast_hits, unsigned flags);     \
    /* Same, also returning the per-ray traversal counters (statistics kernel). */                      \
    BVH_API int bvh##S##_intersect_rays_stats(struct bvh##S* bvh, const struct bvh_ray##S* rays, size_t ray_count, \
                                              struct bvh_hit##S* hits, struct bvh_ray_stats* stats, unsigned flags); \
    /* Wait for the handle's stream. */                                                                 \
    BVH_API int bvh##S##_sync(struct bvh##S* bvh);                                                      \
    /* Longest chain of inner nodes below the root (the traversal stack bound). */                      \
    BVH_API size_t bvh##S##_get_depth(struct bvh##S* bvh);                                              \
    /* enum bvh_property; (size_t)-1 for an unknown property or a failed upload of an edited mirror. */  \
    BVH_API size_t bvh##S##_get_property(struct bvh##S* bvh, int property);                             \
    /* The whole BVH-order -> original primitive id array of the host mirror (bvhNN_get_prim_count entries; what   \
       bvhNN_get_prim_id reads one element of), valid until the handle is destroyed or rebuilt; NULL on failure. */ \
    BVH_API const size_t* bvh##S##_get_prim_ids(struct bvh##S* bvh);

BVH_B200_DECLARE(float, 3f)
BVH_B200_DECLARE(double, 3d)

/* The device-resident tree of a handle, for CUDA kernels of the caller's own (bvhNN_get_device_view), is declared in
 * <bvh_b200_device.h>. */

#ifdef __cplusplus
}
#endif
#endif
