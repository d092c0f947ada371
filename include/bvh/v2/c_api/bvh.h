/* include/bvh/v2/c_api/bvh.h — the reference library's C API surface, re-declared for the CUDA engine.
 *
 * Same include path, names, signatures and POD layouts as the reference header
 * (reference src/bvh/v2/c_api/bvh.h:32-295), so C callers written against the reference
 * (e.g. reference test/c_api_example.c) compile and link against this library unchanged.
 * The declarations are stamped out per suffix by one macro instead of being spelled out four times:
 *
 *   suffix  scalar  dim   handle        node type         callback type
 *   2f      float   2     struct bvh2f  struct bvh_node2f  bvh_intersect_callbackf
 *   3f      float   3     struct bvh3f  struct bvh_node3f  bvh_intersect_callbackf
 *   2d      double  2     struct bvh2d  struct bvh_node2d  bvh_intersect_callbackd
 *   3d      double  3     struct bvh3d  struct bvh_node3d  bvh_intersect_callbackd
 *
 * Semantics that differ from the reference are listed in INTEGRATION.md; in short: bvhNN_build
 * builds on the GPU (the thread pool argument is ignored), bvhNN_optimize keeps the tree as is.
 * The 2-D suffixes build on the GPU as well (boxes lifted to z = 0) and then live on the host: the
 * reference has no 2-D primitive type, leaves are intersected by the caller's callback one ray per call.
 * The batched GPU entry points live in <bvh_b200.h>.
 */
#ifndef BVH_V2_C_API_BVH_H
#define BVH_V2_C_API_BVH_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_MSC_VER)
#define BVH_EXPORT __declspec(dllexport)
#define BVH_IMPORT __declspec(dllimport)
#else
#define BVH_EXPORT __attribute__((visibility("default")))
#define BVH_IMPORT BVH_EXPORT
#endif
#ifdef BVH_BUILD_API
#define BVH_API BVH_EXPORT
#else
#define BVH_API BVH_IMPORT
#endif

#define BVH_ROOT_INDEX 0
#define BVH_INVALID_PRIM_ID SIZE_MAX

struct bvh_thread_pool;

enum bvh_build_quality { BVH_BUILD_QUALITY_LOW, BVH_BUILD_QUALITY_MEDIUM, BVH_BUILD_QUALITY_HIGH };

struct bvh_build_config {
    enum bvh_build_quality quality;
    size_t min_leaf_size, max_leaf_size, parallel_threshold;
};

/* POD geometry: vec = coordinates, bbox = {min, max}, ray = {org, dir, tmin, tmax} */
#define BVH_DECLARE_PODS(T, S, COORDS)                                           \
    struct bvh##S; struct bvh_node##S;                                           \
    struct bvh_vec##S { T COORDS; };                                             \
    struct bvh_bbox##S { struct bvh_vec##S min, max; };                          \
    struct bvh_ray##S { struct bvh_vec##S org, dir; T tmin, tmax; };
#define BVH_COMMA ,
BVH_DECLARE_PODS(float,  2f, x BVH_COMMA y)
BVH_DECLARE_PODS(float,  3f, x BVH_COMMA y BVH_COMMA z)
BVH_DECLARE_PODS(double, 2d, x BVH_COMMA y)
BVH_DECLARE_PODS(double, 3d, x BVH_COMMA y BVH_COMMA z)

/* Leaf callback of the per-ray API: user_fn(user_data, &t, begin, end) intersects BVH-order
 * primitives [begin, end), writes the new closest distance through t and returns whether anything
 * was hit (for *_any a true return ends the traversal). */
struct bvh_intersect_callbackf { void* user_data; bool (*user_fn)(void*, float*,  size_t begin, size_t end); };
struct bvh_intersect_callbackd { void* user_data; bool (*user_fn)(void*, double*, size_t begin, size_t end); };

/* A thread count of zero means "as many as the machine has".  Kept for source compatibility: the
 * GPU builder does not use host threads. */
BVH_API struct bvh_thread_pool* bvh_thread_pool_create(size_t thread_count);
BVH_API void bvh_thread_pool_destroy(struct bvh_thread_pool*);

#define BVH_DECLARE_API(T, S, CALLBACK)                                                                     \
    /* construction: pool and config may be NULL */                                                         \
    BVH_API struct bvh##S* bvh##S##_build(struct bvh_thread_pool*, const struct bvh_bbox##S* bboxes,        \
                                          const struct bvh_vec##S* centers, size_t prim_count,              \
                                          const struct bvh_build_config* config);                           \
    BVH_API void bvh##S##_destroy(struct bvh##S*);                                                          \
    /* serialisation in the reference's binary format */                                                    \
    BVH_API void bvh##S##_save(const struct bvh##S*, FILE*);                                                \
    BVH_API struct bvh##S* bvh##S##_load(FILE*);                                                            \
    /* node / primitive-id access; node pointers are invalidated by bvhNN_append_node */                   \
    BVH_API struct bvh_node##S* bvh##S##_get_node(struct bvh##S*, size_t node_id);                          \
    BVH_API size_t bvh##S##_get_prim_id(const struct bvh##S*, size_t i);                                    \
    BVH_API size_t bvh##S##_get_prim_count(const struct bvh##S*);                                           \
    BVH_API size_t bvh##S##_get_node_count(const struct bvh##S*);                                           \
    BVH_API bool bvh_node##S##_is_leaf(const struct bvh_node##S*);                                          \
    BVH_API size_t bvh_node##S##_get_prim_count(const struct bvh_node##S*);                                 \
    BVH_API void bvh_node##S##_set_prim_count(struct bvh_node##S*, size_t);                                 \
    BVH_API size_t bvh_node##S##_get_first_id(const struct bvh_node##S*);                                   \
    BVH_API void bvh_node##S##_set_first_id(struct bvh_node##S*, size_t);                                   \
    BVH_API struct bvh_bbox##S bvh_node##S##_get_bbox(const struct bvh_node##S*);                           \
    BVH_API void bvh_node##S##_set_bbox(struct bvh_node##S*, const struct bvh_bbox##S*);                    \
    /* modification */                                                                                      \
    BVH_API void bvh##S##_append_node(struct bvh##S*);                                                      \
    BVH_API void bvh##S##_remove_last_node(struct bvh##S*);                                                 \
    BVH_API void bvh##S##_refit(struct bvh##S*);                                                            \
    BVH_API void bvh##S##_optimize(struct bvh_thread_pool*, struct bvh##S*);                                \
    /* one ray, leaf primitives intersected by the callback */                                              \
    BVH_API void bvh##S##_intersect_ray_any(const struct bvh##S*, const struct bvh_ray##S*, const struct CALLBACK*);        \
    BVH_API void bvh##S##_intersect_ray_any_robust(const struct bvh##S*, const struct bvh_ray##S*, const struct CALLBACK*); \
    BVH_API void bvh##S##_intersect_ray(const struct bvh##S*, const struct bvh_ray##S*, const struct CALLBACK*);            \
    BVH_API void bvh##S##_intersect_ray_robust(const struct bvh##S*, const struct bvh_ray##S*, const struct CALLBACK*);

BVH_DECLARE_API(float,  2f, bvh_intersect_callbackf)
BVH_DECLARE_API(float,  3f, bvh_intersect_callbackf)
BVH_DECLARE_API(double, 2d, bvh_intersect_callbackd)
BVH_DECLARE_API(double, 3d, bvh_intersect_callbackd)

#ifdef __cplusplus
}
#endif
#endif
