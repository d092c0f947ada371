/* include/bvh_b200_device.h — C ABI: the device-resident tree of a handle, for CUDA kernels that traverse it with
 * their own leaf functions (include/bvh/v2/cuda/intersect.cuh wraps it for device code).  Exported by libbvh_c.so
 * next to the entry points of <bvh_b200.h>.
 *
 * struct bvh_device_viewNN — all pointers are device pointers on `device`:
 *   nodes     node_count + 1 records; reference node i (what bvhNN_get_node(bvh, i) shows) is record i + 1,
 *             record 0 is padding.  A record is the node padded to 32 bytes (3f: float bounds[6] as
 *             minx,maxx,miny,maxy,minz,maxz, uint32_t index, uint32_t pad) / 64 bytes (3d: double bounds[6],
 *             uint64_t index, uint64_t pad); index = first_id << 4 | prim_count, as in the reference.
 *   prim_ids  prim_count original primitive ids (32-bit) in BVH order: the device copy of bvhNN_get_prim_ids
 *   tris      prim_count BVH-order PrecomputedTri records (48 / 96 bytes: p0, e1 = p0 - p1, e2 = p2 - p0,
 *             n = cross(e1, e2)), or NULL when no triangles are attached
 *   depth     longest chain of inner nodes below the root: a traversal's stack holds at most depth + 1 entries
 *   stream    the handle's cudaStream_t
 *
 * When a view stops being valid:
 *   - the handle is rebuilt, loaded or destroyed;
 *   - its tree is uploaded again: the first batched call (or bvhNN_get_device_view) after an edit of the host mirror
 *     (bvh_nodeNN_set_*, bvhNN_refit, bvhNN_optimize, ...) replaces nodes and prim_ids;
 *   - bvhNN_set_triangles replaces the triangle array (tris).
 * bvhNN_refit_triangles keeps every pointer and rewrites the boxes and triangles in place.
 *
 * Ordering: launch kernels that use a view on its stream, or call bvhNN_sync first, so that the library's own work
 * on the tree has finished. */
#ifndef BVH_B200_DEVICE_H
#define BVH_B200_DEVICE_H

#include <bvh_b200.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BVH_B200_DECLARE_VIEW(S)                                                                                   \
    struct bvh_device_view##S {                                                                                   \
        int device;                                                                                               \
        void* stream;                                                                                             \
        const void* nodes;                                                                                        \
        const uint32_t* prim_ids;                                                                                 \
        const void* tris;                                                                                         \
        size_t node_count, prim_count, depth;                                                                     \
    };                                                                                                            \
    /* Fills *view with the device tree, uploading an edited host mirror first, like every batched call.           \
       Non-zero, with a message from bvh_last_error(), for a NULL argument or a handle without a tree. */          \
    BVH_API int bvh##S##_get_device_view(struct bvh##S* bvh, struct bvh_device_view##S* view);

BVH_B200_DECLARE_VIEW(3f)
BVH_B200_DECLARE_VIEW(3d)

#ifdef __cplusplus
}
#endif
#endif
