/* include/bvh_b200_device.h — C ABI: the device-resident tree of a handle, for CUDA kernels that traverse it with
 * their own leaf functions (include/bvh/v2/cuda/intersect.cuh wraps it for device code), its build from device-resident
 * boxes and its refit from per-primitive boxes, so that a tree over primitives of the caller's own (spheres,
 * particles, ...) can be built and follow them as they move without leaving the GPU.  Exported by libbvh_c.so next to
 * the entry points of <bvh_b200.h>.
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
 * bvhNN_refit_triangles keeps every pointer and rewrites the boxes and triangles in place; bvhNN_refit_boxes keeps
 * every pointer and rewrites the boxes in place.
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
    BVH_API int bvh##S##_get_device_view(struct bvh##S* bvh, struct bvh_device_view##S* view);                     \
    /* Refit from per-primitive boxes: bboxes[i] is the box of ORIGINAL primitive i (prim_count entries, the tree's      \
       count).  Each leaf box becomes its primitives' boxes folded in BVH order into the empty box (BBox::extend), then \
       every inner box the union of its children (reference Bvh::refit, bvh.h:184-218): bit for bit what writing those   \
       leaf boxes with bvh_nodeNN_set_bbox and calling bvhNN_refit gives.  Topology, primitive ids and attached           \
       triangles are left as they are.  The boxes may be larger than their primitives (e.g. covering the motion over a  \
       time step); a box that does not enclose its primitive loses that primitive's hits, as in the reference.          \
       An edited host mirror is uploaded first; afterwards the mirror is downloaded again on the next call that reads   \
       it, and the wide companion tree, if the handle has one, is rebuilt.  Device pointers of earlier views stay valid. \
       With BVH_DEVICE_POINTERS, bboxes is a device pointer and the call is ordered on the handle's stream without       \
       waiting for the device, except when a wide companion tree is rebuilt (that synchronises the stream).  With a     \
       host pointer the boxes are copied and the call returns when the refit is done.  Non-zero, with a message from     \
       bvh_last_error(), for a NULL handle or bboxes, a prim_count that is not the tree's, or a handle without a tree;    \
       the tree is then left as it was. */                                                                            \
    BVH_API int bvh##S##_refit_boxes(struct bvh##S* bvh, const struct bvh_bbox##S* bboxes, size_t prim_count, unsigned flags); \
    /* bvhNN_build from boxes and centres that may live on the GPU: with BVH_DEVICE_POINTERS, bboxes and centers are     \
       device pointers on the device chosen by bvh_cuda_set_device; without it they are host pointers and the call is    \
       bvhNN_build.  The tree is bit for bit what bvhNN_build gives for the same values and config.  The build runs on  \
       the new handle's stream (the caller's stream after bvh_cuda_set_stream, otherwise a private one) and the call    \
       returns after the build's one synchronisation of that stream, so the inputs are no longer read when it returns.  \
       With a private stream, finish writing the boxes and centres before the call.  NULL, with a message from          \
       bvh_last_error(), for a NULL bboxes or centers or a prim_count of 0 or beyond the index range. */                  \
    BVH_API struct bvh##S* bvh##S##_build_boxes(const struct bvh_bbox##S* bboxes, const struct bvh_vec##S* centers,      \
                                                size_t prim_count, const struct bvh_build_config* config, unsigned flags);

BVH_B200_DECLARE_VIEW(3f)
BVH_B200_DECLARE_VIEW(3d)

#ifdef __cplusplus
}
#endif
#endif
