// tests/device_query_kernels.cu — test kernels for DeviceView::traverse_top_down (include/bvh/v2/cuda/intersect.cuh),
// the traversal with the caller's node test.
//
// Compiled for sm_90a with the library's NVCC_FLAGS (--fmad=false among them) into tests/_build/libdevice_query_kernels.so
// (bvh_b200/build_ext.py build_device_query_tests) and driven by tests/test_device_query_gpu.py and
// scripts/device_query_bench.py.  Every entry point returns 0, or -1 with a message in dq_last_error().
//   dq_overlap*        per query box (min3, max3): the primitives whose boxes overlap it (count and an order-free hash of
//                      the id set), with a per-thread array stack or the shared-memory stack; the node function returns
//                      an aggregate
//   dq_nearest*        per query point: the primitive whose centre is nearest (id, squared distance), descending the
//                      nearer child first, with the leaf shrinking the radius the node test reads; the node function
//                      returns a cuda::std::tuple
//   dq_host_overlap*, dq_host_nearest*  the same functions through Bvh<Node>::traverse_top_down of the C++ surface on the
//                      handle's host mirror
// The device entry points take device pointers and launch on the handle's stream without waiting for it; the recorder
// outputs (leaf calls, a hash of their (begin, end) sequence, node-function calls) may be NULL.
#include <cuda_runtime.h>
#include <cuda/std/tuple>

#include <bvh/v2/bvh.h>
#include <bvh/v2/stack.h>

#include "device_queries.h"

#include <string>
#include <tuple>
#include <vector>

namespace {

using bvh::v2::cuda::DeviceView;

thread_local std::string g_error;

constexpr unsigned kBlock = 128;
constexpr unsigned kSmallStack = 128;   // entries of the per-thread array stack
enum StackKind : int { kArrayStack = 0, kSharedStack = 1 };

#define DQ_TRY(expr)                                                                                        \
    do {                                                                                                    \
        cudaError_t e__ = (expr);                                                                           \
        if (e__ != cudaSuccess) { g_error = std::string(#expr) + ": " + cudaGetErrorString(e__); return -1; } \
    } while (0)

template <typename T> struct Api;
template <> struct Api<float> {
    using Handle = bvh3f; using View = bvh_device_view3f; using BBox = bvh_bbox3f; using Vec = bvh_vec3f;
    static int view(Handle* h, View* v) { return bvh3f_get_device_view(h, v); }
    static const void* node0(Handle* h) { return bvh3f_get_node(h, 0); }
    static size_t node_count(Handle* h) { return bvh3f_get_node_count(h); }
    static size_t prim_count(Handle* h) { return bvh3f_get_prim_count(h); }
    static const size_t* prim_ids(Handle* h) { return bvh3f_get_prim_ids(h); }
};
template <> struct Api<double> {
    using Handle = bvh3d; using View = bvh_device_view3d; using BBox = bvh_bbox3d; using Vec = bvh_vec3d;
    static int view(Handle* h, View* v) { return bvh3d_get_device_view(h, v); }
    static const void* node0(Handle* h) { return bvh3d_get_node(h, 0); }
    static size_t node_count(Handle* h) { return bvh3d_get_node_count(h); }
    static size_t prim_count(Handle* h) { return bvh3d_get_prim_count(h); }
    static const size_t* prim_ids(Handle* h) { return bvh3d_get_prim_ids(h); }
};

// One overlap query's state: the node test and the leaf, the same code on both sides.
template <typename T> struct Overlap {
    const T* boxes;      // prim_count x (min3, max3), original order
    const T* q;
    uint32_t count = 0;
    uint64_t ids = 0;
    template <typename B> BVH_HD dq::Pick pick(const B& l, const B& r) const {
        return dq::Pick { dq::overlaps<T>(l, q), dq::overlaps<T>(r, q), false };
    }
    BVH_HD void visit(uint64_t id) {
        if (dq::overlaps<T>(dq::AsNode<T>{ boxes + 6 * id }, q)) { ++count; ids += dq::id_hash(id); }
    }
};

// One nearest-centre query's state: the leaf shrinks `best`, which the next node test reads.
template <typename T> struct Nearest {
    const T* centers;    // prim_count x 3, original order
    const T* p;
    T best;
    uint32_t id = 0xFFFFFFFFu;
    template <typename B> BVH_HD dq::Pick pick(const B& l, const B& r) const {
        const T dl = dq::box_dist2<T>(l, p), dr = dq::box_dist2<T>(r, p);
        return dq::Pick { dl < best, dr < best, dl > dr };
    }
    BVH_HD void visit(uint64_t k) {
        const T d = dq::point_dist2<T>(centers + 3 * k, p);
        if (d < best) { best = d; id = (uint32_t)k; }
    }
};

struct Recorder {
    uint32_t leaves = 0, nodes = 0;
    uint64_t hash = dq::kHashSeed;
    BVH_HD void leaf(size_t begin, size_t end) { ++leaves; hash = dq::mix(dq::mix(hash, begin), end); }
};

template <typename T, typename Stack>
__device__ void overlap_one(const DeviceView<T>& view, Stack& stack, const T* boxes, const T* q, size_t i, uint32_t* counts,
                            uint64_t* idsums, uint32_t* leaves, uint64_t* hashes, uint32_t* nodes) {
    using Node = typename DeviceView<T>::Node;
    Overlap<T> o { boxes, q };
    Recorder rec;
    view.template traverse_top_down<false>(view.root_index(), stack,
        [&](size_t begin, size_t end) {
            rec.leaf(begin, end);
            for (size_t k = begin; k < end; ++k) o.visit(view.prim_id(k));
            return false;
        },
        [&](const Node& l, const Node& r) { ++rec.nodes; return o.pick(l.bounds, r.bounds); });
    counts[i] = o.count;
    if (idsums) idsums[i] = o.ids;
    if (leaves) { leaves[i] = rec.leaves; hashes[i] = rec.hash; nodes[i] = rec.nodes; }
}

template <typename T, int kStack>
__global__ void __launch_bounds__(kBlock)
overlap_kernel(DeviceView<T> view, const T* __restrict__ boxes, const T* __restrict__ queries, size_t m, uint32_t* counts,
               uint64_t* idsums, uint32_t* leaves, uint64_t* hashes, uint32_t* nodes) {
    extern __shared__ __align__(128) unsigned char smem[];
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (i >= m) return;
    T q[6];
    for (int k = 0; k < 6; ++k) q[k] = queries[6 * i + k];
    if constexpr (kStack == kSharedStack) {
        auto stack = DeviceView<T>::shared_stack(smem, kBlock);
        overlap_one<T>(view, stack, boxes, q, i, counts, idsums, leaves, hashes, nodes);
    } else {
        typename DeviceView<T>::template SmallStack<kSmallStack> stack;
        overlap_one<T>(view, stack, boxes, q, i, counts, idsums, leaves, hashes, nodes);
    }
}

template <typename T, typename Stack>
__device__ void nearest_one(const DeviceView<T>& view, Stack& stack, const T* centers, const T* p, size_t i, uint32_t* ids,
                            T* dist2, uint32_t* leaves, uint64_t* hashes, uint32_t* nodes) {
    using Node = typename DeviceView<T>::Node;
    Nearest<T> s { centers, p, T(1) / T(0) };
    Recorder rec;
    view.template traverse_top_down<false>(view.root_index(), stack,
        [&](size_t begin, size_t end) {
            rec.leaf(begin, end);
            for (size_t k = begin; k < end; ++k) s.visit(view.prim_id(k));
            return false;
        },
        [&](const Node& l, const Node& r) {
            ++rec.nodes;
            const dq::Pick d = s.pick(l.bounds, r.bounds);
            return cuda::std::make_tuple(d.hit_left, d.hit_right, d.should_swap);
        });
    ids[i] = s.id;
    dist2[i] = s.best;
    if (leaves) { leaves[i] = rec.leaves; hashes[i] = rec.hash; nodes[i] = rec.nodes; }
}

template <typename T, int kStack>
__global__ void __launch_bounds__(kBlock)
nearest_kernel(DeviceView<T> view, const T* __restrict__ centers, const T* __restrict__ points, size_t m, uint32_t* ids,
               T* dist2, uint32_t* leaves, uint64_t* hashes, uint32_t* nodes) {
    extern __shared__ __align__(128) unsigned char smem[];
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (i >= m) return;
    const T p[3] = { points[3 * i], points[3 * i + 1], points[3 * i + 2] };
    if constexpr (kStack == kSharedStack) {
        auto stack = DeviceView<T>::shared_stack(smem, kBlock);
        nearest_one<T>(view, stack, centers, p, i, ids, dist2, leaves, hashes, nodes);
    } else {
        typename DeviceView<T>::template SmallStack<kSmallStack> stack;
        nearest_one<T>(view, stack, centers, p, i, ids, dist2, leaves, hashes, nodes);
    }
}

// The handle's device view, its stack capacity checked on the host (DeviceView::from throws when it is too small).
template <typename T> int get_view(typename Api<T>::Handle* h, DeviceView<T>& view) {
    typename Api<T>::View c {};
    if (Api<T>::view(h, &c)) { g_error = bvh_last_error(); return -1; }
    try { view = DeviceView<T>::from(c, kSmallStack); } catch (const std::exception& e) { g_error = e.what(); return -1; }
    DQ_TRY(cudaSetDevice(c.device));
    return 0;
}

template <typename Kernel>
int launch(Kernel kernel, int stack_kind, size_t smem_bytes, size_t m, cudaStream_t stream, auto... args) {
    const size_t smem = stack_kind == kSharedStack ? smem_bytes : 0;
    DQ_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<(unsigned)((m + kBlock - 1) / kBlock), kBlock, smem, stream>>>(args...);
    DQ_TRY(cudaGetLastError());
    return 0;
}

template <typename T>
int overlap(typename Api<T>::Handle* h, const T* boxes, const T* queries, size_t m, int stack_kind, uint32_t* counts,
            uint64_t* idsums, uint32_t* leaves, uint64_t* hashes, uint32_t* nodes) {
    if (!h || !boxes || !queries || !counts || (leaves && (!hashes || !nodes))) { g_error = "null argument"; return -1; }
    DeviceView<T> view;
    if (get_view(h, view)) return -1;
    if (m == 0) return 0;
    cudaStream_t stream = static_cast<cudaStream_t>(view.stream);
    const size_t smem = view.shared_stack_bytes(kBlock);
    if (stack_kind == kSharedStack)
        return launch(overlap_kernel<T, kSharedStack>, stack_kind, smem, m, stream, view, boxes, queries, m, counts, idsums, leaves, hashes, nodes);
    return launch(overlap_kernel<T, kArrayStack>, stack_kind, smem, m, stream, view, boxes, queries, m, counts, idsums, leaves, hashes, nodes);
}

template <typename T>
int nearest(typename Api<T>::Handle* h, const T* centers, const T* points, size_t m, int stack_kind, uint32_t* ids, T* dist2,
            uint32_t* leaves, uint64_t* hashes, uint32_t* nodes) {
    if (!h || !centers || !points || !ids || !dist2 || (leaves && (!hashes || !nodes))) { g_error = "null argument"; return -1; }
    DeviceView<T> view;
    if (get_view(h, view)) return -1;
    if (m == 0) return 0;
    cudaStream_t stream = static_cast<cudaStream_t>(view.stream);
    const size_t smem = view.shared_stack_bytes(kBlock);
    if (stack_kind == kSharedStack)
        return launch(nearest_kernel<T, kSharedStack>, stack_kind, smem, m, stream, view, centers, points, m, ids, dist2, leaves, hashes, nodes);
    return launch(nearest_kernel<T, kArrayStack>, stack_kind, smem, m, stream, view, centers, points, m, ids, dist2, leaves, hashes, nodes);
}

// The handle's host mirror as a Bvh<Node> of the C++ surface.
template <typename T> int mirror(typename Api<T>::Handle* h, bvh::v2::Bvh<bvh::v2::Node<T, 3>>& bvh) {
    using Node = bvh::v2::Node<T, 3>;
    bvh.nodes.resize(Api<T>::node_count(h));
    if (bvh.nodes.empty()) { g_error = bvh_last_error(); return -1; }
    std::memcpy(bvh.nodes.data(), Api<T>::node0(h), bvh.nodes.size() * sizeof(Node));
    bvh.prim_ids.assign(Api<T>::prim_ids(h), Api<T>::prim_ids(h) + Api<T>::prim_count(h));
    return 0;
}

// Host arrays throughout.
template <typename T>
int host_overlap(typename Api<T>::Handle* h, const T* boxes, const T* queries, size_t m, uint32_t* counts, uint64_t* idsums,
                 uint32_t* leaves, uint64_t* hashes, uint32_t* nodes) {
    using Node = bvh::v2::Node<T, 3>;
    if (!h || !boxes || !queries || !counts || !idsums || !leaves || !hashes || !nodes) { g_error = "null argument"; return -1; }
    bvh::v2::Bvh<Node> bvh;
    if (mirror<T>(h, bvh)) return -1;
    for (size_t i = 0; i < m; ++i) {
        Overlap<T> o { boxes, queries + 6 * i };
        Recorder rec;
        bvh::v2::GrowingStack<typename Node::Index> stack;
        bvh.template traverse_top_down<false>(bvh.get_root().index, stack,
            [&](size_t begin, size_t end) {
                rec.leaf(begin, end);
                for (size_t k = begin; k < end; ++k) o.visit(bvh.prim_ids[k]);
                return false;
            },
            [&](const Node& l, const Node& r) {
                ++rec.nodes;
                const dq::Pick d = o.pick(l.bounds, r.bounds);
                return std::make_tuple(d.hit_left, d.hit_right, d.should_swap);
            });
        counts[i] = o.count; idsums[i] = o.ids; leaves[i] = rec.leaves; hashes[i] = rec.hash; nodes[i] = rec.nodes;
    }
    return 0;
}

template <typename T>
int host_nearest(typename Api<T>::Handle* h, const T* centers, const T* points, size_t m, uint32_t* ids, T* dist2,
                 uint32_t* leaves, uint64_t* hashes, uint32_t* nodes) {
    using Node = bvh::v2::Node<T, 3>;
    if (!h || !centers || !points || !ids || !dist2 || !leaves || !hashes || !nodes) { g_error = "null argument"; return -1; }
    bvh::v2::Bvh<Node> bvh;
    if (mirror<T>(h, bvh)) return -1;
    for (size_t i = 0; i < m; ++i) {
        Nearest<T> s { centers, points + 3 * i, T(1) / T(0) };
        Recorder rec;
        bvh::v2::GrowingStack<typename Node::Index> stack;
        bvh.template traverse_top_down<false>(bvh.get_root().index, stack,
            [&](size_t begin, size_t end) {
                rec.leaf(begin, end);
                for (size_t k = begin; k < end; ++k) s.visit(bvh.prim_ids[k]);
                return false;
            },
            [&](const Node& l, const Node& r) {
                ++rec.nodes;
                const dq::Pick d = s.pick(l.bounds, r.bounds);
                return std::make_tuple(d.hit_left, d.hit_right, d.should_swap);
            });
        ids[i] = s.id; dist2[i] = s.best; leaves[i] = rec.leaves; hashes[i] = rec.hash; nodes[i] = rec.nodes;
    }
    return 0;
}

// bvh::v2::cuda::Accel<T>::from_boxes: the node count and depth of its device view, or -1
template <typename T>
int accel_from_boxes(const T* boxes, const T* centers, size_t n, unsigned flags, size_t* node_count, size_t* depth) {
    try {
        auto accel = bvh::v2::cuda::Accel<T>::from_boxes(reinterpret_cast<const bvh::v2::BBox<T, 3>*>(boxes),
                                                         reinterpret_cast<const bvh::v2::Vec<T, 3>*>(centers), n, nullptr, flags);
        const auto v = accel.device_view();
        *node_count = v.node_count; *depth = v.depth;
        return 0;
    } catch (const std::exception& e) {
        g_error = e.what();
        return -1;
    }
}

} // namespace

#define DQ_EXPORT extern "C" __attribute__((visibility("default")))
#define DQ_ENTRY(T, S)                                                                                                 \
    DQ_EXPORT int dq_overlap##S(bvh##S* h, const T* boxes, const T* queries, size_t m, int stack_kind, uint32_t* counts,  \
                                uint64_t* idsums, uint32_t* leaves, uint64_t* hashes, uint32_t* nodes) {               \
        return overlap<T>(h, boxes, queries, m, stack_kind, counts, idsums, leaves, hashes, nodes); }                  \
    DQ_EXPORT int dq_nearest##S(bvh##S* h, const T* centers, const T* points, size_t m, int stack_kind, uint32_t* ids,   \
                                T* dist2, uint32_t* leaves, uint64_t* hashes, uint32_t* nodes) {                       \
        return nearest<T>(h, centers, points, m, stack_kind, ids, dist2, leaves, hashes, nodes); }                     \
    DQ_EXPORT int dq_host_overlap##S(bvh##S* h, const T* boxes, const T* queries, size_t m, uint32_t* counts,           \
                                     uint64_t* idsums, uint32_t* leaves, uint64_t* hashes, uint32_t* nodes) {          \
        return host_overlap<T>(h, boxes, queries, m, counts, idsums, leaves, hashes, nodes); }                         \
    DQ_EXPORT int dq_host_nearest##S(bvh##S* h, const T* centers, const T* points, size_t m, uint32_t* ids, T* dist2,   \
                                     uint32_t* leaves, uint64_t* hashes, uint32_t* nodes) {                            \
        return host_nearest<T>(h, centers, points, m, ids, dist2, leaves, hashes, nodes); }                            \
    DQ_EXPORT int dq_accel_from_boxes##S(const T* boxes, const T* centers, size_t n, unsigned flags, size_t* node_count, \
                                         size_t* depth) {                                                              \
        return accel_from_boxes<T>(boxes, centers, n, flags, node_count, depth); }

DQ_ENTRY(float, 3f)
DQ_ENTRY(double, 3d)

DQ_EXPORT const char* dq_last_error() { return g_error.c_str(); }
