// tests/device_query_batch_kernels.cu — test queriers for DeviceView::query (include/bvh/v2/cuda/intersect.cuh), the
// batch form of traverse_top_down on the persistent scheduler.
//
// Compiled for sm_90a with the library's NVCC_FLAGS (--fmad=false among them) into
// tests/_build/libdevice_query_batch_kernels.so (bvh_b200/build_ext.py build_device_query_batch_tests) and driven by
// tests/test_device_query_batch_gpu.py, scripts/device_query_bench.py and scripts/bottom_up_bench.py.  Every array is
// device-resident; the calls launch on `stream` (the handle's when null) without waiting for it.  Every entry point
// returns 0; -1 with a message in dqb_last_error(); -2 when query threw std::length_error, with its message.
//   dqb_query{3f,3d}      one batch of m queries of `kind` through DeviceView::query (per_thread = 0) or through a kernel
//                         of one thread per query that runs the same querier through traverse_top_down with a
//                         shared-memory stack (per_thread = 1).  Kinds, with the node and leaf functions of
//                         tests/device_query_kernels.cu (same arithmetic, so the same results bit for bit):
//                           0 overlap   prims: boxes (min3, max3), queries: boxes; r0 the count of overlapping boxes, r1
//                                       (u64) the sum of their id hashes
//                           1 nearest   prims: centres, queries: points; r0 the nearest centre's id, r1 (T) its squared
//                                       distance; the leaf shrinks the radius the node test reads, nearer child first
//                           2 contains  prims: boxes, queries: points (x, y, z); the node test is containment; r0 the last
//                                       containing primitive's id (all ones: none), r1 (u32) how many the leaves found;
//                                       any_hit makes it IsAnyHit, where a leaf that finds one ends the query
//                         Recorders (all three or none): leaf calls, a 64-bit hash of the (begin, end) sequence, node
//                         calls.  counts (nullable): 1 is added to counts[i] when query i finishes.
//   dqb_potential{3f,3d}  the Barnes-Hut potential of tests/device_bottom_up.h (bu::Potential) at `count` points, through
//                         query with the three-argument node test, which reads node mass and centre by the left child's
//                         index
//   dqb_workspace_bytes{3f,3d}  DeviceView::query_workspace_bytes
#include <cuda_runtime.h>

#include "device_bottom_up.h"

#include <stdexcept>
#include <string>

namespace {

using bvh::v2::cuda::DeviceView;

thread_local std::string g_error;
constexpr unsigned kBlock = 128;

enum Kind : int { kOverlap = 0, kNearest = 1, kContains = 2 };

template <typename T> struct Api;
template <> struct Api<float> {
    using Handle = bvh3f; using View = bvh_device_view3f;
    static int view(Handle* h, View* v) { return bvh3f_get_device_view(h, v); }
};
template <> struct Api<double> {
    using Handle = bvh3d; using View = bvh_device_view3d;
    static int view(Handle* h, View* v) { return bvh3d_get_device_view(h, v); }
};

struct Outputs {
    uint32_t* r0; void* r1; uint32_t* leaves; uint64_t* hashes; uint32_t* nodes; uint32_t* counts;
};

// The recorder's part of a payload; kRecord = false keeps none of it.
template <bool kRecord> struct Record {
    uint32_t leaves, nodes;
    uint64_t hash;
    __device__ void clear() { leaves = nodes = 0; hash = dq::kHashSeed; }
    __device__ void leaf(size_t begin, size_t end) { ++leaves; hash = dq::mix(dq::mix(hash, begin), end); }
    __device__ void node() { ++nodes; }
    __device__ void write(const Outputs& o, size_t i) const { o.leaves[i] = leaves; o.hashes[i] = hash; o.nodes[i] = nodes; }
};
template <> struct Record<false> {
    __device__ void clear() {}
    __device__ void leaf(size_t, size_t) {}
    __device__ void node() {}
    __device__ void write(const Outputs&, size_t) const {}
};

// The three test queriers: one struct, the kind chosen at compile time.
template <typename T, int kKind, bool kRecord> struct TestQuerier {
    using Node = typename DeviceView<T>::Node;
    struct Payload {
        T q[6];               // overlap: the query box (min3, max3); nearest, contains: the point in q[0..2]
        T best;               // nearest: the squared search radius
        uint32_t r0;
        uint64_t r1;
        Record<kRecord> rec;
    };
    const uint32_t* prim_ids;
    const T* prims;
    const T* queries;
    Outputs out;

    __device__ void start(size_t i, Payload& p) const {
        const int dims = kKind == kOverlap ? 6 : 3;
        for (int k = 0; k < dims; ++k) p.q[k] = queries[dims * i + k];
        p.best = T(1) / T(0);
        p.r0 = kKind == kOverlap ? 0u : 0xFFFFFFFFu;
        p.r1 = 0;
        p.rec.clear();
    }
    __device__ dq::Pick node(Payload& p, const Node& l, const Node& r) const {
        p.rec.node();
        if (kKind == kOverlap) return dq::Pick { dq::overlaps<T>(l.bounds, p.q), dq::overlaps<T>(r.bounds, p.q), false };
        if (kKind == kContains) return dq::Pick { dq::contains<T>(l.bounds, p.q), dq::contains<T>(r.bounds, p.q), false };
        const T dl = dq::box_dist2<T>(l.bounds, p.q), dr = dq::box_dist2<T>(r.bounds, p.q);
        return dq::Pick { dl < p.best, dr < p.best, dl > dr };
    }
    __device__ bool leaf(Payload& p, size_t begin, size_t end) const {
        p.rec.leaf(begin, end);
        bool found = false;
        for (size_t k = begin; k < end; ++k) {
            const uint32_t id = prim_ids[k];
            if (kKind == kOverlap) {
                if (dq::overlaps<T>(dq::AsNode<T>{ prims + 6 * (size_t)id }, p.q)) { ++p.r0; p.r1 += dq::id_hash(id); }
            } else if (kKind == kNearest) {
                const T d = dq::point_dist2<T>(prims + 3 * (size_t)id, p.q);
                if (d < p.best) { p.best = d; p.r0 = id; }
            } else if (dq::contains<T>(dq::AsNode<T>{ prims + 6 * (size_t)id }, p.q)) {
                p.r0 = id; ++p.r1; found = true;
            }
        }
        return found;
    }
    __device__ void finish(size_t i, const Payload& p) const {
        out.r0[i] = p.r0;
        if (kKind == kOverlap) static_cast<uint64_t*>(out.r1)[i] = p.r1;
        else if (kKind == kNearest) static_cast<T*>(out.r1)[i] = p.best;
        else static_cast<uint32_t*>(out.r1)[i] = (uint32_t)p.r1;
        p.rec.write(out, i);
        if (out.counts) atomicAdd(out.counts + i, 1u);
    }
};

// Barnes-Hut through the three-argument node test: bu::Potential's functions, its state kept in the payload.
template <typename T> struct PotentialQuerier {
    using Node = typename DeviceView<T>::Node;
    struct Payload { T p[3]; T sum; uint32_t approximated; };
    const uint32_t* prim_ids;
    const T* pos; const T* mass; const T* node_mass; const T* node_centre; const T* points;
    T theta2, eps2;
    T* phi;
    uint32_t* approximated;

    __device__ bu::Potential<T> potential(const Payload& p) const {
        bu::Potential<T> pot { prim_ids, pos, mass, node_mass, node_centre, p.p, theta2, eps2 };
        pot.sum = p.sum;
        pot.approximated = p.approximated;
        return pot;
    }
    __device__ void start(size_t i, Payload& p) const {
        for (int a = 0; a < 3; ++a) p.p[a] = points[3 * i + a];
        p.sum = T(0);
        p.approximated = 0;
    }
    __device__ dq::Pick node(Payload& p, const Node& l, const Node& r, size_t left) const {
        bu::Potential<T> pot = potential(p);
        const dq::Pick pick = pot.node(l.bounds, r.bounds, left);
        p.sum = pot.sum;
        p.approximated = pot.approximated;
        return pick;
    }
    __device__ bool leaf(Payload& p, size_t begin, size_t end) const {
        bu::Potential<T> pot = potential(p);
        const bool hit = pot.leaf(begin, end);
        p.sum = pot.sum;
        return hit;
    }
    __device__ void finish(size_t i, const Payload& p) const {
        phi[i] = p.sum;
        if (approximated) approximated[i] = p.approximated;
    }
};

// Any querier one thread per query through DeviceView::traverse_top_down: what a user kernel without query looks like.
template <typename T, bool kAny, typename Querier>
__global__ void __launch_bounds__(kBlock) per_thread_kernel(DeviceView<T> view, Querier querier, size_t n) {
    using Payload = typename Querier::Payload;
    extern __shared__ __align__(128) unsigned char smem[];
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (i >= n) return;
    auto stack = DeviceView<T>::shared_stack(smem, kBlock);
    Payload p;
    querier.start(i, p);
    view.template traverse_top_down<kAny>(view.root_index(), stack,
                                          [&](size_t begin, size_t end) { return querier.leaf(p, begin, end); },
                                          bvh::v2::cuda::detail::BoundNode<Querier, Payload, typename DeviceView<T>::Node> { querier, p });
    querier.finish(i, p);
}

template <typename T, bool kAny, typename Querier>
int run_querier(const DeviceView<T>& view, bool per_thread, size_t n, const Querier& querier, void* workspace, size_t bytes,
                cudaStream_t stream) {
    if (!per_thread) {
        view.template query<kAny>(n, querier, workspace, bytes, stream);
        return 0;
    }
    if (n == 0) return 0;
    const size_t smem = view.shared_stack_bytes(kBlock);
    cudaError_t e = cudaFuncSetAttribute(per_thread_kernel<T, kAny, Querier>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) {
        per_thread_kernel<T, kAny, Querier><<<(unsigned)((n + kBlock - 1) / kBlock), kBlock, smem, stream>>>(view, querier, n);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { g_error = std::string("per-thread kernel: ") + cudaGetErrorString(e); return -1; }
    return 0;
}

template <typename T, int kKind, bool kRecord>
int run_kind(const DeviceView<T>& view, bool per_thread, bool any_hit, size_t m, const T* prims, const T* queries,
             const Outputs& out, void* workspace, size_t bytes, cudaStream_t stream) {
    const TestQuerier<T, kKind, kRecord> querier { view.prim_ids, prims, queries, out };
    if constexpr (kKind == kContains)
        if (any_hit) return run_querier<T, true>(view, per_thread, m, querier, workspace, bytes, stream);
    return run_querier<T, false>(view, per_thread, m, querier, workspace, bytes, stream);
}

template <typename T, bool kRecord>
int run_record(int kind, const DeviceView<T>& view, bool per_thread, bool any_hit, size_t m, const T* prims, const T* queries,
               const Outputs& out, void* workspace, size_t bytes, cudaStream_t stream) {
    switch (kind) {
    case kOverlap: return run_kind<T, kOverlap, kRecord>(view, per_thread, any_hit, m, prims, queries, out, workspace, bytes, stream);
    case kNearest: return run_kind<T, kNearest, kRecord>(view, per_thread, any_hit, m, prims, queries, out, workspace, bytes, stream);
    case kContains: return run_kind<T, kContains, kRecord>(view, per_thread, any_hit, m, prims, queries, out, workspace, bytes, stream);
    }
    g_error = "no such kind";
    return -1;
}

template <typename T> int get_view(typename Api<T>::Handle* h, DeviceView<T>& view) {
    typename Api<T>::View c {};
    if (!h || Api<T>::view(h, &c)) { g_error = h ? bvh_last_error() : "null handle"; return -1; }
    view = DeviceView<T>::from(c);
    return 0;
}

// std::length_error -> -2, anything else -> -1, with the message
template <typename Fn> int guarded(Fn&& fn) {
    try {
        return fn();
    } catch (const std::length_error& e) {
        g_error = e.what();
        return -2;
    } catch (const std::exception& e) {
        g_error = e.what();
        return -1;
    }
}

template <typename T>
int query(typename Api<T>::Handle* h, int kind, int per_thread, int any_hit, const T* prims, const T* queries, size_t m,
          const Outputs& out, void* workspace, size_t bytes, void* stream) {
    if (!prims || !queries || !out.r0 || !out.r1 || (out.leaves && (!out.hashes || !out.nodes))) { g_error = "null argument"; return -1; }
    DeviceView<T> view;
    if (get_view(h, view)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : view.stream);
    return guarded([&] {
        if (out.leaves) return run_record<T, true>(kind, view, per_thread, any_hit, m, prims, queries, out, workspace, bytes, s);
        return run_record<T, false>(kind, view, per_thread, any_hit, m, prims, queries, out, workspace, bytes, s);
    });
}

template <typename T>
int potential(typename Api<T>::Handle* h, const T* pos, const T* m, const T* node_mass, const T* node_centre, const T* points,
              size_t count, T theta2, T eps2, T* phi, uint32_t* approximated, void* workspace, size_t bytes, void* stream) {
    if (!pos || !m || !node_mass || !node_centre || !points || !phi) { g_error = "null argument"; return -1; }
    DeviceView<T> view;
    if (get_view(h, view)) return -1;
    const PotentialQuerier<T> querier { view.prim_ids, pos, m, node_mass, node_centre, points, theta2, eps2, phi, approximated };
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : view.stream);
    return guarded([&] { return run_querier<T, false>(view, false, count, querier, workspace, bytes, s); });
}

} // namespace

#define DQB_EXPORT extern "C" __attribute__((visibility("default")))
#define DQB_ENTRY(T, S)                                                                                                  \
    DQB_EXPORT int dqb_query##S(bvh##S* h, int kind, int per_thread, int any_hit, const T* prims, const T* queries,      \
                                size_t m, uint32_t* r0, void* r1, uint32_t* leaves, uint64_t* hashes, uint32_t* nodes,   \
                                uint32_t* counts, void* workspace, size_t workspace_bytes, void* stream) {               \
        return query<T>(h, kind, per_thread, any_hit, prims, queries, m, Outputs { r0, r1, leaves, hashes, nodes, counts }, \
                        workspace, workspace_bytes, stream);                                                            \
    }                                                                                                                    \
    DQB_EXPORT int dqb_potential##S(bvh##S* h, const T* pos, const T* m, const T* node_mass, const T* node_centre,       \
                                    const T* points, size_t count, T theta2, T eps2, T* phi, uint32_t* approximated,     \
                                    void* workspace, size_t workspace_bytes, void* stream) {                             \
        return potential<T>(h, pos, m, node_mass, node_centre, points, count, theta2, eps2, phi, approximated, workspace,  \
                            workspace_bytes, stream);                                                                    \
    }                                                                                                                    \
    DQB_EXPORT size_t dqb_workspace_bytes##S(bvh##S* h) {                                                                \
        DeviceView<T> view;                                                                                              \
        return get_view<T>(h, view) ? 0 : view.query_workspace_bytes();                                                  \
    }

DQB_ENTRY(float, 3f)
DQB_ENTRY(double, 3d)

DQB_EXPORT const char* dqb_last_error() { return g_error.c_str(); }
