// tests/device_api_kernels.cu — test kernels for the device traversal API (include/bvh/v2/cuda/intersect.cuh).
//
// Compiled for sm_90a with the library's NVCC_FLAGS (--fmad=false among them) into tests/_build/libdevice_api_kernels.so
// (bvh_b200/build_ext.py build_device_api_tests) and driven by tests/test_device_api_gpu.py and
// scripts/device_api_bench.py.  Every entry point takes a handle and host arrays and returns 0, or -1 with a message
// in dapi_last_error().
//   dapi_trace*    the triangle leaf (DeviceView::intersect_tri, the reference's `t <= tmax` acceptance) with the
//                  shared-memory stack: one thread per ray, what a user kernel looks like
//   dapi_record*   leaf None / Tri / Sphere with a per-thread array stack, recording per ray the leaf calls, a 64-bit
//                  hash of their (begin, end) sequence and the inner-hook calls
//   dapi_host_record*  the same leaves through Bvh<Node>::intersect of the C++ surface on the handle's host mirror
#include <cuda_runtime.h>

#include <bvh/v2/bvh.h>
#include <bvh/v2/cuda/intersect.cuh>
#include <bvh/v2/stack.h>
#include <bvh/v2/tri.h>

#include <cmath>
#include <string>
#include <vector>

namespace {

using bvh::v2::cuda::DeviceView;

thread_local std::string g_error;

constexpr unsigned kBlock = 128;
constexpr unsigned kSmallStack = 128;   // entries of the recorder's per-thread stack

enum Leaf : int { kLeafNone = 0, kLeafTri = 1, kLeafSphere = 2 };

#define DAPI_TRY(expr)                                                                                      \
    do {                                                                                                    \
        cudaError_t e__ = (expr);                                                                           \
        if (e__ != cudaSuccess) { g_error = std::string(#expr) + ": " + cudaGetErrorString(e__); return -1; } \
    } while (0)

template <typename T> struct Api;
template <> struct Api<float> {
    using Handle = bvh3f; using View = bvh_device_view3f; using Ray = bvh_ray3f;
    static int view(Handle* h, View* v) { return bvh3f_get_device_view(h, v); }
    static const void* node0(Handle* h) { return bvh3f_get_node(h, 0); }
    static size_t node_count(Handle* h) { return bvh3f_get_node_count(h); }
    static size_t prim_count(Handle* h) { return bvh3f_get_prim_count(h); }
    static const size_t* prim_ids(Handle* h) { return bvh3f_get_prim_ids(h); }
};
template <> struct Api<double> {
    using Handle = bvh3d; using View = bvh_device_view3d; using Ray = bvh_ray3d;
    static int view(Handle* h, View* v) { return bvh3d_get_device_view(h, v); }
    static const void* node0(Handle* h) { return bvh3d_get_node(h, 0); }
    static size_t node_count(Handle* h) { return bvh3d_get_node_count(h); }
    static size_t prim_count(Handle* h) { return bvh3d_get_prim_count(h); }
    static const size_t* prim_ids(Handle* h) { return bvh3d_get_prim_ids(h); }
};

// reference sphere.h:15-50 (Sphere::intersect, AssumeNormalized = false) on a centre and a radius: the entry distance
// t0 and exit distance t1 clipped to [tmin, tmax], or false.  Vec dot is ((0 + a0 b0) + a1 b1) + a2 b2 (vec.h).
template <typename T>
__host__ __device__ inline bool sphere_hit(const T* c, T radius, const T org[3], const T dir[3], T tmin, T tmax, T& t0, T& t1) {
    const T oc[3] = { org[0] - c[0], org[1] - c[1], org[2] - c[2] };
    auto dot = [] (const T* a, const T* b) { T s = T(0) + a[0] * b[0]; s = s + a[1] * b[1]; return s + a[2] * b[2]; };
    const T a = dot(dir, dir);
    const T b = T(2.) * dot(dir, oc);
    const T cc = dot(oc, oc) - radius * radius;
    const T delta = b * b - T(4.) * a * cc;
    if (delta >= 0) {
        const T inv = -T(0.5) / a;
        const T sqrt_delta = std::sqrt(delta);
        const T n0 = (b + sqrt_delta) * inv, n1 = (b - sqrt_delta) * inv;
        t0 = n0 > tmin ? n0 : tmin;          // robust_max(n0, tmin)
        t1 = n1 < tmax ? n1 : tmax;          // robust_min(n1, tmax)
        if (t0 <= t1) return true;
    }
    return false;
}

// 64-bit hash of a leaf-call sequence
__host__ __device__ inline uint64_t mix(uint64_t h, uint64_t x) { return (h ^ x) * 1099511628211ull; }
constexpr uint64_t kHashSeed = 1469598103934665603ull;

template <typename T, bool kAny, bool kRobust>
__global__ void __launch_bounds__(kBlock)
trace_kernel(DeviceView<T> view, const typename Api<T>::Ray* __restrict__ rays, size_t n,
             uint32_t* __restrict__ ids, T* __restrict__ ts, T* __restrict__ us, T* __restrict__ vs, uint32_t* __restrict__ inner) {
    extern __shared__ __align__(128) unsigned char smem[];
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (i >= n) return;
    auto stack = DeviceView<T>::shared_stack(smem, kBlock);
    typename Api<T>::Ray ray = rays[i];
    size_t best = SIZE_MAX;
    T best_u = T(0), best_v = T(0);
    uint32_t steps = 0;
    auto leaf = [&](size_t begin, size_t end) {
        for (size_t k = begin; k < end; ++k) {
            T t, u, v;
            if (view.intersect_tri(k, ray, t, u, v)) { ray.tmax = t; best = k; best_u = u; best_v = v; }
        }
        return best != SIZE_MAX;
    };
    if (inner) view.template intersect<kAny, kRobust>(ray, view.root_index(), stack, leaf, [&](size_t) { ++steps; });
    else       view.template intersect<kAny, kRobust>(ray, view.root_index(), stack, leaf);
    ids[i] = best == SIZE_MAX ? 0xFFFFFFFFu : (uint32_t)view.prim_id(best);
    ts[i] = ray.tmax;
    us[i] = best_u; vs[i] = best_v;
    if (inner) inner[i] = steps;
}

template <typename T, bool kAny, bool kRobust, int kLeaf>
__global__ void __launch_bounds__(kBlock)
record_kernel(DeviceView<T> view, const typename Api<T>::Ray* __restrict__ rays, size_t n, const T* __restrict__ spheres,
              size_t start, uint32_t* __restrict__ ids, T* __restrict__ ts, uint32_t* __restrict__ leaves,
              uint64_t* __restrict__ hashes, uint32_t* __restrict__ inner) {
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (i >= n) return;
    typename DeviceView<T>::template SmallStack<kSmallStack> stack;
    typename Api<T>::Ray ray = rays[i];
    size_t best = SIZE_MAX;
    uint32_t calls = 0, steps = 0;
    uint64_t h = kHashSeed;
    const T org[3] = { ray.org.x, ray.org.y, ray.org.z }, dir[3] = { ray.dir.x, ray.dir.y, ray.dir.z };
    const auto start_index = start == SIZE_MAX ? view.root_index() : view.node(start).index;
    view.template intersect<kAny, kRobust>(ray, start_index, stack, [&](size_t begin, size_t end) {
        ++calls;
        h = mix(mix(h, begin), end);
        for (size_t k = begin; k < end; ++k) {
            if (kLeaf == kLeafTri) {
                T t, u, v;
                if (view.intersect_tri(k, ray, t, u, v)) { ray.tmax = t; best = k; }
            } else if (kLeaf == kLeafSphere) {
                const size_t id = view.prim_id(k);
                T t0, t1;
                if (sphere_hit<T>(spheres + 4 * id, spheres[4 * id + 3], org, dir, ray.tmin, ray.tmax, t0, t1)) { ray.tmax = t0; best = k; }
            }
        }
        return best != SIZE_MAX;
    }, [&](size_t) { ++steps; });
    ids[i] = best == SIZE_MAX ? 0xFFFFFFFFu : (uint32_t)view.prim_id(best);
    ts[i] = ray.tmax;
    leaves[i] = calls; hashes[i] = h; inner[i] = steps;
}

template <typename X> struct DeviceBuf {
    X* p = nullptr;
    ~DeviceBuf() { if (p) cudaFree(p); }
    int alloc(size_t n) { DAPI_TRY(cudaMalloc(&p, (n ? n : 1) * sizeof(X))); return 0; }
    int upload(const X* h, size_t n) { if (alloc(n)) return -1; if (n) DAPI_TRY(cudaMemcpy(p, h, n * sizeof(X), cudaMemcpyHostToDevice)); return 0; }
    int download(X* h, size_t n) const { if (h && n) DAPI_TRY(cudaMemcpy(h, p, n * sizeof(X), cudaMemcpyDeviceToHost)); return 0; }
};

template <typename T>
int get_view(typename Api<T>::Handle* h, DeviceView<T>& view, bool need_tris) {
    typename Api<T>::View c {};
    if (Api<T>::view(h, &c)) { g_error = bvh_last_error(); return -1; }
    if (need_tris && !c.tris) { g_error = "no triangles attached"; return -1; }
    view = DeviceView<T>::from(c);
    DAPI_TRY(cudaSetDevice(c.device));
    DAPI_TRY(cudaStreamSynchronize(static_cast<cudaStream_t>(c.stream)));     // the library's work on the tree is done
    return 0;
}

template <typename T, bool kAny, bool kRobust>
int launch_trace(const DeviceView<T>& view, const typename Api<T>::Ray* rays, size_t n, uint32_t* ids, T* t, T* u, T* v,
                 uint32_t* inner, cudaStream_t stream) {
    const size_t smem = view.shared_stack_bytes(kBlock);
    DAPI_TRY(cudaFuncSetAttribute(trace_kernel<T, kAny, kRobust>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    trace_kernel<T, kAny, kRobust><<<(unsigned)((n + kBlock - 1) / kBlock), kBlock, smem, stream>>>(view, rays, n, ids, t, u, v, inner);
    DAPI_TRY(cudaGetLastError());
    return 0;
}

template <typename T>
int trace_device(const DeviceView<T>& view, const typename Api<T>::Ray* rays, size_t n, unsigned flags, uint32_t* ids,
                 T* t, T* u, T* v, uint32_t* inner, cudaStream_t stream) {
    const bool any = flags & BVH_ANY_HIT, robust = flags & BVH_ROBUST;
    if (any) return robust ? launch_trace<T, true, true>(view, rays, n, ids, t, u, v, inner, stream)
                           : launch_trace<T, true, false>(view, rays, n, ids, t, u, v, inner, stream);
    return robust ? launch_trace<T, false, true>(view, rays, n, ids, t, u, v, inner, stream)
                  : launch_trace<T, false, false>(view, rays, n, ids, t, u, v, inner, stream);
}

template <typename T>
int trace(typename Api<T>::Handle* h, const typename Api<T>::Ray* rays, size_t n, unsigned flags, uint32_t* ids, T* t, T* u,
          T* v, uint32_t* inner) {
    if (!h || !rays || !ids || !t || !u || !v) { g_error = "null argument"; return -1; }
    DeviceView<T> view;
    if (get_view(h, view, true)) return -1;
    DeviceBuf<typename Api<T>::Ray> d_rays; DeviceBuf<uint32_t> d_ids, d_inner; DeviceBuf<T> d_t, d_u, d_v;
    if (d_rays.upload(rays, n) || d_ids.alloc(n) || d_t.alloc(n) || d_u.alloc(n) || d_v.alloc(n) || (inner && d_inner.alloc(n))) return -1;
    if (n && trace_device<T>(view, d_rays.p, n, flags, d_ids.p, d_t.p, d_u.p, d_v.p, inner ? d_inner.p : nullptr, nullptr)) return -1;
    DAPI_TRY(cudaDeviceSynchronize());
    if (d_ids.download(ids, n) || d_t.download(t, n) || d_u.download(u, n) || d_v.download(v, n) || (inner && d_inner.download(inner, n))) return -1;
    return 0;
}

template <typename T, bool kAny, bool kRobust>
void launch_record(int leaf, const DeviceView<T>& view, const typename Api<T>::Ray* rays, size_t n, const T* spheres, size_t start,
                   uint32_t* ids, T* t, uint32_t* leaves, uint64_t* hashes, uint32_t* inner) {
    const unsigned grid = (unsigned)((n + kBlock - 1) / kBlock);
    if (leaf == kLeafTri) record_kernel<T, kAny, kRobust, kLeafTri><<<grid, kBlock>>>(view, rays, n, spheres, start, ids, t, leaves, hashes, inner);
    else if (leaf == kLeafSphere) record_kernel<T, kAny, kRobust, kLeafSphere><<<grid, kBlock>>>(view, rays, n, spheres, start, ids, t, leaves, hashes, inner);
    else record_kernel<T, kAny, kRobust, kLeafNone><<<grid, kBlock>>>(view, rays, n, spheres, start, ids, t, leaves, hashes, inner);
}

// spheres: prim_count x {cx, cy, cz, radius} in original order (leaf kSphere only); start: reference node index to start
// at (SIZE_MAX: the root)
template <typename T>
int record(typename Api<T>::Handle* h, int leaf, const typename Api<T>::Ray* rays, size_t n, const T* spheres, size_t start,
           unsigned flags, uint32_t* ids, T* t, uint32_t* leaves, uint64_t* hashes, uint32_t* inner) {
    if (!h || !rays || !ids || !t || !leaves || !hashes || !inner || (leaf == kLeafSphere && !spheres)) { g_error = "null argument"; return -1; }
    DeviceView<T> view;
    if (get_view(h, view, leaf == kLeafTri)) return -1;
    if (view.stack_bound() > kSmallStack) { g_error = "tree too deep for the test's stack"; return -1; }
    if (start != SIZE_MAX && start >= view.node_count) { g_error = "start node out of range"; return -1; }
    DeviceBuf<typename Api<T>::Ray> d_rays; DeviceBuf<T> d_spheres, d_t; DeviceBuf<uint32_t> d_ids, d_leaves, d_inner; DeviceBuf<uint64_t> d_hashes;
    if (d_rays.upload(rays, n) || d_spheres.upload(spheres, leaf == kLeafSphere ? 4 * view.prim_count : 0) || d_ids.alloc(n) ||
        d_t.alloc(n) || d_leaves.alloc(n) || d_hashes.alloc(n) || d_inner.alloc(n)) return -1;
    const bool any = flags & BVH_ANY_HIT, robust = flags & BVH_ROBUST;
    if (n) {
        if (any) { if (robust) launch_record<T, true, true>(leaf, view, d_rays.p, n, d_spheres.p, start, d_ids.p, d_t.p, d_leaves.p, d_hashes.p, d_inner.p);
                   else        launch_record<T, true, false>(leaf, view, d_rays.p, n, d_spheres.p, start, d_ids.p, d_t.p, d_leaves.p, d_hashes.p, d_inner.p); }
        else     { if (robust) launch_record<T, false, true>(leaf, view, d_rays.p, n, d_spheres.p, start, d_ids.p, d_t.p, d_leaves.p, d_hashes.p, d_inner.p);
                   else        launch_record<T, false, false>(leaf, view, d_rays.p, n, d_spheres.p, start, d_ids.p, d_t.p, d_leaves.p, d_hashes.p, d_inner.p); }
        DAPI_TRY(cudaGetLastError());
    }
    DAPI_TRY(cudaDeviceSynchronize());
    if (d_ids.download(ids, n) || d_t.download(t, n) || d_leaves.download(leaves, n) || d_hashes.download(hashes, n) ||
        d_inner.download(inner, n)) return -1;
    return 0;
}

// The same leaves through Bvh<Node>::intersect (include/bvh/v2/b200_surface.h) on the handle's host mirror.
// verts: prim_count x 9 in original order (leaf kTri only).
template <typename T>
int host_record(typename Api<T>::Handle* h, int leaf, const typename Api<T>::Ray* rays, size_t n, const T* verts, const T* spheres,
                size_t start, unsigned flags, uint32_t* ids, T* t, uint32_t* leaves, uint64_t* hashes, uint32_t* inner) {
    using Node = bvh::v2::Node<T, 3>;
    using Vec3 = bvh::v2::Vec<T, 3>;
    if (!h || !rays || (leaf == kLeafTri && !verts) || (leaf == kLeafSphere && !spheres)) { g_error = "null argument"; return -1; }
    bvh::v2::Bvh<Node> bvh;
    bvh.nodes.resize(Api<T>::node_count(h));
    if (bvh.nodes.empty()) { g_error = bvh_last_error(); return -1; }
    std::memcpy(bvh.nodes.data(), Api<T>::node0(h), bvh.nodes.size() * sizeof(Node));
    bvh.prim_ids.assign(Api<T>::prim_ids(h), Api<T>::prim_ids(h) + Api<T>::prim_count(h));
    if (start != SIZE_MAX && start >= bvh.nodes.size()) { g_error = "start node out of range"; return -1; }
    std::vector<bvh::v2::PrecomputedTri<T>> tris;
    if (leaf == kLeafTri) {
        tris.resize(bvh.prim_ids.size());
        for (size_t k = 0; k < tris.size(); ++k) {
            const T* v = verts + 9 * bvh.prim_ids[k];
            tris[k] = bvh::v2::PrecomputedTri<T>(Vec3(v[0], v[1], v[2]), Vec3(v[3], v[4], v[5]), Vec3(v[6], v[7], v[8]));
        }
    }
    const bool any = flags & BVH_ANY_HIT, robust = flags & BVH_ROBUST;
    for (size_t i = 0; i < n; ++i) {
        const auto& rp = rays[i];
        bvh::v2::Ray<T, 3> ray(Vec3(rp.org.x, rp.org.y, rp.org.z), Vec3(rp.dir.x, rp.dir.y, rp.dir.z), rp.tmin, rp.tmax);
        const T org[3] = { rp.org.x, rp.org.y, rp.org.z }, dir[3] = { rp.dir.x, rp.dir.y, rp.dir.z };
        bvh::v2::GrowingStack<typename Node::Index> stack;
        size_t best = SIZE_MAX;
        uint32_t calls = 0, steps = 0;
        uint64_t hh = kHashSeed;
        auto leaf_fn = [&](size_t begin, size_t end) {
            ++calls;
            hh = mix(mix(hh, begin), end);
            for (size_t k = begin; k < end; ++k) {
                if (leaf == kLeafTri) {
                    if (auto hit = tris[k].intersect(ray)) { ray.tmax = std::get<0>(*hit); best = k; }
                } else if (leaf == kLeafSphere) {
                    const size_t id = bvh.prim_ids[k];
                    T t0, t1;
                    if (sphere_hit<T>(spheres + 4 * id, spheres[4 * id + 3], org, dir, ray.tmin, ray.tmax, t0, t1)) { ray.tmax = t0; best = k; }
                }
            }
            return best != SIZE_MAX;
        };
        auto inner_fn = [&](const Node&, const Node&) { ++steps; };
        const auto root = start == SIZE_MAX ? bvh.get_root().index : bvh.nodes[start].index;
        if (any) { if (robust) bvh.template intersect<true, true>(ray, root, stack, leaf_fn, inner_fn);
                   else        bvh.template intersect<true, false>(ray, root, stack, leaf_fn, inner_fn); }
        else     { if (robust) bvh.template intersect<false, true>(ray, root, stack, leaf_fn, inner_fn);
                   else        bvh.template intersect<false, false>(ray, root, stack, leaf_fn, inner_fn); }
        ids[i] = best == SIZE_MAX ? 0xFFFFFFFFu : (uint32_t)bvh.prim_ids[best];
        t[i] = ray.tmax;
        leaves[i] = calls; hashes[i] = hh; inner[i] = steps;
    }
    return 0;
}

// Times `steps` launches of the triangle kernel on device-resident rays (CUDA events); writes each launch's milliseconds.
template <typename T>
int bench(typename Api<T>::Handle* h, const typename Api<T>::Ray* d_rays, size_t n, unsigned flags, void* d_hits_scratch,
          int steps, float* ms) {
    DeviceView<T> view;
    if (get_view(h, view, true)) return -1;
    cudaStream_t stream = static_cast<cudaStream_t>(view.stream);
    uint32_t* ids = static_cast<uint32_t*>(d_hits_scratch);
    T* t = reinterpret_cast<T*>(static_cast<unsigned char*>(d_hits_scratch) + n * sizeof(uint32_t) * 2);
    cudaEvent_t a, b;
    DAPI_TRY(cudaEventCreate(&a)); DAPI_TRY(cudaEventCreate(&b));
    int rc = 0;
    for (int s = 0; s < steps && !rc; ++s) {
        cudaEventRecord(a, stream);
        rc = trace_device<T>(view, d_rays, n, flags, ids, t, t + n, t + 2 * n, nullptr, stream);
        cudaEventRecord(b, stream);
        if (cudaEventSynchronize(b) != cudaSuccess) { g_error = "bench: launch failed"; rc = -1; }
        else cudaEventElapsedTime(ms + s, a, b);
    }
    cudaEventDestroy(a); cudaEventDestroy(b);
    return rc;
}

// bvh::v2::cuda::Accel<T>::device_view(capacity) on a handle built here: 1 when it threw std::length_error, 0 when it did not
template <typename T>
int accel_capacity_check(const T* verts, size_t n, size_t capacity, size_t* depth) {
    try {
        bvh::v2::cuda::Accel<T> accel(std::span<const bvh::v2::Tri<T, 3>>(reinterpret_cast<const bvh::v2::Tri<T, 3>*>(verts), n));
        *depth = accel.device_view().depth;
        try { (void)accel.device_view(capacity); } catch (const std::length_error&) { return 1; }
        return 0;
    } catch (const std::exception& e) {
        g_error = e.what();
        return -1;
    }
}

} // namespace

#define DAPI_EXPORT extern "C" __attribute__((visibility("default")))
#define DAPI_ENTRY(T, S)                                                                                               \
    DAPI_EXPORT int dapi_trace##S(bvh##S* h, const bvh_ray##S* rays, size_t n, unsigned flags, uint32_t* ids, T* t, T* u, \
                                  T* v, uint32_t* inner) { return trace<T>(h, rays, n, flags, ids, t, u, v, inner); }   \
    DAPI_EXPORT int dapi_record##S(bvh##S* h, int leaf, const bvh_ray##S* rays, size_t n, const T* spheres, size_t start, \
                                   unsigned flags, uint32_t* ids, T* t, uint32_t* leaves, uint64_t* hashes, uint32_t* inner) { \
        return record<T>(h, leaf, rays, n, spheres, start, flags, ids, t, leaves, hashes, inner); }                      \
    DAPI_EXPORT int dapi_host_record##S(bvh##S* h, int leaf, const bvh_ray##S* rays, size_t n, const T* verts, const T* spheres, \
                                        size_t start, unsigned flags, uint32_t* ids, T* t, uint32_t* leaves, uint64_t* hashes, \
                                        uint32_t* inner) {                                                              \
        return host_record<T>(h, leaf, rays, n, verts, spheres, start, flags, ids, t, leaves, hashes, inner); }          \
    DAPI_EXPORT int dapi_bench##S(bvh##S* h, const bvh_ray##S* d_rays, size_t n, unsigned flags, void* d_scratch, int steps, \
                                  float* ms) { return bench<T>(h, d_rays, n, flags, d_scratch, steps, ms); }            \
    DAPI_EXPORT int dapi_accel_capacity_check##S(const T* verts, size_t n, size_t capacity, size_t* depth) {           \
        return accel_capacity_check<T>(verts, n, capacity, depth); }

DAPI_ENTRY(float, 3f)
DAPI_ENTRY(double, 3d)

DAPI_EXPORT const char* dapi_last_error() { return g_error.c_str(); }
