// tests/device_trace_kernels.cu — test tracers for DeviceView::trace (include/bvh/v2/cuda/intersect.cuh).
//
// Compiled for sm_90a with the library's NVCC_FLAGS (--fmad=false among them) into
// tests/_build/libdevice_trace_kernels.so (bvh_b200/build_ext.py build_device_trace_tests) and driven by
// tests/test_device_trace_gpu.py and scripts/device_api_bench.py.  Every array is device-resident.
//   dtr_run{3f,3d}    one batch with the test tracer, through DeviceView::trace (per_thread = 0) or through a kernel of one
//                     thread per ray calling DeviceView::intersect with the same leaf and a shared-memory stack
//                     (per_thread = 1).  Leaves: 0 none, 1 the triangle test (DeviceView::intersect_tri), 2 the
//                     reference's sphere test, 3 the triangle test that makes the interval NaN on its second call.  Per
//                     ray i it writes, for every output that is not null: the hit's original id (all ones: none), the
//                     final tmax, the hit's barycentrics (triangle leaves), the leaf-call count, a 64-bit hash of the
//                     (begin, end) sequence, and it adds 1 to counts[i].  Returns 0; -1 with a message in
//                     dtr_last_error(); -2 when trace threw std::length_error, with its message.
#include <cuda_runtime.h>

#include <bvh/v2/cuda/intersect.cuh>

#include <cmath>
#include <cstdint>
#include <stdexcept>
#include <string>

namespace {

using bvh::v2::cuda::DeviceView;

thread_local std::string g_error;
constexpr unsigned kBlock = 128;

enum Leaf : int { kLeafNone = 0, kLeafTri = 1, kLeafSphere = 2, kLeafTriNan = 3 };

template <typename T> struct Api;
template <> struct Api<float> {
    using Handle = bvh3f; using View = bvh_device_view3f;
    static int view(Handle* h, View* v) { return bvh3f_get_device_view(h, v); }
};
template <> struct Api<double> {
    using Handle = bvh3d; using View = bvh_device_view3d;
    static int view(Handle* h, View* v) { return bvh3d_get_device_view(h, v); }
};

// reference sphere.h:15-50 (Sphere::intersect, AssumeNormalized = false): the same arithmetic as
// tests/device_api_kernels.cu sphere_hit
template <typename T>
__device__ inline bool sphere_hit(const T* c, T radius, const T org[3], const T dir[3], T tmin, T tmax, T& t0, T& t1) {
    const T oc[3] = { org[0] - c[0], org[1] - c[1], org[2] - c[2] };
    auto dot = [] (const T* a, const T* b) { T s = T(0) + a[0] * b[0]; s = s + a[1] * b[1]; return s + a[2] * b[2]; };
    const T a = dot(dir, dir);
    const T b = T(2.) * dot(dir, oc);
    const T cc = dot(oc, oc) - radius * radius;
    const T delta = b * b - T(4.) * a * cc;
    if (delta >= 0) {
        const T inv = -T(0.5) / a;
        const T sqrt_delta = sqrt(delta);
        const T n0 = (b + sqrt_delta) * inv, n1 = (b - sqrt_delta) * inv;
        t0 = n0 > tmin ? n0 : tmin;
        t1 = n1 < tmax ? n1 : tmax;
        if (t0 <= t1) return true;
    }
    return false;
}

__device__ inline uint64_t mix(uint64_t h, uint64_t x) { return (h ^ x) * 1099511628211ull; }
constexpr uint64_t kHashSeed = 1469598103934665603ull;

template <typename T> struct Outputs {
    uint32_t* ids; T* t; T* u; T* v; uint32_t* calls; uint64_t* hashes; uint32_t* counts;
};

// The test tracer: rays from an array, the leaf chosen by kLeaf, the record to Outputs.
template <typename T, int kLeaf> struct TestTracer {
    using Ray = typename DeviceView<T>::Ray;
    struct Payload { size_t best; T u, v; uint32_t calls; uint64_t hash; };
    DeviceView<T> view;
    const Ray* rays;
    const T* spheres;          // prim_count x {cx, cy, cz, radius}, original order
    Outputs<T> out;

    __device__ Ray start(size_t i, Payload& p) const {
        p.best = SIZE_MAX; p.u = p.v = T(0); p.calls = 0; p.hash = kHashSeed;
        return rays[i];
    }
    __device__ bool leaf(Payload& p, Ray& ray, size_t begin, size_t end) const {
        ++p.calls;
        p.hash = mix(mix(p.hash, begin), end);
        for (size_t k = begin; k < end; ++k) {
            if (kLeaf == kLeafTri || kLeaf == kLeafTriNan) {
                T t, u, v;
                if (view.intersect_tri(k, ray, t, u, v)) { ray.tmax = t; p.best = k; p.u = u; p.v = v; }
            } else if (kLeaf == kLeafSphere) {
                const size_t id = view.prim_id(k);
                const T org[3] = { ray.org.x, ray.org.y, ray.org.z }, dir[3] = { ray.dir.x, ray.dir.y, ray.dir.z };
                T t0, t1;
                if (sphere_hit<T>(spheres + 4 * id, spheres[4 * id + 3], org, dir, ray.tmin, ray.tmax, t0, t1)) { ray.tmax = t0; p.best = k; }
            }
        }
        if (kLeaf == kLeafTriNan && p.calls == 2) ray.tmax = T(NAN);
        return p.best != SIZE_MAX;
    }
    __device__ void finish(size_t i, const Payload& p, const Ray& ray) const {
        if (out.ids) out.ids[i] = p.best == SIZE_MAX ? 0xFFFFFFFFu : (uint32_t)view.prim_id(p.best);
        if (out.t) out.t[i] = ray.tmax;
        if (out.u) { out.u[i] = p.u; out.v[i] = p.v; }
        if (out.calls) out.calls[i] = p.calls;
        if (out.hashes) out.hashes[i] = p.hash;
        if (out.counts) atomicAdd(out.counts + i, 1u);
    }
};

// The same tracer, one thread per ray through DeviceView::intersect (what a user kernel without trace looks like).
template <typename T, bool kAny, bool kRobust, typename Tracer>
__global__ void __launch_bounds__(kBlock) per_thread_kernel(Tracer tracer, size_t n) {
    extern __shared__ __align__(128) unsigned char smem[];
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (i >= n) return;
    auto stack = DeviceView<T>::shared_stack(smem, kBlock);
    typename Tracer::Payload p;
    typename Tracer::Ray ray = tracer.start(i, p);
    tracer.view.template intersect<kAny, kRobust>(ray, tracer.view.root_index(), stack,
                                                  [&](size_t begin, size_t end) { return tracer.leaf(p, ray, begin, end); });
    tracer.finish(i, p, ray);
}

template <typename T, bool kAny, bool kRobust, int kLeaf>
int run_leaf(const DeviceView<T>& view, bool per_thread, size_t n, const void* rays, const T* spheres, const Outputs<T>& out,
             void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    using Tracer = TestTracer<T, kLeaf>;
    const Tracer tracer { view, static_cast<const typename Tracer::Ray*>(rays), spheres, out };
    if (!per_thread) {
        view.template trace<kAny, kRobust>(n, tracer, workspace, workspace_bytes, stream);
        return 0;
    }
    if (n == 0) return 0;
    const size_t smem = view.shared_stack_bytes(kBlock);
    cudaError_t e = cudaFuncSetAttribute(per_thread_kernel<T, kAny, kRobust, Tracer>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) {
        per_thread_kernel<T, kAny, kRobust, Tracer><<<(unsigned)((n + kBlock - 1) / kBlock), kBlock, smem, stream>>>(tracer, n);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { g_error = std::string("per-thread kernel: ") + cudaGetErrorString(e); return -1; }
    return 0;
}

template <typename T, bool kAny, bool kRobust>
int run_flags(int leaf, const DeviceView<T>& view, bool per_thread, size_t n, const void* rays, const T* spheres,
              const Outputs<T>& out, void* workspace, size_t bytes, cudaStream_t stream) {
    switch (leaf) {
    case kLeafNone: return run_leaf<T, kAny, kRobust, kLeafNone>(view, per_thread, n, rays, spheres, out, workspace, bytes, stream);
    case kLeafTri: return run_leaf<T, kAny, kRobust, kLeafTri>(view, per_thread, n, rays, spheres, out, workspace, bytes, stream);
    case kLeafSphere: return run_leaf<T, kAny, kRobust, kLeafSphere>(view, per_thread, n, rays, spheres, out, workspace, bytes, stream);
    case kLeafTriNan: return run_leaf<T, kAny, kRobust, kLeafTriNan>(view, per_thread, n, rays, spheres, out, workspace, bytes, stream);
    }
    g_error = "no such leaf";
    return -1;
}

template <typename T>
int run(typename Api<T>::Handle* h, int per_thread, int leaf, unsigned flags, const void* rays, size_t n, const T* spheres,
        Outputs<T> out, void* workspace, size_t workspace_bytes, void* stream) {
    typename Api<T>::View c {};
    if (Api<T>::view(h, &c)) { g_error = bvh_last_error(); return -1; }
    if ((leaf == kLeafTri || leaf == kLeafTriNan) && !c.tris) { g_error = "no triangles attached"; return -1; }
    const DeviceView<T> view = DeviceView<T>::from(c);
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : c.stream);
    const bool any = flags & BVH_ANY_HIT, robust = flags & BVH_ROBUST;
    try {
        if (any) return robust ? run_flags<T, true, true>(leaf, view, per_thread, n, rays, spheres, out, workspace, workspace_bytes, s)
                               : run_flags<T, true, false>(leaf, view, per_thread, n, rays, spheres, out, workspace, workspace_bytes, s);
        return robust ? run_flags<T, false, true>(leaf, view, per_thread, n, rays, spheres, out, workspace, workspace_bytes, s)
                      : run_flags<T, false, false>(leaf, view, per_thread, n, rays, spheres, out, workspace, workspace_bytes, s);
    } catch (const std::length_error& e) {
        g_error = e.what();
        return -2;
    } catch (const std::exception& e) {
        g_error = e.what();
        return -1;
    }
}

} // namespace

#define DTR_EXPORT extern "C" __attribute__((visibility("default")))
#define DTR_ENTRY(T, S)                                                                                                   \
    DTR_EXPORT int dtr_run##S(bvh##S* h, int per_thread, int leaf, unsigned flags, const void* rays, size_t n,            \
                              const T* spheres, uint32_t* ids, T* t, T* u, T* v, uint32_t* calls, uint64_t* hashes,        \
                              uint32_t* counts, void* workspace, size_t workspace_bytes, void* stream) {                   \
        return run<T>(h, per_thread, leaf, flags, rays, n, spheres, Outputs<T> { ids, t, u, v, calls, hashes, counts },     \
                      workspace, workspace_bytes, stream);                                                               \
    }                                                                                                                     \
    DTR_EXPORT size_t dtr_workspace_bytes##S(bvh##S* h) {                                                                 \
        bvh_device_view##S c {};                                                                                          \
        if (bvh##S##_get_device_view(h, &c)) return 0;                                                                    \
        return DeviceView<T>::from(c).trace_workspace_bytes();                                                            \
    }

DTR_ENTRY(float, 3f)
DTR_ENTRY(double, 3d)

DTR_EXPORT const char* dtr_last_error() { return g_error.c_str(); }
