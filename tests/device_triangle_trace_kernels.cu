// tests/device_triangle_trace_kernels.cu — test shaders for DeviceView::trace_triangles (include/bvh/v2/cuda/intersect.cuh).
//
// Compiled for sm_90a with the library's NVCC_FLAGS (--fmad=false among them) into
// tests/_build/libdevice_triangle_trace_kernels.so (bvh_b200/build_ext.py build_device_triangle_trace_tests) and driven
// by tests/test_device_triangle_trace_gpu.py and scripts/triangle_trace_bench.py.  Every array is device-resident.
//   dtt_run{3f,3d}      one batch of rays from an array, through DeviceView::trace_triangles (per_thread = 0) or through a
//                       kernel of one thread per ray calling DeviceView::intersect with a leaf built from intersect_tri,
//                       the same tie rule and the same filter (per_thread = 1).  Filters: 0 accept all, 1 reject all,
//                       2 reject odd ids, 3 an alpha cut-out on (u, v), 4 reject the ray's origin triangle (origins[i]).
//                       Flags: BVH_ANY_HIT, BVH_ROBUST, BVH_TIE_LAST_VISITED.  Per ray i it writes, for every output
//                       that is not null: the record's id (all ones: none), t, u, v, the accept-call count, a 64-bit
//                       hash of the accept sequence (original id and the bits of t, u, v), and it adds 1 to counts[i].
//   dtt_plain3f         the float closest-hit, canonical-tie, accept-all shader with an empty payload: rays from an array,
//                       16-byte records to an array, as bvh3f_intersect_rays writes them.
//   dtt_camera3f        a pinhole camera computes ray i from i inside the shader; finish writes only t (depth).
//   dtt_camera_rays3f   the same camera's rays written to an array by a kernel of its own.
// Each returns 0; -1 with a message in dtt_last_error(); -2 when the call threw std::length_error, -3 when it threw
// std::invalid_argument, with its message.
#include <cuda_runtime.h>

#include <bvh/v2/cuda/intersect.cuh>

#include <cstdint>
#include <stdexcept>
#include <string>

namespace {

using bvh::v2::cuda::DeviceView;

thread_local std::string g_error;
constexpr unsigned kBlock = 128;
constexpr uint32_t kNone = 0xFFFFFFFFu;

enum Filter : int { kAll = 0, kRejectAll, kEvenIds, kAlpha, kNotOrigin };

template <typename T> struct Api;
template <> struct Api<float> {
    using Handle = bvh3f; using View = bvh_device_view3f;
    static int view(Handle* h, View* v) { return bvh3f_get_device_view(h, v); }
};
template <> struct Api<double> {
    using Handle = bvh3d; using View = bvh_device_view3d;
    static int view(Handle* h, View* v) { return bvh3d_get_device_view(h, v); }
};

__host__ __device__ inline uint64_t mix(uint64_t h, uint64_t x) { return (h ^ x) * 1099511628211ull; }
constexpr uint64_t kHashSeed = 1469598103934665603ull;
__device__ inline uint64_t bits(float x) { return __float_as_uint(x); }
__device__ inline uint64_t bits(double x) { return (uint64_t)__double_as_longlong(x); }

template <int kFilter, typename T> __device__ inline bool keep(size_t id, T u, T v, uint32_t origin) {
    if (kFilter == kRejectAll) return false;
    if (kFilter == kEvenIds) return (id & 1) == 0;
    if (kFilter == kAlpha) return u < T(0.5) || v < T(0.25);     // the corner u >= 0.5, v >= 0.25 is cut out
    if (kFilter == kNotOrigin) return id != origin;
    return true;
}

template <typename T> struct Outputs {
    uint32_t* ids; T* t; T* u; T* v; uint32_t* calls; uint64_t* hashes; uint32_t* counts;
};

template <typename T> __device__ inline void write(const Outputs<T>& out, size_t i, uint32_t id, T t, T u, T v, uint32_t calls,
                                                   uint64_t hash) {
    if (out.ids) out.ids[i] = id;
    if (out.t) out.t[i] = t;
    if (out.u) { out.u[i] = u; out.v[i] = v; }
    if (out.calls) out.calls[i] = calls;
    if (out.hashes) out.hashes[i] = hash;
    if (out.counts) atomicAdd(out.counts + i, 1u);
}

// The recording shader: rays from an array, the filter chosen by kFilter, the record to Outputs.
template <typename T, int kFilter> struct TestShader {
    using View = DeviceView<T>;
    using Ray = typename View::Ray;
    struct Payload { uint32_t origin, calls; uint64_t hash; };
    const Ray* rays;
    const uint32_t* origins;            // per ray, or null
    Outputs<T> out;

    __device__ Ray start(size_t i, Payload& p) const {
        p.origin = origins ? origins[i] : kNone; p.calls = 0; p.hash = kHashSeed;
        return rays[i];
    }
    __device__ bool accept(Payload& p, size_t prim_id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(p.hash, prim_id), bits(t)), bits(u)), bits(v));
        return keep<kFilter>(prim_id, u, v, p.origin);
    }
    __device__ void finish(size_t i, const Payload& p, const typename View::Hit& hit) const {
        write(out, i, (uint32_t)hit.prim_id, hit.t, hit.u, hit.v, p.calls, p.hash);
    }
};

// The same shader, one thread per ray through DeviceView::intersect: a leaf of intersect_tri calls, the tie rule and the
// filter, as a user kernel without trace_triangles writes it.
template <typename T, bool kAny, bool kRobust, bool kLast, int kFilter>
__global__ void __launch_bounds__(kBlock) per_thread_kernel(DeviceView<T> view, TestShader<T, kFilter> shader, size_t n) {
    using Shader = TestShader<T, kFilter>;
    extern __shared__ __align__(128) unsigned char smem[];
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (i >= n) return;
    auto stack = DeviceView<T>::shared_stack(smem, kBlock);
    typename Shader::Payload p;
    typename Shader::Ray ray = shader.start(i, p);
    const T tmax_in = ray.tmax;
    size_t best = SIZE_MAX;
    T bu = T(0), bv = T(0);
    view.template intersect<kAny, kRobust>(ray, view.root_index(), stack, [&](size_t begin, size_t end) {
        for (size_t k = begin; k < end; ++k) {
            T t, u, v;
            if (!view.intersect_tri(k, ray, t, u, v)) continue;
            const size_t id = view.prim_id(k);
            if (!kLast && best != SIZE_MAX && !(t < ray.tmax) && !(id < view.prim_id(best))) continue;   // canonical tie rule
            ++p.calls;
            p.hash = mix(mix(mix(mix(p.hash, id), bits(t)), bits(u)), bits(v));
            if (!keep<kFilter>(id, u, v, p.origin)) continue;
            ray.tmax = t; best = k; bu = u; bv = v;
        }
        return best != SIZE_MAX;
    });
    const bool hit = best != SIZE_MAX;
    write(shader.out, i, hit ? (uint32_t)view.prim_id(best) : kNone, hit ? ray.tmax : tmax_in, bu, bv, p.calls, p.hash);
}

template <typename T, bool kAny, bool kRobust, bool kLast, int kFilter>
int run_filter(const DeviceView<T>& view, bool per_thread, size_t n, const void* rays, const uint32_t* origins,
               const Outputs<T>& out, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    using Shader = TestShader<T, kFilter>;
    const Shader shader { static_cast<const typename Shader::Ray*>(rays), origins, out };
    if (!per_thread) {
        view.template trace_triangles<kAny, kRobust, kLast>(n, shader, workspace, workspace_bytes, stream);
        return 0;
    }
    if (n == 0) return 0;
    const size_t smem = view.shared_stack_bytes(kBlock);
    auto kernel = per_thread_kernel<T, kAny, kRobust, kLast, kFilter>;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) {
        kernel<<<(unsigned)((n + kBlock - 1) / kBlock), kBlock, smem, stream>>>(view, shader, n);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { g_error = std::string("per-thread kernel: ") + cudaGetErrorString(e); return -1; }
    return 0;
}

template <typename T, bool kAny, bool kRobust, bool kLast>
int run_flags(int filter, const DeviceView<T>& view, bool per_thread, size_t n, const void* rays, const uint32_t* origins,
              const Outputs<T>& out, void* ws, size_t bytes, cudaStream_t s) {
    switch (filter) {
    case kAll: return run_filter<T, kAny, kRobust, kLast, kAll>(view, per_thread, n, rays, origins, out, ws, bytes, s);
    case kRejectAll: return run_filter<T, kAny, kRobust, kLast, kRejectAll>(view, per_thread, n, rays, origins, out, ws, bytes, s);
    case kEvenIds: return run_filter<T, kAny, kRobust, kLast, kEvenIds>(view, per_thread, n, rays, origins, out, ws, bytes, s);
    case kAlpha: return run_filter<T, kAny, kRobust, kLast, kAlpha>(view, per_thread, n, rays, origins, out, ws, bytes, s);
    case kNotOrigin: return run_filter<T, kAny, kRobust, kLast, kNotOrigin>(view, per_thread, n, rays, origins, out, ws, bytes, s);
    }
    g_error = "no such filter";
    return -1;
}

// The errors of a call, as return codes (see the top of this file)
template <typename F> int guarded(F&& f) {
    try {
        return f();
    } catch (const std::length_error& e) {
        g_error = e.what();
        return -2;
    } catch (const std::invalid_argument& e) {
        g_error = e.what();
        return -3;
    } catch (const std::exception& e) {
        g_error = e.what();
        return -1;
    }
}

template <typename T> bool get_view(typename Api<T>::Handle* h, DeviceView<T>& view) {
    typename Api<T>::View c {};
    if (Api<T>::view(h, &c)) { g_error = bvh_last_error(); return false; }
    view = DeviceView<T>::from(c);
    return true;
}

template <typename T>
int run(typename Api<T>::Handle* h, int per_thread, int filter, unsigned flags, const void* rays, size_t n, const uint32_t* origins,
        Outputs<T> out, void* ws, size_t bytes, void* stream) {
    DeviceView<T> view;
    if (!get_view<T>(h, view)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : view.stream);
    const bool any = flags & BVH_ANY_HIT, robust = flags & BVH_ROBUST, last = flags & BVH_TIE_LAST_VISITED;
    return guarded([&] {
        const int k = (any ? 1 : 0) | (robust ? 2 : 0) | (last ? 4 : 0);
        switch (k) {
        case 0: return run_flags<T, false, false, false>(filter, view, per_thread, n, rays, origins, out, ws, bytes, s);
        case 1: return run_flags<T, true, false, false>(filter, view, per_thread, n, rays, origins, out, ws, bytes, s);
        case 2: return run_flags<T, false, true, false>(filter, view, per_thread, n, rays, origins, out, ws, bytes, s);
        case 3: return run_flags<T, true, true, false>(filter, view, per_thread, n, rays, origins, out, ws, bytes, s);
        case 4: return run_flags<T, false, false, true>(filter, view, per_thread, n, rays, origins, out, ws, bytes, s);
        case 5: return run_flags<T, true, false, true>(filter, view, per_thread, n, rays, origins, out, ws, bytes, s);
        case 6: return run_flags<T, false, true, true>(filter, view, per_thread, n, rays, origins, out, ws, bytes, s);
        default: return run_flags<T, true, true, true>(filter, view, per_thread, n, rays, origins, out, ws, bytes, s);
        }
    });
}

// The smallest shader: rays in, the library's records out, nothing per ray beyond the traversal's own state.
struct PlainShader {
    struct Payload {};
    const bvh_ray3f* rays;
    bvh_hit3f* hits;
    __device__ bvh_ray3f start(size_t i, Payload&) const { return rays[i]; }
    __device__ bool accept(Payload&, size_t, float, float, float) const { return true; }
    __device__ void finish(size_t i, const Payload&, const bvh_hit3f& hit) const { hits[i] = hit; }
};

// A pinhole camera at `eye` looking along +z through a [x0, x1] x [y0, y1] window at z = eye.z + 1: ray i is pixel
// (i % width, i / width), through the pixel's centre.
struct Camera {
    float eye[3];
    float x0, x1, y0, y1;
    uint32_t width, height;
};
__device__ inline bvh_ray3f camera_ray(const Camera& c, size_t i) {
    const uint32_t px = (uint32_t)(i % c.width), py = (uint32_t)(i / c.width);
    const float sx = __fdiv_rn(__fadd_rn((float)px, 0.5f), (float)c.width), sy = __fdiv_rn(__fadd_rn((float)py, 0.5f), (float)c.height);
    bvh_ray3f r;
    r.org.x = c.eye[0]; r.org.y = c.eye[1]; r.org.z = c.eye[2];
    r.dir.x = __fsub_rn(__fadd_rn(c.x0, __fmul_rn(sx, __fsub_rn(c.x1, c.x0))), c.eye[0]);
    r.dir.y = __fsub_rn(__fadd_rn(c.y0, __fmul_rn(sy, __fsub_rn(c.y1, c.y0))), c.eye[1]);
    r.dir.z = 1.0f;
    r.tmin = 0.0f; r.tmax = INFINITY;
    return r;
}
struct CameraShader {
    struct Payload {};
    Camera camera;
    float* depth;
    __device__ bvh_ray3f start(size_t i, Payload&) const { return camera_ray(camera, i); }
    __device__ bool accept(Payload&, size_t, float, float, float) const { return true; }
    __device__ void finish(size_t i, const Payload&, const bvh_hit3f& hit) const { depth[i] = hit.t; }
};
__global__ void camera_rays_kernel(Camera c, size_t n, bvh_ray3f* rays) {
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) rays[i] = camera_ray(c, i);
}

} // namespace

#define DTT_EXPORT extern "C" __attribute__((visibility("default")))
#define DTT_ENTRY(T, S)                                                                                                   \
    DTT_EXPORT int dtt_run##S(bvh##S* h, int per_thread, int filter, unsigned flags, const void* rays, size_t n,          \
                              const uint32_t* origins, uint32_t* ids, T* t, T* u, T* v, uint32_t* calls, uint64_t* hashes, \
                              uint32_t* counts, void* workspace, size_t workspace_bytes, void* stream) {                   \
        return run<T>(h, per_thread, filter, flags, rays, n, origins, Outputs<T> { ids, t, u, v, calls, hashes, counts },   \
                      workspace, workspace_bytes, stream);                                                               \
    }

DTT_ENTRY(float, 3f)
DTT_ENTRY(double, 3d)

DTT_EXPORT int dtt_plain3f(bvh3f* h, const void* rays, size_t n, void* hits, void* workspace, size_t workspace_bytes, void* stream) {
    DeviceView<float> view;
    if (!get_view<float>(h, view)) return -1;
    return guarded([&] {
        view.trace_triangles<false, false>(n, PlainShader { static_cast<const bvh_ray3f*>(rays), static_cast<bvh_hit3f*>(hits) },
                                           workspace, workspace_bytes, stream ? stream : view.stream);
        return 0;
    });
}

DTT_EXPORT int dtt_camera3f(bvh3f* h, const float* camera, uint32_t width, uint32_t height, float* depth, void* workspace,
                            size_t workspace_bytes, void* stream) {
    DeviceView<float> view;
    if (!get_view<float>(h, view)) return -1;
    const Camera c { { camera[0], camera[1], camera[2] }, camera[3], camera[4], camera[5], camera[6], width, height };
    return guarded([&] {
        view.trace_triangles<false, false>((size_t)width * height, CameraShader { c, depth }, workspace, workspace_bytes,
                                           stream ? stream : view.stream);
        return 0;
    });
}

DTT_EXPORT int dtt_camera_rays3f(const float* camera, uint32_t width, uint32_t height, void* rays, void* stream) {
    const Camera c { { camera[0], camera[1], camera[2] }, camera[3], camera[4], camera[5], camera[6], width, height };
    const size_t n = (size_t)width * height;
    if (n == 0) return 0;
    camera_rays_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(c, n, static_cast<bvh_ray3f*>(rays));
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { g_error = cudaGetErrorString(e); return -1; }
    return 0;
}

DTT_EXPORT size_t dtt_workspace_bytes3f(bvh3f* h) {
    DeviceView<float> view;
    return get_view<float>(h, view) ? view.trace_workspace_bytes() : 0;
}

DTT_EXPORT const char* dtt_last_error() { return g_error.c_str(); }
