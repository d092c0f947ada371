// tests/device_path_trace_kernels.cu — test shaders for DeviceView::trace_paths (include/bvh/v2/cuda/intersect.cuh).
//
// Compiled for sm_90a with the library's NVCC_FLAGS (--fmad=false among them) into
// tests/_build/libdevice_path_trace_kernels.so (bvh_b200/build_ext.py build_device_path_trace_tests) and driven by
// tests/test_device_path_trace_gpu.py and scripts/path_trace_bench.py.  Every array is device-resident.
//   dpt_tracer{3f,3d}    a grey diffuse path tracer with a point light and next-event estimation (PathTracer below), path i
//                        starting with primary ray i of an array, either
//                        as one DeviceView::trace_paths call (wavefront = 0) or as a wavefront loop of trace_triangles
//                        launches with the path state in arrays (wavefront = 1): per bounce one closest-hit pass and one
//                        occlusion pass over all n paths, a path that is not waiting for that kind of segment drawn as a
//                        NaN ray.  Per path it writes the radiance, the segment count and a 32-bit hash of the segment
//                        records.  The wavefront arm needs dpt_wavefront_bytes{3f,3d}(n) bytes of scratch.
//   dpt_record{3f,3d}    a recording shader whose paths follow scripted segments: path i runs counts[i] segments, segment
//                        k = offsets[i] + j traces rays[seg_ray[k]] as seg_kind[k] (1 Closest, 2 Occlusion).  Through
//                        trace_paths (per_thread = 0) or one thread per segment through DeviceView::intersect with a leaf
//                        of intersect_tri calls, the same tie rule and the same filter (per_thread = 1).  The filter
//                        drops ids with id % 3 == 1.  Per segment k, for every output that is not null: the record's id,
//                        t, u, v, the accept-call count and a 64-bit hash of the accept sequence.  Per path (trace_paths
//                        only): starts[i] and finishes[i] count the calls, done[i] is the segment count finish saw;
//                        bad_rays[0] counts next calls whose ray was not the scripted one.  depth > 0 replaces the
//                        view's depth (a tree the shared-memory stack cannot hold).
//   dpt_plain3f          the smallest path shader (PlainPaths): ray i as a closest-hit segment, then on a hit as an
//                        occlusion segment, both records to an array.
// Each returns 0; -1 with a message in dpt_last_error(); -2 when the call threw std::length_error, -3 when it threw
// std::invalid_argument, with its message.
#include <cuda_runtime.h>

#include <bvh/v2/cuda/intersect.cuh>

#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>

namespace {

using bvh::v2::cuda::DeviceView;
using bvh::v2::cuda::PathStep;

thread_local std::string g_error;
constexpr unsigned kBlock = 128;
constexpr uint32_t kNone = 0xFFFFFFFFu;

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
__device__ inline uint32_t mix32(uint32_t h, uint32_t x) { return (h ^ x) * 16777619u; }
__device__ inline uint32_t fold(uint64_t x) { return (uint32_t)x ^ (uint32_t)(x >> 32); }
// a 32-bit integer hash (lowbias32)
__device__ inline uint32_t hash32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}

template <typename T> __device__ inline bool same_ray(const T& a, const T& b) {
    return bits(a.org.x) == bits(b.org.x) && bits(a.org.y) == bits(b.org.y) && bits(a.org.z) == bits(b.org.z) &&
           bits(a.dir.x) == bits(b.dir.x) && bits(a.dir.y) == bits(b.dir.y) && bits(a.dir.z) == bits(b.dir.z) &&
           bits(a.tmin) == bits(b.tmin) && bits(a.tmax) == bits(b.tmax);
}

// ---------------------------------------------------------------------------------------------------------------------
// The path tracer
// ---------------------------------------------------------------------------------------------------------------------

// Grey diffuse surfaces (albedo kAlbedo) lit by a point light and a constant sky.  At every closest hit the light's
// share is computed; when the light is above the surface a shadow segment to it follows, and its share counts when the
// segment misses.  Then the path bounces in a direction drawn from a hash of (path, segment), up to max_bounces times.
// Every segment skips the triangle the path stands on.  The payload: the throughput, the radiance so far, the pending
// light share (non-zero while a shadow segment runs), the triangle the path stands on, the bounce count with the side of
// that triangle the path is on in bit 0, the segment count and the hash of the records.
template <typename T> struct PathTracer {
    using View = DeviceView<T>;
    using Ray = typename View::Ray;
    using Hit = typename View::Hit;
    struct Payload { T throughput, radiance, pending; uint32_t prim, bounce, segments, hash; };
    static constexpr T kAlbedo = T(0.7), kSky = T(0.25), kLight = T(2.0);

    const Ray* primary;                 // path i starts with primary[i]
    T light[3];
    const T* verts;                     // 9 per triangle, original order
    uint32_t max_bounces;
    T* radiance; uint32_t* segments; uint32_t* hashes;

    __device__ void normal(uint32_t prim, bool flip, T n[3]) const {
        const T* v = verts + 9 * (size_t)prim;
        const T e1[3] = { v[3] - v[0], v[4] - v[1], v[5] - v[2] }, e2[3] = { v[6] - v[0], v[7] - v[1], v[8] - v[2] };
        T c[3] = { e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0] };
        const T len = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
        const T s = flip ? T(-1) / len : T(1) / len;
        for (int a = 0; a < 3; ++a) n[a] = c[a] * s;
    }

    __device__ PathStep start(size_t i, Payload& p, Ray& ray) const {
        ray = primary[i];
        p.throughput = T(1); p.radiance = T(0); p.pending = T(0);
        p.prim = kNone; p.bounce = 0; p.segments = 0; p.hash = 2166136261u;
        return PathStep::Closest;
    }
    __device__ bool accept(Payload& p, size_t prim_id, T, T, T) const { return prim_id != p.prim; }

    // the next bounce from the surface point ray.org, or the path's end
    __device__ PathStep bounce(size_t i, Payload& p, Ray& ray) const {
        if ((p.bounce >> 1) >= max_bounces) return PathStep::End;
        const uint32_t h = hash32((uint32_t)i * 0x9E3779B9u ^ hash32(p.segments));
        const T u1 = T(h >> 16) * T(1.0 / 65536), u2 = T(h & 0xFFFFu) * T(1.0 / 65536);
        const T z = T(1) - T(2) * u1, rr = sqrt(fmax(T(0), T(1) - z * z)), phi = T(6.283185307179586) * u2;
        T d[3] = { rr * cos(phi), rr * sin(phi), z }, n[3];
        normal(p.prim, p.bounce & 1u, n);
        T c = d[0] * n[0] + d[1] * n[1] + d[2] * n[2];
        if (c < T(0)) { for (int a = 0; a < 3; ++a) d[a] = -d[a]; c = -c; }
        p.throughput = p.throughput * (T(2) * kAlbedo * c);
        p.bounce += 2;
        ray.dir.x = d[0]; ray.dir.y = d[1]; ray.dir.z = d[2];
        ray.tmin = T(0); ray.tmax = T(INFINITY);
        return PathStep::Closest;
    }

    __device__ PathStep next(size_t i, Payload& p, const Hit& hit, Ray& ray) const {
        ++p.segments;
        p.hash = mix32(mix32(mix32(mix32(p.hash, (uint32_t)hit.prim_id), fold(bits(hit.t))), fold(bits(hit.u))), fold(bits(hit.v)));
        const bool miss = hit.prim_id == (decltype(hit.prim_id))~(decltype(hit.prim_id))0;
        if (p.pending != T(0)) {                             // a shadow segment ended: ray.org is the surface point
            if (miss) p.radiance = p.radiance + p.pending;
            p.pending = T(0);
            return bounce(i, p, ray);
        }
        if (miss) { p.radiance = p.radiance + p.throughput * kSky; return PathStep::End; }
        p.prim = (uint32_t)hit.prim_id;
        const T x[3] = { ray.org.x + hit.t * ray.dir.x, ray.org.y + hit.t * ray.dir.y, ray.org.z + hit.t * ray.dir.z };
        T n[3];
        normal(p.prim, false, n);
        const bool flip = n[0] * ray.dir.x + n[1] * ray.dir.y + n[2] * ray.dir.z > T(0);   // face the incoming ray
        p.bounce = (p.bounce & ~1u) | (flip ? 1u : 0u);
        if (flip) for (int a = 0; a < 3; ++a) n[a] = -n[a];
        const T l[3] = { light[0] - x[0], light[1] - x[1], light[2] - x[2] };
        const T d2 = l[0] * l[0] + l[1] * l[1] + l[2] * l[2];
        const T c = n[0] * l[0] + n[1] * l[1] + n[2] * l[2];
        ray.org.x = x[0]; ray.org.y = x[1]; ray.org.z = x[2];
        if (c > T(0)) {
            p.pending = p.throughput * kAlbedo * kLight * c / (d2 * sqrt(d2));
            ray.dir.x = l[0]; ray.dir.y = l[1]; ray.dir.z = l[2];
            ray.tmin = T(0); ray.tmax = T(1);
            return PathStep::Occlusion;
        }
        return bounce(i, p, ray);
    }
    __device__ void finish(size_t i, const Payload& p) const {
        radiance[i] = p.radiance; segments[i] = p.segments; hashes[i] = p.hash;
    }
};

// The wavefront form of a path shader: the path state in arrays, one trace_triangles pass per segment kind.
template <typename Shader> struct WavefrontState {
    typename Shader::Ray* rays;
    typename Shader::Payload* payloads;
    uint8_t* steps;                     // the path's pending PathStep
};

template <typename Shader>
__global__ void wavefront_start_kernel(Shader shader, WavefrontState<Shader> st, size_t n) {
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    typename Shader::Payload p;
    typename Shader::Ray ray;
    const PathStep step = shader.start(i, p, ray);
    if (step == PathStep::End) shader.finish(i, p);
    st.rays[i] = ray; st.payloads[i] = p; st.steps[i] = (uint8_t)step;
}

// One pass: the paths waiting for a segment of kind `kind` trace it and run next; the others are NaN rays whose
// finish does nothing.
template <typename Shader> struct WavefrontPass {
    using T = typename Shader::View::Scalar;
    using Ray = typename Shader::Ray;
    struct Payload { typename Shader::Payload p; bool live; };
    Shader shader;
    WavefrontState<Shader> st;
    PathStep kind;

    __device__ Ray start(size_t i, Payload& q) const {
        q.live = st.steps[i] == (uint8_t)kind;
        if (q.live) { q.p = st.payloads[i]; return st.rays[i]; }
        Ray ray {};
        ray.tmin = ray.tmax = T(NAN);
        return ray;
    }
    __device__ bool accept(Payload& q, size_t prim_id, T t, T u, T v) const { return shader.accept(q.p, prim_id, t, u, v); }
    __device__ void finish(size_t i, const Payload& q, const typename Shader::Hit& hit) const {
        if (!q.live) return;
        typename Shader::Payload p = q.p;
        Ray ray = st.rays[i];
        const PathStep step = shader.next(i, p, hit, ray);
        if (step == PathStep::End) shader.finish(i, p);
        st.rays[i] = ray; st.payloads[i] = p; st.steps[i] = (uint8_t)step;
    }
};

template <typename Shader> size_t wavefront_bytes(size_t n) {
    return n * (sizeof(typename Shader::Ray) + sizeof(typename Shader::Payload) + 1) + 256;
}
template <typename Shader> WavefrontState<Shader> wavefront_state(void* scratch, size_t n) {
    unsigned char* b = static_cast<unsigned char*>(scratch);
    WavefrontState<Shader> st;
    st.rays = reinterpret_cast<typename Shader::Ray*>(b);
    st.payloads = reinterpret_cast<typename Shader::Payload*>(b + ((n * sizeof(typename Shader::Ray) + 127) & ~(size_t)127));
    st.steps = reinterpret_cast<uint8_t*>(st.payloads + n);
    return st;
}

// `passes` rounds of one closest-hit and one occlusion trace_triangles pass, all on `stream`, no host synchronisation
template <typename T, bool kRobust, bool kLast, typename Shader>
void run_wavefront(const DeviceView<T>& view, const Shader& shader, size_t n, uint32_t passes, void* scratch, void* ws,
                   size_t bytes, cudaStream_t s) {
    if (n == 0) return;
    const WavefrontState<Shader> st = wavefront_state<Shader>(scratch, n);
    wavefront_start_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(shader, st, n);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("wavefront start: ") + cudaGetErrorString(e));
    for (uint32_t k = 0; k < passes; ++k) {
        view.template trace_triangles<false, kRobust, kLast>(n, WavefrontPass<Shader> { shader, st, PathStep::Closest }, ws, bytes, s);
        view.template trace_triangles<true, kRobust, kLast>(n, WavefrontPass<Shader> { shader, st, PathStep::Occlusion }, ws, bytes, s);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// The recording shader
// ---------------------------------------------------------------------------------------------------------------------

template <typename T> __device__ inline bool keep(size_t id) { return id % 3 != 1; }

template <typename T> struct Outputs {
    uint32_t* ids; T* t; T* u; T* v; uint32_t* calls; uint64_t* hashes;
};

template <typename T> __device__ inline void write(const Outputs<T>& out, size_t k, uint32_t id, T t, T u, T v, uint32_t calls,
                                                   uint64_t hash) {
    if (out.ids) out.ids[k] = id;
    if (out.t) out.t[k] = t;
    if (out.u) { out.u[k] = u; out.v[k] = v; }
    if (out.calls) out.calls[k] = calls;
    if (out.hashes) out.hashes[k] = hash;
}

struct Script {
    const uint64_t* offsets;            // first segment of each path
    const uint32_t* counts;             // segments of each path
    const uint32_t* seg_ray;            // per segment: the ray's index in `rays`
    const uint8_t* seg_kind;            // per segment: 1 Closest, 2 Occlusion
};

template <typename T> struct RecordShader {
    using View = DeviceView<T>;
    using Ray = typename View::Ray;
    using Hit = typename View::Hit;
    struct Payload { uint32_t seg, calls; uint64_t hash; };
    const Ray* rays;
    Script script;
    Outputs<T> out;
    uint32_t* starts; uint32_t* finishes; uint32_t* done; unsigned long long* bad_rays;

    __device__ PathStep segment(size_t k, Ray& ray) const {
        ray = rays[script.seg_ray[k]];
        return (PathStep)script.seg_kind[k];
    }
    __device__ PathStep start(size_t i, Payload& p, Ray& ray) const {
        if (starts) atomicAdd(starts + i, 1u);
        p.seg = 0; p.calls = 0; p.hash = kHashSeed;
        return script.counts[i] ? segment(script.offsets[i], ray) : PathStep::End;
    }
    __device__ bool accept(Payload& p, size_t prim_id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(p.hash, prim_id), bits(t)), bits(u)), bits(v));
        return keep<T>(prim_id);
    }
    __device__ PathStep next(size_t i, Payload& p, const Hit& hit, Ray& ray) const {
        const size_t k = script.offsets[i] + p.seg;
        if (bad_rays && !same_ray(ray, rays[script.seg_ray[k]])) atomicAdd(bad_rays, 1ull);
        write(out, k, (uint32_t)hit.prim_id, hit.t, hit.u, hit.v, p.calls, p.hash);
        ++p.seg; p.calls = 0; p.hash = kHashSeed;
        return p.seg < script.counts[i] ? segment(k + 1, ray) : PathStep::End;
    }
    __device__ void finish(size_t i, const Payload& p) const {
        if (finishes) atomicAdd(finishes + i, 1u);
        if (done) done[i] = p.seg;
    }
};

// One thread per scripted segment through DeviceView::intersect: a leaf of intersect_tri calls, the tie rule and the
// filter, as a user kernel without trace_paths writes it.
template <typename T, bool kAny, bool kRobust, bool kLast>
__device__ void per_thread_segment(const DeviceView<T>& view, const RecordShader<T>& shader, size_t k,
                                   typename DeviceView<T>::SharedStack& stack) {
    typename RecordShader<T>::Ray ray = shader.rays[shader.script.seg_ray[k]];
    const T tmax_in = ray.tmax;
    size_t best = SIZE_MAX;
    T bu = T(0), bv = T(0);
    uint32_t calls = 0;
    uint64_t hash = kHashSeed;
    view.template intersect<kAny, kRobust>(ray, view.root_index(), stack, [&](size_t begin, size_t end) {
        for (size_t kk = begin; kk < end; ++kk) {
            T t, u, v;
            if (!view.intersect_tri(kk, ray, t, u, v)) continue;
            const size_t id = view.prim_id(kk);
            if (!kLast && best != SIZE_MAX && !(t < ray.tmax) && !(id < view.prim_id(best))) continue;   // canonical tie rule
            ++calls;
            hash = mix(mix(mix(mix(hash, id), bits(t)), bits(u)), bits(v));
            if (!keep<T>(id)) continue;
            ray.tmax = t; best = kk; bu = u; bv = v;
        }
        return best != SIZE_MAX;
    });
    const bool hit = best != SIZE_MAX;
    write(shader.out, k, hit ? (uint32_t)view.prim_id(best) : kNone, hit ? ray.tmax : tmax_in, bu, bv, calls, hash);
}

template <typename T, bool kRobust, bool kLast>
__global__ void __launch_bounds__(kBlock) per_thread_kernel(DeviceView<T> view, RecordShader<T> shader, size_t segments) {
    extern __shared__ __align__(128) unsigned char smem[];
    const size_t k = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (k >= segments) return;
    auto stack = DeviceView<T>::shared_stack(smem, kBlock);
    if (shader.script.seg_kind[k] == (uint8_t)PathStep::Occlusion) per_thread_segment<T, true, kRobust, kLast>(view, shader, k, stack);
    else per_thread_segment<T, false, kRobust, kLast>(view, shader, k, stack);
}

// The smallest path shader: ray i from an array as a closest-hit segment, then, on a hit, the same ray again as an
// occlusion segment; both records to an array (2 per path).  Its register use is what the kernel itself costs.
struct PlainPaths {
    struct Payload { uint32_t seg; };
    const bvh_ray3f* rays;
    bvh_hit3f* hits;
    __device__ PathStep start(size_t i, Payload& p, bvh_ray3f& ray) const { p.seg = 0; ray = rays[i]; return PathStep::Closest; }
    __device__ bool accept(Payload&, size_t, float, float, float) const { return true; }
    __device__ PathStep next(size_t i, Payload& p, const bvh_hit3f& hit, bvh_ray3f&) const {
        hits[2 * i + p.seg] = hit;
        return p.seg++ == 0 && hit.prim_id != kNone ? PathStep::Occlusion : PathStep::End;
    }
    __device__ void finish(size_t, const Payload&) const {}
};

// ---------------------------------------------------------------------------------------------------------------------
// Entry points
// ---------------------------------------------------------------------------------------------------------------------

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

// f.template operator()<kRobust, kLast>() for the flags' combination
template <typename F> int dispatch(unsigned flags, F&& f) {
    const bool robust = flags & BVH_ROBUST, last = flags & BVH_TIE_LAST_VISITED;
    if (!robust && !last) return f.template operator()<false, false>();
    if (robust && !last) return f.template operator()<true, false>();
    if (!robust) return f.template operator()<false, true>();
    return f.template operator()<true, true>();
}

template <typename T>
int tracer(typename Api<T>::Handle* h, int wavefront, unsigned flags, size_t n, const void* primary, const T* light, const T* verts, uint32_t max_bounces, T* radiance, uint32_t* segments, uint32_t* hashes, void* scratch,
           void* ws, size_t bytes, void* stream) {
    DeviceView<T> view;
    if (!get_view<T>(h, view)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : view.stream);
    PathTracer<T> shader;
    shader.primary = static_cast<const typename DeviceView<T>::Ray*>(primary);
    for (int a = 0; a < 3; ++a) shader.light[a] = light[a];
    shader.verts = verts; shader.max_bounces = max_bounces;
    shader.radiance = radiance; shader.segments = segments; shader.hashes = hashes;
    return guarded([&] {
        return dispatch(flags, [&]<bool kRobust, bool kLast>() {
            if (wavefront) run_wavefront<T, kRobust, kLast>(view, shader, n, max_bounces + 1, scratch, ws, bytes, s);
            else view.template trace_paths<kRobust, kLast>(n, shader, ws, bytes, s);
            return 0;
        });
    });
}

template <typename T>
int record(typename Api<T>::Handle* h, int per_thread, unsigned flags, size_t n, const void* rays, Script script, size_t segments,
           Outputs<T> out, uint32_t* starts, uint32_t* finishes, uint32_t* done, unsigned long long* bad_rays, size_t depth,
           void* ws, size_t bytes, void* stream) {
    DeviceView<T> view;
    if (!get_view<T>(h, view)) return -1;
    if (depth) view.depth = depth;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : view.stream);
    const RecordShader<T> shader { static_cast<const typename DeviceView<T>::Ray*>(rays), script, out, starts, finishes, done, bad_rays };
    return guarded([&] {
        return dispatch(flags, [&]<bool kRobust, bool kLast>() {
            if (!per_thread) {
                view.template trace_paths<kRobust, kLast>(n, shader, ws, bytes, s);
                return 0;
            }
            if (segments == 0) return 0;
            const size_t smem = view.shared_stack_bytes(kBlock);
            auto kernel = per_thread_kernel<T, kRobust, kLast>;
            cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e == cudaSuccess) {
                kernel<<<(unsigned)((segments + kBlock - 1) / kBlock), kBlock, smem, s>>>(view, shader, segments);
                e = cudaGetLastError();
            }
            if (e != cudaSuccess) { g_error = std::string("per-thread kernel: ") + cudaGetErrorString(e); return -1; }
            return 0;
        });
    });
}

} // namespace

#define DPT_EXPORT extern "C" __attribute__((visibility("default")))
#define DPT_ENTRY(T, S)                                                                                                        \
    DPT_EXPORT int dpt_tracer##S(bvh##S* h, int wavefront, unsigned flags, size_t n, const void* primary, const T* light,      \
                                 const T* verts, uint32_t max_bounces, T* radiance, uint32_t* segments,       \
                                 uint32_t* hashes, void* scratch, void* workspace, size_t workspace_bytes, void* stream) {    \
        return tracer<T>(h, wavefront, flags, n, primary, light, verts, max_bounces, radiance, segments, hashes,     \
                         scratch, workspace, workspace_bytes, stream);                                                        \
    }                                                                                                                         \
    DPT_EXPORT size_t dpt_wavefront_bytes##S(size_t n) { return wavefront_bytes<PathTracer<T>>(n); }                          \
    DPT_EXPORT int dpt_record##S(bvh##S* h, int per_thread, unsigned flags, size_t n, const void* rays, const uint64_t* offsets, \
                                 const uint32_t* counts, const uint32_t* seg_ray, const uint8_t* seg_kind, size_t segments,     \
                                 uint32_t* ids, T* t, T* u, T* v, uint32_t* calls, uint64_t* hashes, uint32_t* starts,         \
                                 uint32_t* finishes, uint32_t* done, unsigned long long* bad_rays, size_t depth,                 \
                                 void* workspace, size_t workspace_bytes, void* stream) {                                      \
        return record<T>(h, per_thread, flags, n, rays, Script { offsets, counts, seg_ray, seg_kind }, segments,                \
                         Outputs<T> { ids, t, u, v, calls, hashes }, starts, finishes, done, bad_rays, depth, workspace,       \
                         workspace_bytes, stream);                                                                            \
    }

DPT_ENTRY(float, 3f)
DPT_ENTRY(double, 3d)

DPT_EXPORT int dpt_plain3f(bvh3f* h, const void* rays, size_t n, void* hits, void* workspace, size_t workspace_bytes, void* stream) {
    DeviceView<float> view;
    if (!get_view<float>(h, view)) return -1;
    return guarded([&] {
        view.trace_paths<false>(n, PlainPaths { static_cast<const bvh_ray3f*>(rays), static_cast<bvh_hit3f*>(hits) }, workspace,
                                workspace_bytes, stream ? stream : view.stream);
        return 0;
    });
}

DPT_EXPORT const char* dpt_last_error() { return g_error.c_str(); }
