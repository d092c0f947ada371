// tests/device_instance_path_trace_kernels.cu — test shaders for DeviceView::trace_instance_paths
// (include/bvh/v2/cuda/intersect.cuh).
//
// Compiled for sm_90a with the library's NVCC_FLAGS (--fmad=false among them) into
// tests/_build/libdevice_instance_path_trace_kernels.so (bvh_b200/build_ext.py build_device_instance_path_trace_tests) and
// driven by tests/test_device_instance_path_trace_gpu.py and scripts/instance_path_trace_bench.py.  Instance records are
// made and prepared by tests/device_instance_trace_kernels.cu (dit_records, dit_prepare); every array is device-resident.
//   dipt_tracer{3f,3d}    a grey diffuse path tracer with a point light and next-event estimation (InstancePathTracer
//                         below) over a top tree `top` and its records, path i starting with primary ray i, run as
//                           mode 0: one DeviceView::trace_instance_paths call;
//                           mode 1: a wavefront loop of trace_instances launches with the path state in arrays: a start
//                                   kernel, then per bounce one closest-hit and one occlusion pass over all n paths, a path
//                                   that is not waiting for that kind of segment drawn as a NaN ray;
//                           mode 2: DeviceView::trace_paths with `top` as a mesh handle (instance 0, no records).
//                         verts[k] is the vertex array (9 per triangle, original order) of instance k's mesh.  Per path it
//                         writes the radiance, the segment count and a 32-bit hash of the segment records and instances.
//                         Mode 1 needs dipt_wavefront_bytes{3f,3d}(n) bytes of scratch.
//   dipt_record{3f,3d}    a recording shader whose paths follow scripted segments: path i runs counts[i] segments, segment
//                         k = offsets[i] + j traces rays[seg_ray[k]] as seg_kind[k] (1 Closest, 2 Occlusion), through
//                         trace_instance_paths (per_thread = 0) or one thread per segment that nests DeviceView::intersect
//                         by hand (per_thread = 1).  Filters: 0 accept all, 1 reject odd instances.  Per segment k, for every
//                         output that is not null: the record's id, t, u, v, its instance, the accept-call count and a
//                         64-bit hash of the accept sequence (instance, original id, bits of t, u, v).  Per path
//                         (trace_instance_paths only): starts[i] and finishes[i] count the calls, done[i] is the segment
//                         count finish saw; bad_rays[0] counts next calls whose ray was not the scripted one.
// Each returns 0; -1 with a message in dipt_last_error(); -2 when the call threw std::length_error, -3 when it threw
// std::invalid_argument, with its message.
#include <cuda_runtime.h>

#include <bvh/v2/cuda/intersect.cuh>

#include <cstdint>
#include <stdexcept>
#include <string>

namespace {

namespace cu = bvh::v2::cuda;
using cu::DeviceView;
using cu::Instance;
using cu::Instances;
using cu::PathStep;

thread_local std::string g_error;
constexpr unsigned kBlock = 128;
constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr unsigned kStack = 96;         // per-thread stack of the hand-nested traversals

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
__device__ inline uint32_t hash32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}

template <typename R> __device__ inline bool same_ray(const R& a, const R& b) {
    return bits(a.org.x) == bits(b.org.x) && bits(a.org.y) == bits(b.org.y) && bits(a.org.z) == bits(b.org.z) &&
           bits(a.dir.x) == bits(b.dir.x) && bits(a.dir.y) == bits(b.dir.y) && bits(a.dir.z) == bits(b.dir.z) &&
           bits(a.tmin) == bits(b.tmin) && bits(a.tmax) == bits(b.tmax);
}

// ---------------------------------------------------------------------------------------------------------------------
// The path tracer
// ---------------------------------------------------------------------------------------------------------------------

// tests/device_path_trace_kernels.cu's PathTracer over placed meshes.  Grey diffuse surfaces lit by a point light and a
// constant sky; at every closest hit a shadow segment to the light follows when the light is above the surface, then
// the path bounces in a direction drawn from a hash of (path, segment).  Every segment skips the (instance, triangle)
// the path stands on.  The normal is that of the world-space triangle: its vertices through the instance's
// object_to_world with detail::affine_row, so that under the identity they are the mesh's own bits.  Without records
// (trace_paths on one mesh) the mesh's vertices are used as they are.
template <typename T> struct InstancePathTracer {
    using View = DeviceView<T>;
    using Ray = typename View::Ray;
    using Hit = typename View::Hit;
    struct Payload { T throughput, radiance, pending; uint32_t prim, inst, bounce, segments, hash; };
    static constexpr T kAlbedo = T(0.7), kSky = T(0.25), kLight = T(2.0);

    const Ray* primary;
    T light[3];
    const T* const* verts;              // per instance: its mesh's vertices, 9 per triangle, original order
    const Instance<T>* records;         // nullptr: one mesh, unplaced
    uint32_t max_bounces;
    T* radiance; uint32_t* segments; uint32_t* hashes;

    __device__ void normal(uint32_t inst, uint32_t prim, bool flip, T n[3]) const {
        const T* v = verts[inst] + 9 * (size_t)prim;
        T w[9];
        for (int k = 0; k < 3; ++k)
            for (int a = 0; a < 3; ++a)
                w[3 * k + a] = records ? cu::detail::affine_row(records[inst].object_to_world + 4 * a, v + 3 * k, true) : v[3 * k + a];
        const T e1[3] = { w[3] - w[0], w[4] - w[1], w[5] - w[2] }, e2[3] = { w[6] - w[0], w[7] - w[1], w[8] - w[2] };
        const T c[3] = { e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0] };
        const T len = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
        const T s = flip ? T(-1) / len : T(1) / len;
        for (int a = 0; a < 3; ++a) n[a] = c[a] * s;
    }

    __device__ PathStep start(size_t i, Payload& p, Ray& ray) const {
        ray = primary[i];
        p.throughput = T(1); p.radiance = T(0); p.pending = T(0);
        p.prim = kNone; p.inst = kNone; p.bounce = 0; p.segments = 0; p.hash = 2166136261u;
        return PathStep::Closest;
    }
    __device__ bool accept(Payload& p, uint32_t inst, size_t prim_id, T, T, T) const {
        return !(inst == p.inst && prim_id == p.prim);
    }

    __device__ PathStep bounce(size_t i, Payload& p, Ray& ray) const {
        if ((p.bounce >> 1) >= max_bounces) return PathStep::End;
        const uint32_t h = hash32((uint32_t)i * 0x9E3779B9u ^ hash32(p.segments));
        const T u1 = T(h >> 16) * T(1.0 / 65536), u2 = T(h & 0xFFFFu) * T(1.0 / 65536);
        const T z = T(1) - T(2) * u1, rr = sqrt(fmax(T(0), T(1) - z * z)), phi = T(6.283185307179586) * u2;
        T d[3] = { rr * cos(phi), rr * sin(phi), z }, n[3];
        normal(p.inst, p.prim, p.bounce & 1u, n);
        T c = d[0] * n[0] + d[1] * n[1] + d[2] * n[2];
        if (c < T(0)) { for (int a = 0; a < 3; ++a) d[a] = -d[a]; c = -c; }
        p.throughput = p.throughput * (T(2) * kAlbedo * c);
        p.bounce += 2;
        ray.dir.x = d[0]; ray.dir.y = d[1]; ray.dir.z = d[2];
        ray.tmin = T(0); ray.tmax = T(INFINITY);
        return PathStep::Closest;
    }

    __device__ PathStep next(size_t i, Payload& p, const Hit& hit, uint32_t inst, Ray& ray) const {
        ++p.segments;
        p.hash = mix32(mix32(mix32(mix32(mix32(p.hash, (uint32_t)hit.prim_id), inst), fold(bits(hit.t))), fold(bits(hit.u))),
                       fold(bits(hit.v)));
        const bool miss = hit.prim_id == (decltype(hit.prim_id))~(decltype(hit.prim_id))0;
        if (p.pending != T(0)) {                             // a shadow segment ended: ray.org is the surface point
            if (miss) p.radiance = p.radiance + p.pending;
            p.pending = T(0);
            return bounce(i, p, ray);
        }
        if (miss) { p.radiance = p.radiance + p.throughput * kSky; return PathStep::End; }
        p.prim = (uint32_t)hit.prim_id;
        p.inst = inst;
        const T x[3] = { ray.org.x + hit.t * ray.dir.x, ray.org.y + hit.t * ray.dir.y, ray.org.z + hit.t * ray.dir.z };
        T n[3];
        normal(p.inst, p.prim, false, n);
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

// The same shader through trace_paths on one mesh: instance 0 for every triangle, kNoInstance for a miss
template <typename T> struct MeshPaths {
    using S = InstancePathTracer<T>;
    using Payload = typename S::Payload;
    S s;
    __device__ PathStep start(size_t i, Payload& p, typename S::Ray& ray) const { return s.start(i, p, ray); }
    __device__ bool accept(Payload& p, size_t id, T t, T u, T v) const { return s.accept(p, 0, id, t, u, v); }
    __device__ PathStep next(size_t i, Payload& p, const typename S::Hit& hit, typename S::Ray& ray) const {
        return s.next(i, p, hit, hit.prim_id == (decltype(hit.prim_id))~(decltype(hit.prim_id))0 ? kNone : 0u, ray);
    }
    __device__ void finish(size_t i, const Payload& p) const { s.finish(i, p); }
};

// The wavefront form: the path state in arrays, one trace_instances pass per segment kind.
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
    __device__ bool accept(Payload& q, uint32_t inst, size_t prim_id, T t, T u, T v) const { return shader.accept(q.p, inst, prim_id, t, u, v); }
    __device__ void finish(size_t i, const Payload& q, const typename Shader::Hit& hit, uint32_t inst) const {
        if (!q.live) return;
        typename Shader::Payload p = q.p;
        Ray ray = st.rays[i];
        const PathStep step = shader.next(i, p, hit, inst, ray);
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

// `passes` rounds of one closest-hit and one occlusion trace_instances pass, all on `stream`, no host synchronisation
template <typename T, bool kRobust, bool kLast, typename Shader>
void run_wavefront(const DeviceView<T>& top, const Instances<T>& inst, const Shader& shader, size_t n, uint32_t passes, void* scratch,
                   void* ws, size_t bytes, cudaStream_t s) {
    if (n == 0) return;
    const WavefrontState<Shader> st = wavefront_state<Shader>(scratch, n);
    wavefront_start_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(shader, st, n);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("wavefront start: ") + cudaGetErrorString(e));
    for (uint32_t k = 0; k < passes; ++k) {
        top.template trace_instances<false, kRobust, kLast>(n, inst, WavefrontPass<Shader> { shader, st, PathStep::Closest }, ws, bytes, s);
        top.template trace_instances<true, kRobust, kLast>(n, inst, WavefrontPass<Shader> { shader, st, PathStep::Occlusion }, ws, bytes, s);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// The recording shader
// ---------------------------------------------------------------------------------------------------------------------

__device__ inline bool keep(int filter, uint32_t inst) { return filter == 0 || (inst & 1) == 0; }

template <typename T> struct Outputs {
    uint32_t* ids; T* t; T* u; T* v; uint32_t* inst; uint32_t* calls; uint64_t* hashes;
};
template <typename T> __device__ inline void write(const Outputs<T>& out, size_t k, uint32_t id, T t, T u, T v, uint32_t inst,
                                                   uint32_t calls, uint64_t hash) {
    if (out.ids) out.ids[k] = id;
    if (out.t) out.t[k] = t;
    if (out.u) { out.u[k] = u; out.v[k] = v; }
    if (out.inst) out.inst[k] = inst;
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
    using Ray = typename DeviceView<T>::Ray;
    using Hit = typename DeviceView<T>::Hit;
    struct Payload { uint32_t seg, calls; uint64_t hash; };
    const Ray* rays;
    Script script;
    int filter;
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
    __device__ bool accept(Payload& p, uint32_t inst, size_t prim_id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(mix(p.hash, inst), prim_id), bits(t)), bits(u)), bits(v));
        return keep(filter, inst);
    }
    __device__ PathStep next(size_t i, Payload& p, const Hit& hit, uint32_t inst, Ray& ray) const {
        const size_t k = script.offsets[i] + p.seg;
        if (bad_rays && !same_ray(ray, rays[script.seg_ray[k]])) atomicAdd(bad_rays, 1ull);
        write(out, k, (uint32_t)hit.prim_id, hit.t, hit.u, hit.v, inst, p.calls, p.hash);
        ++p.seg; p.calls = 0; p.hash = kHashSeed;
        return p.seg < script.counts[i] ? segment(k + 1, ray) : PathStep::End;
    }
    __device__ void finish(size_t i, const Payload& p) const {
        if (finishes) atomicAdd(finishes + i, 1u);
        if (done) done[i] = p.seg;
    }
};

// One segment through the two levels by hand: the top view's intersect, whose leaf transforms the ray
// (detail::object_ray) and runs the bottom view's intersect with intersect_tri, the tie rule on (instance, id) and the
// filter, as a user kernel without trace_instance_paths writes it.
template <typename T, bool kAny, bool kRobust, bool kLast>
__device__ void per_thread_segment(const DeviceView<T>& top, const Instance<T>* records, const RecordShader<T>& shader, size_t k) {
    using View = DeviceView<T>;
    typename View::Ray ray = shader.rays[shader.script.seg_ray[k]];
    const T tmax_in = ray.tmax;
    uint32_t best_inst = kNone, best_id = kNone, calls = 0;
    T bu = T(0), bv = T(0);
    uint64_t hash = kHashSeed;
    if (ray.tmin == ray.tmin && ray.tmax == ray.tmax) {                    // a NaN interval: a miss, no accept call
        typename View::template SmallStack<kStack> stack;
        top.template intersect<kAny, kRobust>(ray, top.root_index(), stack, [&](size_t b, size_t e) {
            for (size_t q = b; q < e; ++q) {
                const uint32_t inst = top.prim_id(q);
                const Instance<T>& rec = records[inst];
                if (cu::detail::instance_is_singular(rec.world_to_object)) continue;
                View bottom;
                bottom.nodes = rec.nodes; bottom.prim_ids = rec.prim_ids; bottom.tris = rec.tris; bottom.depth = rec.depth;
                bvhb200::RayCtx<T> w, o;
                cu::detail::load_ray<T>(ray, w);
                cu::detail::object_ray(rec.world_to_object, w, o);
                typename View::Ray oray = cu::detail::make_ray<typename View::Ray>(o);
                typename View::template SmallStack<kStack> bstack;
                bottom.template intersect<kAny, kRobust>(oray, rec.root_index, bstack, [&](size_t lb, size_t le) {
                    for (size_t x = lb; x < le; ++x) {
                        T t, u, v;
                        if (!bottom.intersect_tri(x, oray, t, u, v)) continue;
                        const uint32_t id = (uint32_t)bottom.prim_id(x);
                        if (!kLast && best_inst != kNone && !(t < oray.tmax) &&
                            !(inst < best_inst || (inst == best_inst && id < best_id))) continue;      // canonical tie rule
                        ++calls;
                        hash = mix(mix(mix(mix(mix(hash, inst), id), bits(t)), bits(u)), bits(v));
                        if (!keep(shader.filter, inst)) continue;
                        oray.tmax = t; best_inst = inst; best_id = id; bu = u; bv = v;
                    }
                    return best_inst != kNone;
                });
                ray.tmax = oray.tmax;
                if (kAny && best_inst != kNone) return true;
            }
            return best_inst != kNone;
        });
    }
    const bool hit = best_inst != kNone;
    write(shader.out, k, hit ? best_id : kNone, hit ? ray.tmax : tmax_in, bu, bv, best_inst, calls, hash);
}

template <typename T, bool kRobust, bool kLast>
__global__ void __launch_bounds__(kBlock) per_thread_kernel(DeviceView<T> top, const Instance<T>* records, RecordShader<T> shader,
                                                          size_t segments) {
    const size_t k = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (k >= segments) return;
    if (shader.script.seg_kind[k] == (uint8_t)PathStep::Occlusion) per_thread_segment<T, true, kRobust, kLast>(top, records, shader, k);
    else per_thread_segment<T, false, kRobust, kLast>(top, records, shader, k);
}

// ---------------------------------------------------------------------------------------------------------------------
// Entry points
// ---------------------------------------------------------------------------------------------------------------------

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
int tracer(typename Api<T>::Handle* h, void* records, size_t count, size_t max_depth, int mode, unsigned flags, size_t n,
           const void* primary, const T* light, const T* const* verts, uint32_t max_bounces, T* radiance, uint32_t* segments,
           uint32_t* hashes, void* scratch, void* ws, size_t bytes, void* stream) {
    DeviceView<T> top;
    if (!get_view<T>(h, top)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : top.stream);
    const Instances<T> inst { static_cast<Instance<T>*>(records), count, max_depth };
    InstancePathTracer<T> shader;
    shader.primary = static_cast<const typename DeviceView<T>::Ray*>(primary);
    for (int a = 0; a < 3; ++a) shader.light[a] = light[a];
    shader.verts = verts; shader.records = mode == 2 ? nullptr : inst.records; shader.max_bounces = max_bounces;
    shader.radiance = radiance; shader.segments = segments; shader.hashes = hashes;
    return guarded([&] {
        return dispatch(flags, [&]<bool kRobust, bool kLast>() {
            if (mode == 0) top.template trace_instance_paths<kRobust, kLast>(n, inst, shader, ws, bytes, s);
            else if (mode == 1) run_wavefront<T, kRobust, kLast>(top, inst, shader, n, max_bounces + 1, scratch, ws, bytes, s);
            else top.template trace_paths<kRobust, kLast>(n, MeshPaths<T> { shader }, ws, bytes, s);
            return 0;
        });
    });
}

template <typename T>
int record(typename Api<T>::Handle* h, void* records, size_t count, size_t max_depth, int per_thread, int filter, unsigned flags,
           size_t n, const void* rays, Script script, size_t segments, Outputs<T> out, uint32_t* starts, uint32_t* finishes,
           uint32_t* done, unsigned long long* bad_rays, void* ws, size_t bytes, void* stream) {
    DeviceView<T> top;
    if (!get_view<T>(h, top)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : top.stream);
    const Instances<T> inst { static_cast<Instance<T>*>(records), count, max_depth };
    const RecordShader<T> shader { static_cast<const typename DeviceView<T>::Ray*>(rays), script, filter, out, starts, finishes, done,
                                   bad_rays };
    return guarded([&] {
        return dispatch(flags, [&]<bool kRobust, bool kLast>() {
            if (!per_thread) {
                top.template trace_instance_paths<kRobust, kLast>(n, inst, shader, ws, bytes, s);
                return 0;
            }
            if (top.depth + 1 > kStack || max_depth + 1 > kStack) { g_error = "per-thread kernel: tree too deep"; return -1; }
            if (segments == 0) return 0;
            per_thread_kernel<T, kRobust, kLast><<<(unsigned)((segments + kBlock - 1) / kBlock), kBlock, 0, s>>>(top, inst.records, shader,
                                                                                                                 segments);
            const cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) { g_error = std::string("per-thread kernel: ") + cudaGetErrorString(e); return -1; }
            return 0;
        });
    });
}

} // namespace

#define DIPT_EXPORT extern "C" __attribute__((visibility("default")))
#define DIPT_ENTRY(T, S)                                                                                                      \
    DIPT_EXPORT int dipt_tracer##S(bvh##S* top, void* records, size_t count, size_t max_depth, int mode, unsigned flags,      \
                                   size_t n, const void* primary, const T* light, const void* verts, uint32_t max_bounces,    \
                                   T* radiance, uint32_t* segments, uint32_t* hashes, void* scratch, void* workspace,         \
                                   size_t workspace_bytes, void* stream) {                                                    \
        return tracer<T>(top, records, count, max_depth, mode, flags, n, primary, light, static_cast<const T* const*>(verts), \
                         max_bounces, radiance, segments, hashes, scratch, workspace, workspace_bytes, stream);              \
    }                                                                                                                         \
    DIPT_EXPORT size_t dipt_wavefront_bytes##S(size_t n) { return wavefront_bytes<InstancePathTracer<T>>(n); }               \
    DIPT_EXPORT int dipt_record##S(bvh##S* top, void* records, size_t count, size_t max_depth, int per_thread, int filter,     \
                                   unsigned flags, size_t n, const void* rays, const uint64_t* offsets, const uint32_t* counts, \
                                   const uint32_t* seg_ray, const uint8_t* seg_kind, size_t segments, uint32_t* ids, T* t,     \
                                   T* u, T* v, uint32_t* inst, uint32_t* calls, uint64_t* hashes, uint32_t* starts,            \
                                   uint32_t* finishes, uint32_t* done, unsigned long long* bad_rays, void* workspace,          \
                                   size_t workspace_bytes, void* stream) {                                                    \
        return record<T>(top, records, count, max_depth, per_thread, filter, flags, n, rays,                                  \
                         Script { offsets, counts, seg_ray, seg_kind }, segments, Outputs<T> { ids, t, u, v, inst, calls, hashes }, \
                         starts, finishes, done, bad_rays, workspace, workspace_bytes, stream);                               \
    }

DIPT_ENTRY(float, 3f)
DIPT_ENTRY(double, 3d)

DIPT_EXPORT const char* dipt_last_error() { return g_error.c_str(); }
