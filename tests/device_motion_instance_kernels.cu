// tests/device_motion_instance_kernels.cu — test shaders for the motion forms of DeviceView::trace_instances and
// trace_instance_paths, prepare_motion_instances and instance_at (include/bvh/v2/cuda/intersect.cuh).
//
// Compiled for sm_90a with the library's NVCC_FLAGS (--fmad=false among them) into
// tests/_build/libdevice_motion_instance_kernels.so (bvh_b200/build_ext.py build_device_motion_instance_tests) and driven
// by tests/test_device_motion_instance_gpu.py and scripts/motion_instance_trace_bench.py.  The recording shader and the
// path tracer are those of tests/device_instance_trace_kernels.cu and tests/device_instance_path_trace_kernels.cu, with a
// time per ray or path, so that their outputs compare bit for bit with the static calls there.  Every array is
// device-resident unless said otherwise.
//   dmi_records{3f,3d}     motion records from mesh handles (host array), the mesh of each record and two count x 12 key
//                          arrays (host), through make_motion_instance, copied to `records`; the largest bottom depth
//                          through *max_depth.
//   dmi_set_keys{3f,3d}    both keys of every record from device arrays of count x 12 values (a kernel on `stream`).
//   dmi_prepare{3f,3d}     prepare_motion_instances on `stream`.
//   dmi_static_at{3f,3d}   static records (Instance<T>, device) whose object_to_world is instance_at(records[k], tau)'s.
//   dmi_placement{3f,3d}   instance_at(records[k], times[k]) for k < count, object_to_world then world_to_object (24
//                          values per k), for the tests' float64 checks.
//   dmi_run{3f,3d}         one batch of rays, ray i at times[i], through the motion trace_instances (per_thread = 0) or one
//                          thread per ray that calls instance_at per entered record and nests DeviceView::intersect by hand
//                          (per_thread = 1).  Filters, flags and outputs as dit_run.
//   dmi_tracer{3f,3d}      the grey diffuse path tracer of dipt_tracer, path i at times[i], through one motion
//                          trace_instance_paths call (mode 0) or a wavefront loop of motion trace_instances launches
//                          (mode 1, dmi_wavefront_bytes(n) bytes of scratch).  finish adds 1 to counts[i] when counts is
//                          not null.
//   dmi_plain3f            float, closest-hit, accept all: 16-byte records and the instance per ray through the motion
//                          trace_instances (the benchmark's shader).
// Each returns 0; -1 with a message in dmi_last_error(); -2 when the call threw std::length_error, -3 when it threw
// std::invalid_argument, with its message.
#include <cuda_runtime.h>

#include <bvh/v2/cuda/intersect.cuh>

#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

namespace {

namespace cu = bvh::v2::cuda;
using cu::DeviceView;
using cu::Instance;
using cu::MotionInstance;
using cu::MotionInstances;
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

template <int kFilter> __device__ inline bool keep(uint32_t inst) { return kFilter == 0 || (inst & 1) == 0; }

template <typename T> struct Outputs {
    uint32_t* ids; T* t; T* u; T* v; uint32_t* inst; uint32_t* calls; uint64_t* hashes; uint32_t* counts;
};
template <typename T> __device__ inline void write(const Outputs<T>& out, size_t i, uint32_t id, T t, T u, T v, uint32_t inst,
                                                   uint32_t calls, uint64_t hash) {
    if (out.ids) out.ids[i] = id;
    if (out.t) out.t[i] = t;
    if (out.u) { out.u[i] = u; out.v[i] = v; }
    if (out.inst) out.inst[i] = inst;
    if (out.calls) out.calls[i] = calls;
    if (out.hashes) out.hashes[i] = hash;
    if (out.counts) atomicAdd(out.counts + i, 1u);
}

// dit_run's recording shader, ray i at times[i]
template <typename T, int kFilter> struct TestShader {
    using Ray = typename DeviceView<T>::Ray;
    struct Payload { uint32_t calls; uint64_t hash; };
    const Ray* rays;
    const T* times;
    Outputs<T> out;
    __device__ Ray start(size_t i, Payload& p, T& time) const { p.calls = 0; p.hash = kHashSeed; time = times[i]; return rays[i]; }
    __device__ bool accept(Payload& p, uint32_t inst, size_t id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(mix(p.hash, inst), id), bits(t)), bits(u)), bits(v));
        return keep<kFilter>(inst);
    }
    __device__ void finish(size_t i, const Payload& p, const typename DeviceView<T>::Hit& hit, uint32_t inst) const {
        write(out, i, (uint32_t)hit.prim_id, hit.t, hit.u, hit.v, inst, p.calls, p.hash);
    }
};

// One ray at `time` through the two levels by hand: the top view's intersect, whose leaf builds each record's placement
// with instance_at, transforms the ray (detail::object_ray) and runs the bottom view's intersect with intersect_tri, the
// tie rule on (instance, id) and the filter (visit).  Returns the instance of the hit (kNone: none); ray.tmax is its t.
template <typename T, bool kAny, bool kRobust, bool kLast, typename Visit>
__device__ uint32_t nested_ray(const DeviceView<T>& top, const MotionInstance<T>* records, T time, typename DeviceView<T>::Ray& ray,
                               uint32_t& best_id, T& bu, T& bv, Visit&& visit) {
    using View = DeviceView<T>;
    uint32_t best_inst = kNone;
    best_id = kNone; bu = T(0); bv = T(0);
    if (ray.tmin != ray.tmin || ray.tmax != ray.tmax) return kNone;      // a NaN interval: a miss, no accept call
    typename View::template SmallStack<kStack> stack;
    top.template intersect<kAny, kRobust>(ray, top.root_index(), stack, [&](size_t b, size_t e) {
        for (size_t k = b; k < e; ++k) {
            const uint32_t inst = top.prim_id(k);
            const Instance<T> rec = cu::instance_at(records[inst], time);
            if (cu::detail::instance_is_singular(rec.world_to_object)) continue;
            View bottom;
            bottom.nodes = rec.nodes; bottom.prim_ids = rec.prim_ids; bottom.tris = rec.tris; bottom.depth = rec.depth;
            bvhb200::RayCtx<T> w, o;
            cu::detail::load_ray<T>(ray, w);
            cu::detail::object_ray(rec.world_to_object, w, o);
            typename View::Ray oray = cu::detail::make_ray<typename View::Ray>(o);
            typename View::template SmallStack<kStack> bstack;
            bottom.template intersect<kAny, kRobust>(oray, rec.root_index, bstack, [&](size_t lb, size_t le) {
                for (size_t q = lb; q < le; ++q) {
                    T t, u, v;
                    if (!bottom.intersect_tri(q, oray, t, u, v)) continue;
                    const uint32_t id = (uint32_t)bottom.prim_id(q);
                    if (!kLast && best_inst != kNone && !(t < oray.tmax) &&
                        !(inst < best_inst || (inst == best_inst && id < best_id))) continue;      // canonical tie rule
                    if (!visit(inst, id, t, u, v)) continue;
                    oray.tmax = t; best_inst = inst; best_id = id; bu = u; bv = v;
                }
                return best_inst != kNone;
            });
            ray.tmax = oray.tmax;
            if (kAny && best_inst != kNone) return true;
        }
        return best_inst != kNone;
    });
    return best_inst;
}

template <typename T, bool kAny, bool kRobust, bool kLast, int kFilter>
__global__ void __launch_bounds__(kBlock) per_thread_kernel(DeviceView<T> top, const MotionInstance<T>* records,
                                                          TestShader<T, kFilter> shader, size_t n) {
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (i >= n) return;
    typename TestShader<T, kFilter>::Payload p;
    T time;
    typename DeviceView<T>::Ray ray = shader.start(i, p, time);
    const T tmax_in = ray.tmax;
    uint32_t id;
    T u, v;
    const uint32_t inst = nested_ray<T, kAny, kRobust, kLast>(top, records, time, ray, id, u, v, [&](uint32_t k, uint32_t pid, T t, T bu, T bv) {
        ++p.calls;
        p.hash = mix(mix(mix(mix(mix(p.hash, k), pid), bits(t)), bits(bu)), bits(bv));
        return keep<kFilter>(k);
    });
    write(shader.out, i, inst == kNone ? kNone : id, inst == kNone ? tmax_in : ray.tmax, u, v, inst, p.calls, p.hash);
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

// f.template operator()<kAny, kRobust, kLast>() for the flags' combination
template <typename F> int by_flags(unsigned flags, F&& f) {
    const bool any = flags & BVH_ANY_HIT, robust = flags & BVH_ROBUST, last = flags & BVH_TIE_LAST_VISITED;
    if (!last) {
        if (!any) return robust ? f.template operator()<false, true, false>() : f.template operator()<false, false, false>();
        return robust ? f.template operator()<true, true, false>() : f.template operator()<true, false, false>();
    }
    if (!any) return robust ? f.template operator()<false, true, true>() : f.template operator()<false, false, true>();
    return robust ? f.template operator()<true, true, true>() : f.template operator()<true, false, true>();
}

// f.template operator()<kRobust, kLast>() for the flags' combination (paths)
template <typename F> int by_path_flags(unsigned flags, F&& f) {
    const bool robust = flags & BVH_ROBUST, last = flags & BVH_TIE_LAST_VISITED;
    if (!last) return robust ? f.template operator()<true, false>() : f.template operator()<false, false>();
    return robust ? f.template operator()<true, true>() : f.template operator()<false, true>();
}

template <typename T, bool kAny, bool kRobust, bool kLast, int kFilter>
int run_filter(const DeviceView<T>& top, const MotionInstances<T>& inst, bool per_thread, size_t n, const void* rays, const T* times,
               const Outputs<T>& out, void* ws, size_t bytes, cudaStream_t stream) {
    const TestShader<T, kFilter> shader { static_cast<const typename DeviceView<T>::Ray*>(rays), times, out };
    if (!per_thread) {
        top.template trace_instances<kAny, kRobust, kLast>(n, inst, shader, ws, bytes, stream);
        return 0;
    }
    if (top.depth + 1 > kStack || inst.max_depth + 1 > kStack) { g_error = "per-thread kernel: tree too deep"; return -1; }
    if (n == 0) return 0;
    per_thread_kernel<T, kAny, kRobust, kLast, kFilter><<<(unsigned)((n + kBlock - 1) / kBlock), kBlock, 0, stream>>>(top, inst.records,
                                                                                                                    shader, n);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { g_error = std::string("per-thread kernel: ") + cudaGetErrorString(e); return -1; }
    return 0;
}

template <typename T>
int run(typename Api<T>::Handle* h, MotionInstance<T>* recs, size_t count, size_t max_depth, int per_thread, int filter, unsigned flags,
        const void* rays, const T* times, size_t n, Outputs<T> out, void* ws, size_t bytes, void* stream) {
    DeviceView<T> top;
    if (!get_view<T>(h, top)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : top.stream);
    const MotionInstances<T> inst { recs, count, max_depth };
    return guarded([&] {
        return by_flags(flags, [&]<bool kAny, bool kRobust, bool kLast>() {
            if (filter == 0) return run_filter<T, kAny, kRobust, kLast, 0>(top, inst, per_thread, n, rays, times, out, ws, bytes, s);
            return run_filter<T, kAny, kRobust, kLast, 1>(top, inst, per_thread, n, rays, times, out, ws, bytes, s);
        });
    });
}

template <typename T>
int make_records(typename Api<T>::Handle* const* meshes, const uint32_t* mesh_of, const T* keys0, const T* keys1, size_t count,
                 MotionInstance<T>* d_records, size_t* max_depth, void* stream) {
    std::vector<MotionInstance<T>> recs(count);
    size_t depth = 0;
    for (size_t k = 0; k < count; ++k) {
        DeviceView<T> view;
        if (!get_view<T>(meshes[mesh_of[k]], view)) return -1;
        recs[k] = cu::make_motion_instance(view, keys0 + 12 * k, keys1 + 12 * k);
        depth = view.depth > depth ? view.depth : depth;
    }
    *max_depth = depth;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemcpyAsync(d_records, recs.data(), count * sizeof(MotionInstance<T>), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { g_error = cudaGetErrorString(e); return -1; }
    return 0;
}

template <typename T> __global__ void set_keys_kernel(MotionInstance<T>* records, const T* keys0, const T* keys1, size_t count) {
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= 12 * count) return;
    records[i / 12].object_to_world[0][i % 12] = keys0[i];
    records[i / 12].object_to_world[1][i % 12] = keys1[i];
}

template <typename T> __global__ void static_at_kernel(const MotionInstance<T>* records, size_t count, T tau, Instance<T>* out) {
    const size_t k = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (k < count) out[k] = cu::instance_at(records[k], tau);
}

template <typename T> __global__ void placement_kernel(const MotionInstance<T>* records, const T* times, size_t count, T* out) {
    const size_t k = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= count) return;
    const Instance<T> a = cu::instance_at(records[k], times[k]);
    for (int j = 0; j < 12; ++j) { out[24 * k + j] = a.object_to_world[j]; out[24 * k + 12 + j] = a.world_to_object[j]; }
}

// ---------------------------------------------------------------------------------------------------------------------
// The path tracer
// ---------------------------------------------------------------------------------------------------------------------

// dipt_tracer's InstancePathTracer over motion records: the same arithmetic, with the path's time in its payload and the
// normal's vertices through instance_at(records[inst], time).object_to_world (with equal keys, the key's own bits).
template <typename T> struct MotionPathTracer {
    using View = DeviceView<T>;
    using Ray = typename View::Ray;
    using Hit = typename View::Hit;
    struct Payload { T throughput, radiance, pending, time; uint32_t prim, inst, bounce, segments, hash; };
    static constexpr T kAlbedo = T(0.7), kSky = T(0.25), kLight = T(2.0);

    const Ray* primary;
    const T* times;
    T light[3];
    const T* const* verts;              // per instance: its mesh's vertices, 9 per triangle, original order
    const MotionInstance<T>* records;
    uint32_t max_bounces;
    T* radiance; uint32_t* segments; uint32_t* hashes; uint32_t* counts;

    __device__ void normal(uint32_t inst, uint32_t prim, bool flip, T time, T n[3]) const {
        const T* v = verts[inst] + 9 * (size_t)prim;
        const Instance<T> at = cu::instance_at(records[inst], time);
        T w[9];
        for (int k = 0; k < 3; ++k)
            for (int a = 0; a < 3; ++a) w[3 * k + a] = cu::detail::affine_row(at.object_to_world + 4 * a, v + 3 * k, true);
        const T e1[3] = { w[3] - w[0], w[4] - w[1], w[5] - w[2] }, e2[3] = { w[6] - w[0], w[7] - w[1], w[8] - w[2] };
        const T c[3] = { e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0] };
        const T len = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
        const T s = flip ? T(-1) / len : T(1) / len;
        for (int a = 0; a < 3; ++a) n[a] = c[a] * s;
    }

    __device__ PathStep start(size_t i, Payload& p, Ray& ray, T& time) const {
        ray = primary[i];
        p.throughput = T(1); p.radiance = T(0); p.pending = T(0); p.time = times[i];
        p.prim = kNone; p.inst = kNone; p.bounce = 0; p.segments = 0; p.hash = 2166136261u;
        time = p.time;
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
        normal(p.inst, p.prim, p.bounce & 1u, p.time, n);
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
        normal(p.inst, p.prim, false, p.time, n);
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
        if (counts) atomicAdd(counts + i, 1u);
    }
};

// The wavefront form: the path state in arrays, one motion trace_instances pass per segment kind, the path's time
// carried in its payload.
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
    typename Shader::View::Scalar time;
    const PathStep step = shader.start(i, p, ray, time);
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

    __device__ Ray start(size_t i, Payload& q, T& time) const {
        q.live = st.steps[i] == (uint8_t)kind;
        time = T(0);
        if (q.live) { q.p = st.payloads[i]; time = q.p.time; return st.rays[i]; }
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

template <typename T>
int tracer(typename Api<T>::Handle* h, void* records, size_t count, size_t max_depth, int mode, unsigned flags, size_t n,
           const void* primary, const T* times, const T* light, const T* const* verts, uint32_t max_bounces, T* radiance,
           uint32_t* segments, uint32_t* hashes, uint32_t* counts, void* scratch, void* ws, size_t bytes, void* stream) {
    DeviceView<T> top;
    if (!get_view<T>(h, top)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : top.stream);
    const MotionInstances<T> inst { static_cast<MotionInstance<T>*>(records), count, max_depth };
    MotionPathTracer<T> shader;
    shader.primary = static_cast<const typename DeviceView<T>::Ray*>(primary);
    shader.times = times;
    for (int a = 0; a < 3; ++a) shader.light[a] = light[a];
    shader.verts = verts; shader.records = inst.records; shader.max_bounces = max_bounces;
    shader.radiance = radiance; shader.segments = segments; shader.hashes = hashes; shader.counts = counts;
    return guarded([&] {
        return by_path_flags(flags, [&]<bool kRobust, bool kLast>() {
            if (mode == 0) {
                top.template trace_instance_paths<kRobust, kLast>(n, inst, shader, ws, bytes, s);
                return 0;
            }
            if (n == 0) return 0;
            using S = MotionPathTracer<T>;
            const WavefrontState<S> st = wavefront_state<S>(scratch, n);
            wavefront_start_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(shader, st, n);
            const cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) throw std::runtime_error(std::string("wavefront start: ") + cudaGetErrorString(e));
            for (uint32_t k = 0; k < max_bounces + 1; ++k) {
                top.template trace_instances<false, kRobust, kLast>(n, inst, WavefrontPass<S> { shader, st, PathStep::Closest }, ws, bytes, s);
                top.template trace_instances<true, kRobust, kLast>(n, inst, WavefrontPass<S> { shader, st, PathStep::Occlusion }, ws, bytes, s);
            }
            return 0;
        });
    });
}

// The benchmark's shader: rays and times in, 16-byte records and the instance out
struct PlainShader {
    struct Payload {};
    const bvh_ray3f* rays;
    const float* times;
    bvh_hit3f* hits;
    uint32_t* inst;
    __device__ bvh_ray3f start(size_t i, Payload&, float& time) const { time = times[i]; return rays[i]; }
    __device__ bool accept(Payload&, uint32_t, size_t, float, float, float) const { return true; }
    __device__ void finish(size_t i, const Payload&, const bvh_hit3f& hit, uint32_t k) const { hits[i] = hit; inst[i] = k; }
};

} // namespace

#define DMI_EXPORT extern "C" __attribute__((visibility("default")))
#define DMI_LAUNCH(kernel, count, ...)                                                                                    \
    do {                                                                                                                 \
        if ((count) == 0) return 0;                                                                                      \
        kernel<<<(unsigned)(((count) + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(__VA_ARGS__);           \
        const cudaError_t e = cudaGetLastError();                                                                        \
        if (e != cudaSuccess) { g_error = cudaGetErrorString(e); return -1; }                                            \
        return 0;                                                                                                        \
    } while (0)
#define DMI_ENTRY(T, S)                                                                                                   \
    DMI_EXPORT int dmi_records##S(bvh##S* const* meshes, const uint32_t* mesh_of, const T* keys0, const T* keys1,         \
                                  size_t count, void* records, size_t* max_depth, void* stream) {                        \
        return make_records<T>(meshes, mesh_of, keys0, keys1, count, static_cast<MotionInstance<T>*>(records), max_depth, \
                               stream);                                                                                  \
    }                                                                                                                    \
    DMI_EXPORT int dmi_set_keys##S(void* records, const T* keys0, const T* keys1, size_t count, void* stream) {          \
        DMI_LAUNCH(set_keys_kernel<T>, 12 * count, static_cast<MotionInstance<T>*>(records), keys0, keys1, count);         \
    }                                                                                                                    \
    DMI_EXPORT int dmi_static_at##S(const void* records, size_t count, T tau, void* out, void* stream) {                 \
        DMI_LAUNCH(static_at_kernel<T>, count, static_cast<const MotionInstance<T>*>(records), count, tau,                \
                   static_cast<Instance<T>*>(out));                                                                       \
    }                                                                                                                    \
    DMI_EXPORT int dmi_placement##S(const void* records, const T* times, size_t count, T* out, void* stream) {           \
        DMI_LAUNCH(placement_kernel<T>, count, static_cast<const MotionInstance<T>*>(records), times, count, out);        \
    }                                                                                                                    \
    DMI_EXPORT int dmi_prepare##S(void* records, size_t count, size_t max_depth, void* bboxes, void* centers, void* stream) { \
        const MotionInstances<T> inst { static_cast<MotionInstance<T>*>(records), count, max_depth };                     \
        return guarded([&] {                                                                                             \
            cu::prepare_motion_instances(inst, static_cast<bvh_bbox##S*>(bboxes), static_cast<bvh_vec##S*>(centers), stream); \
            return 0;                                                                                                    \
        });                                                                                                              \
    }                                                                                                                    \
    DMI_EXPORT int dmi_run##S(bvh##S* top, void* records, size_t count, size_t max_depth, int per_thread, int filter,     \
                              unsigned flags, const void* rays, const T* times, size_t n, uint32_t* ids, T* t, T* u, T* v, \
                              uint32_t* inst, uint32_t* calls, uint64_t* hashes, uint32_t* counts, void* ws, size_t bytes, \
                              void* stream) {                                                                            \
        return run<T>(top, static_cast<MotionInstance<T>*>(records), count, max_depth, per_thread, filter, flags, rays,    \
                      times, n, Outputs<T> { ids, t, u, v, inst, calls, hashes, counts }, ws, bytes, stream);             \
    }                                                                                                                    \
    DMI_EXPORT int dmi_tracer##S(bvh##S* top, void* records, size_t count, size_t max_depth, int mode, unsigned flags,   \
                                 size_t n, const void* primary, const T* times, const T* light, const void* verts,        \
                                 uint32_t max_bounces, T* radiance, uint32_t* segments, uint32_t* hashes, uint32_t* counts, \
                                 void* scratch, void* ws, size_t bytes, void* stream) {                                   \
        return tracer<T>(top, records, count, max_depth, mode, flags, n, primary, times, light,                           \
                         static_cast<const T* const*>(verts), max_bounces, radiance, segments, hashes, counts, scratch, ws, \
                         bytes, stream);                                                                                 \
    }                                                                                                                    \
    DMI_EXPORT size_t dmi_wavefront_bytes##S(size_t n) { return wavefront_bytes<MotionPathTracer<T>>(n); }               \
    DMI_EXPORT size_t dmi_record_bytes##S() { return sizeof(MotionInstance<T>); }

DMI_ENTRY(float, 3f)
DMI_ENTRY(double, 3d)

DMI_EXPORT int dmi_plain3f(bvh3f* top, void* records, size_t count, size_t max_depth, const void* rays, const float* times, size_t n,
                           void* hits, uint32_t* inst, void* ws, size_t bytes, void* stream) {
    DeviceView<float> view;
    if (!get_view<float>(top, view)) return -1;
    const MotionInstances<float> instances { static_cast<MotionInstance<float>*>(records), count, max_depth };
    return guarded([&] {
        view.trace_instances<false, false>(n, instances, PlainShader { static_cast<const bvh_ray3f*>(rays), times,
                                                                       static_cast<bvh_hit3f*>(hits), inst },
                                           ws, bytes, stream ? stream : view.stream);
        return 0;
    });
}

DMI_EXPORT const char* dmi_last_error() { return g_error.c_str(); }
