// tests/device_instance_trace_kernels.cu — test shaders for DeviceView::trace_instances and prepare_instances
// (include/bvh/v2/cuda/intersect.cuh).
//
// Compiled for sm_90a with the library's NVCC_FLAGS (--fmad=false among them) into
// tests/_build/libdevice_instance_trace_kernels.so (bvh_b200/build_ext.py build_device_instance_trace_tests) and driven by
// tests/test_device_instance_trace_gpu.py and scripts/instance_trace_bench.py.  Every array is device-resident unless
// said otherwise.
//   dit_records{3f,3d}      instance records from mesh handles (host array), the mesh of each instance and 3 x 4
//                           matrices (host arrays), through make_instance, copied to `records`; returns the largest
//                           bottom depth through *max_depth.
//   dit_set_matrices{3f,3d} object_to_world of every record from a device array of count x 12 values (a kernel on
//                           `stream`, for animation on one stream).
//   dit_prepare{3f,3d}      prepare_instances on `stream`.
//   dit_run{3f,3d}          one batch of rays from an array through the top tree `top` over the records: through
//                           DeviceView::trace_instances (per_thread = 0) or through a kernel of one thread per ray that
//                           nests DeviceView::intersect by hand, the top view's leaf transforming the ray and running the
//                           bottom view's intersect with a leaf of intersect_tri calls, the same tie rule and filter
//                           (per_thread = 1).  Filters: 0 accept all, 1 reject odd instances.  Flags: BVH_ANY_HIT,
//                           BVH_ROBUST, BVH_TIE_LAST_VISITED.  Per ray i it writes, for every output that is not null: the
//                           record's id (all ones: none), t, u, v, its instance, the accept-call count, a 64-bit hash of
//                           the accept sequence (instance, original id and the bits of t, u, v), and adds 1 to counts[i].
//   dit_triangles{3f,3d}    the same recording shader, accept all, through DeviceView::trace_triangles on a mesh handle
//                           (instance 0 in the hash; instance 0 on a hit).
//   dit_plain3f             float, closest-hit, canonical ties, accept all, an empty payload: 16-byte records and the
//                           instance per ray through trace_instances (the benchmark's shader).
//   dit_plain_triangles3f   the same records through trace_triangles on one (flattened) mesh handle.
//   dit_nested_trace3f      the same records through DeviceView::trace with a hand-nested tracer: its leaf loops over the
//                           leaf's instances and runs each bottom tree's intersect with a per-thread stack.
// Each returns 0; -1 with a message in dit_last_error(); -2 when the call threw std::length_error, -3 when it threw
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
using cu::Instances;

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

// The recording shader of trace_instances
template <typename T, int kFilter> struct TestShader {
    using Ray = typename DeviceView<T>::Ray;
    struct Payload { uint32_t calls; uint64_t hash; };
    const Ray* rays;
    Outputs<T> out;
    __device__ Ray start(size_t i, Payload& p) const { p.calls = 0; p.hash = kHashSeed; return rays[i]; }
    __device__ bool accept(Payload& p, uint32_t inst, size_t id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(mix(p.hash, inst), id), bits(t)), bits(u)), bits(v));
        return keep<kFilter>(inst);
    }
    __device__ void finish(size_t i, const Payload& p, const typename DeviceView<T>::Hit& hit, uint32_t inst) const {
        write(out, i, (uint32_t)hit.prim_id, hit.t, hit.u, hit.v, inst, p.calls, p.hash);
    }
};
// The same through trace_triangles: one mesh, instance 0
template <typename T> struct TriangleShader {
    TestShader<T, 0> s;
    using Payload = typename TestShader<T, 0>::Payload;
    __device__ typename TestShader<T, 0>::Ray start(size_t i, Payload& p) const { return s.start(i, p); }
    __device__ bool accept(Payload& p, size_t id, T t, T u, T v) const { return s.accept(p, 0, id, t, u, v); }
    __device__ void finish(size_t i, const Payload& p, const typename DeviceView<T>::Hit& hit) const {
        s.finish(i, p, hit, hit.prim_id == (decltype(hit.prim_id))~0ull ? kNone : 0);
    }
};

// One ray through the two levels by hand: the top view's intersect, whose leaf transforms the ray (detail::object_ray)
// and runs the bottom view's intersect with intersect_tri, the tie rule on (instance, id) and the filter.  `visit(inst,
// id, t, u, v)` is the filter after the tie rule; it returns whether the candidate is taken.  Returns the instance of
// the hit (kNone: none); `ray.tmax` is the hit's t.
template <typename T, bool kAny, bool kRobust, bool kLast, typename Visit>
__device__ uint32_t nested_ray(const DeviceView<T>& top, const Instance<T>* records, typename DeviceView<T>::Ray& ray, uint32_t& best_id,
                               T& bu, T& bv, Visit&& visit) {
    using View = DeviceView<T>;
    uint32_t best_inst = kNone;
    best_id = kNone; bu = T(0); bv = T(0);
    if (ray.tmin != ray.tmin || ray.tmax != ray.tmax) return kNone;      // a NaN interval: a miss, no accept call
    typename View::template SmallStack<kStack> stack;
    top.template intersect<kAny, kRobust>(ray, top.root_index(), stack, [&](size_t b, size_t e) {
        for (size_t k = b; k < e; ++k) {
            const uint32_t inst = top.prim_id(k);
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
__global__ void __launch_bounds__(kBlock) per_thread_kernel(DeviceView<T> top, const Instance<T>* records, TestShader<T, kFilter> shader,
                                                          size_t n) {
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (i >= n) return;
    typename TestShader<T, kFilter>::Payload p;
    typename DeviceView<T>::Ray ray = shader.start(i, p);
    const T tmax_in = ray.tmax;
    uint32_t id;
    T u, v;
    const uint32_t inst = nested_ray<T, kAny, kRobust, kLast>(top, records, ray, id, u, v, [&](uint32_t k, uint32_t pid, T t, T bu, T bv) {
        ++p.calls;
        p.hash = mix(mix(mix(mix(mix(p.hash, k), pid), bits(t)), bits(bu)), bits(bv));
        return keep<kFilter>(k);
    });
    write(shader.out, i, inst == kNone ? kNone : id, inst == kNone ? tmax_in : ray.tmax, u, v, inst, p.calls, p.hash);
}

template <typename T, bool kAny, bool kRobust, bool kLast, int kFilter>
int run_filter(const DeviceView<T>& top, const Instances<T>& inst, bool per_thread, size_t n, const void* rays, const Outputs<T>& out,
               void* ws, size_t bytes, cudaStream_t stream) {
    const TestShader<T, kFilter> shader { static_cast<const typename DeviceView<T>::Ray*>(rays), out };
    if (!per_thread) {
        top.template trace_instances<kAny, kRobust, kLast>(n, inst, shader, ws, bytes, stream);
        return 0;
    }
    if (top.depth + 1 > kStack || inst.max_depth + 1 > kStack) { g_error = "per-thread kernel: tree too deep"; return -1; }
    if (n == 0) return 0;
    per_thread_kernel<T, kAny, kRobust, kLast, kFilter><<<(unsigned)((n + kBlock - 1) / kBlock), kBlock, 0, stream>>>(top, inst.records, shader, n);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { g_error = std::string("per-thread kernel: ") + cudaGetErrorString(e); return -1; }
    return 0;
}

template <typename T, bool kAny, bool kRobust, bool kLast>
int run_flags(int filter, const DeviceView<T>& top, const Instances<T>& inst, bool per_thread, size_t n, const void* rays,
              const Outputs<T>& out, void* ws, size_t bytes, cudaStream_t s) {
    if (filter == 0) return run_filter<T, kAny, kRobust, kLast, 0>(top, inst, per_thread, n, rays, out, ws, bytes, s);
    return run_filter<T, kAny, kRobust, kLast, 1>(top, inst, per_thread, n, rays, out, ws, bytes, s);
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

template <typename F> int by_flags(unsigned flags, F&& f) {
    const int k = (flags & BVH_ANY_HIT ? 1 : 0) | (flags & BVH_ROBUST ? 2 : 0) | (flags & BVH_TIE_LAST_VISITED ? 4 : 0);
    using B0 = std::false_type; using B1 = std::true_type;
    switch (k) {
    case 0: return f(B0(), B0(), B0());
    case 1: return f(B1(), B0(), B0());
    case 2: return f(B0(), B1(), B0());
    case 3: return f(B1(), B1(), B0());
    case 4: return f(B0(), B0(), B1());
    case 5: return f(B1(), B0(), B1());
    case 6: return f(B0(), B1(), B1());
    default: return f(B1(), B1(), B1());
    }
}

template <typename T>
int make_records(typename Api<T>::Handle* const* meshes, const uint32_t* mesh_of, const T* matrices, size_t count, Instance<T>* d_records,
            size_t* max_depth, void* stream) {
    std::vector<Instance<T>> recs(count);
    size_t depth = 0;
    for (size_t k = 0; k < count; ++k) {
        DeviceView<T> view;
        if (!get_view<T>(meshes[mesh_of[k]], view)) return -1;
        recs[k] = cu::make_instance(view, matrices + 12 * k);
        depth = view.depth > depth ? view.depth : depth;
    }
    *max_depth = depth;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemcpyAsync(d_records, recs.data(), count * sizeof(Instance<T>), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { g_error = cudaGetErrorString(e); return -1; }
    return 0;
}

template <typename T> __global__ void set_matrices_kernel(Instance<T>* records, const T* matrices, size_t count) {
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i < 12 * count) records[i / 12].object_to_world[i % 12] = matrices[i];
}

template <typename T>
int run(typename Api<T>::Handle* h, Instance<T>* recs, size_t count, size_t max_depth, int per_thread, int filter, unsigned flags,
        const void* rays, size_t n, Outputs<T> out, void* ws, size_t bytes, void* stream) {
    DeviceView<T> top;
    if (!get_view<T>(h, top)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : top.stream);
    const Instances<T> inst { recs, count, max_depth };
    return guarded([&] {
        return by_flags(flags, [&](auto any, auto robust, auto last) {
            return run_flags<T, decltype(any)::value, decltype(robust)::value, decltype(last)::value>(filter, top, inst, per_thread, n, rays,
                                                                                                     out, ws, bytes, s);
        });
    });
}

template <typename T>
int triangles(typename Api<T>::Handle* h, unsigned flags, const void* rays, size_t n, Outputs<T> out, void* ws, size_t bytes, void* stream) {
    DeviceView<T> view;
    if (!get_view<T>(h, view)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : view.stream);
    const TriangleShader<T> shader { { static_cast<const typename DeviceView<T>::Ray*>(rays), out } };
    return guarded([&] {
        return by_flags(flags, [&](auto any, auto robust, auto last) {
            view.template trace_triangles<decltype(any)::value, decltype(robust)::value, decltype(last)::value>(n, shader, ws, bytes, s);
            return 0;
        });
    });
}

// The benchmark's shaders: rays in, 16-byte records and the instance out, nothing per ray beyond the traversal's state.
struct PlainShader {
    struct Payload {};
    const bvh_ray3f* rays;
    bvh_hit3f* hits;
    uint32_t* inst;
    __device__ bvh_ray3f start(size_t i, Payload&) const { return rays[i]; }
    __device__ bool accept(Payload&, uint32_t, size_t, float, float, float) const { return true; }
    __device__ void finish(size_t i, const Payload&, const bvh_hit3f& hit, uint32_t k) const { hits[i] = hit; inst[i] = k; }
};
struct PlainTriangleShader {
    struct Payload {};
    const bvh_ray3f* rays;
    bvh_hit3f* hits;
    __device__ bvh_ray3f start(size_t i, Payload&) const { return rays[i]; }
    __device__ bool accept(Payload&, size_t, float, float, float) const { return true; }
    __device__ void finish(size_t i, const Payload&, const bvh_hit3f& hit) const { hits[i] = hit; }
};
// What a caller writes without trace_instances: a DeviceView::trace tracer whose leaf runs each instance's bottom tree
// with intersect and a per-thread stack (nested_ray's leaf), and carries tmax back.
struct NestedTracer {
    struct Payload { uint32_t inst, id; float u, v; };
    const bvh_ray3f* rays;
    const Instance<float>* records;
    const uint32_t* top_ids;
    bvh_hit3f* hits;
    uint32_t* inst;
    __device__ bvh_ray3f start(size_t i, Payload& p) const { p.inst = kNone; p.id = kNone; p.u = p.v = 0.0f; return rays[i]; }
    __device__ bool leaf(Payload& p, bvh_ray3f& ray, size_t b, size_t e) const {
        using View = DeviceView<float>;
        for (size_t k = b; k < e; ++k) {
            const uint32_t id_inst = top_ids[k];
            const Instance<float>& rec = records[id_inst];
            if (cu::detail::instance_is_singular(rec.world_to_object)) continue;
            View bottom;
            bottom.nodes = rec.nodes; bottom.prim_ids = rec.prim_ids; bottom.tris = rec.tris; bottom.depth = rec.depth;
            bvhb200::RayCtx<float> w, o;
            cu::detail::load_ray<float>(ray, w);
            cu::detail::object_ray(rec.world_to_object, w, o);
            bvh_ray3f oray = cu::detail::make_ray<bvh_ray3f>(o);
            View::SmallStack<kStack> bstack;
            bottom.intersect<false, false>(oray, rec.root_index, bstack, [&](size_t lb, size_t le) {
                for (size_t q = lb; q < le; ++q) {
                    float t, u, v;
                    if (!bottom.intersect_tri(q, oray, t, u, v)) continue;
                    const uint32_t id = (uint32_t)bottom.prim_id(q);
                    if (p.inst != kNone && !(t < oray.tmax) && !(id_inst < p.inst || (id_inst == p.inst && id < p.id))) continue;
                    oray.tmax = t; p.inst = id_inst; p.id = id; p.u = u; p.v = v;
                }
                return false;
            });
            ray.tmax = oray.tmax;
        }
        return p.inst != kNone;
    }
    __device__ void finish(size_t i, const Payload& p, const bvh_ray3f& ray) const {
        bvh_hit3f h;
        h.prim_id = p.inst == kNone ? kNone : p.id;
        h.t = ray.tmax; h.u = p.u; h.v = p.v;
        hits[i] = h;
        inst[i] = p.inst;
    }
};

} // namespace

#define DIT_EXPORT extern "C" __attribute__((visibility("default")))
#define DIT_ENTRY(T, S)                                                                                                   \
    DIT_EXPORT int dit_records##S(bvh##S* const* meshes, const uint32_t* mesh_of, const T* matrices, size_t count,        \
                                  void* records, size_t* max_depth, void* stream) {                                      \
        return make_records<T>(meshes, mesh_of, matrices, count, static_cast<Instance<T>*>(records), max_depth, stream);       \
    }                                                                                                                    \
    DIT_EXPORT int dit_set_matrices##S(void* records, const T* matrices, size_t count, void* stream) {                   \
        if (count == 0) return 0;                                                                                        \
        set_matrices_kernel<T><<<(unsigned)((12 * count + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(     \
            static_cast<Instance<T>*>(records), matrices, count);                                                        \
        const cudaError_t e = cudaGetLastError();                                                                        \
        if (e != cudaSuccess) { g_error = cudaGetErrorString(e); return -1; }                                            \
        return 0;                                                                                                        \
    }                                                                                                                    \
    DIT_EXPORT int dit_prepare##S(void* records, size_t count, size_t max_depth, void* bboxes, void* centers, void* stream) { \
        const Instances<T> inst { static_cast<Instance<T>*>(records), count, max_depth };                                 \
        return guarded([&] {                                                                                             \
            cu::prepare_instances(inst, static_cast<bvh_bbox##S*>(bboxes), static_cast<bvh_vec##S*>(centers), stream);  \
            return 0;                                                                                                    \
        });                                                                                                              \
    }                                                                                                                    \
    DIT_EXPORT int dit_run##S(bvh##S* top, void* records, size_t count, size_t max_depth, int per_thread, int filter,     \
                              unsigned flags, const void* rays, size_t n, uint32_t* ids, T* t, T* u, T* v, uint32_t* inst, \
                              uint32_t* calls, uint64_t* hashes, uint32_t* counts, void* ws, size_t bytes, void* stream) {  \
        return run<T>(top, static_cast<Instance<T>*>(records), count, max_depth, per_thread, filter, flags, rays, n,       \
                      Outputs<T> { ids, t, u, v, inst, calls, hashes, counts }, ws, bytes, stream);                       \
    }                                                                                                                    \
    DIT_EXPORT int dit_triangles##S(bvh##S* mesh, unsigned flags, const void* rays, size_t n, uint32_t* ids, T* t, T* u,   \
                                    T* v, uint32_t* inst, uint32_t* calls, uint64_t* hashes, void* ws, size_t bytes,       \
                                    void* stream) {                                                                      \
        return triangles<T>(mesh, flags, rays, n, Outputs<T> { ids, t, u, v, inst, calls, hashes, nullptr }, ws, bytes,    \
                            stream);                                                                                     \
    }                                                                                                                    \
    DIT_EXPORT size_t dit_record_bytes##S() { return sizeof(Instance<T>); }

DIT_ENTRY(float, 3f)
DIT_ENTRY(double, 3d)

DIT_EXPORT int dit_plain3f(bvh3f* top, void* records, size_t count, size_t max_depth, const void* rays, size_t n, void* hits,
                           uint32_t* inst, void* ws, size_t bytes, void* stream) {
    DeviceView<float> view;
    if (!get_view<float>(top, view)) return -1;
    const Instances<float> instances { static_cast<Instance<float>*>(records), count, max_depth };
    return guarded([&] {
        view.trace_instances<false, false>(n, instances, PlainShader { static_cast<const bvh_ray3f*>(rays), static_cast<bvh_hit3f*>(hits), inst },
                                           ws, bytes, stream ? stream : view.stream);
        return 0;
    });
}

DIT_EXPORT int dit_plain_triangles3f(bvh3f* mesh, const void* rays, size_t n, void* hits, void* ws, size_t bytes, void* stream) {
    DeviceView<float> view;
    if (!get_view<float>(mesh, view)) return -1;
    return guarded([&] {
        view.trace_triangles<false, false>(n, PlainTriangleShader { static_cast<const bvh_ray3f*>(rays), static_cast<bvh_hit3f*>(hits) },
                                           ws, bytes, stream ? stream : view.stream);
        return 0;
    });
}

DIT_EXPORT int dit_nested_trace3f(bvh3f* top, void* records, size_t max_depth, const void* rays, size_t n, void* hits, uint32_t* inst,
                                  void* ws, size_t bytes, void* stream) {
    DeviceView<float> view;
    if (!get_view<float>(top, view)) return -1;
    if (view.depth + 1 > kStack || max_depth + 1 > kStack) { g_error = "nested tracer: tree too deep"; return -1; }
    const NestedTracer tracer { static_cast<const bvh_ray3f*>(rays), static_cast<const Instance<float>*>(records), view.prim_ids,
                                static_cast<bvh_hit3f*>(hits), inst };
    return guarded([&] {
        view.trace<false, false>(n, tracer, ws, bytes, stream ? stream : view.stream);
        return 0;
    });
}

DIT_EXPORT const char* dit_last_error() { return g_error.c_str(); }
