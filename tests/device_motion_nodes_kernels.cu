// tests/device_motion_nodes_kernels.cu — test shaders for prepare_motion_nodes, node_at and the motion-node forms of
// DeviceView::trace_triangles and trace_paths (include/bvh/v2/cuda/intersect.cuh).
//
// Compiled for sm_90a with the library's NVCC_FLAGS (--fmad=false among them) into
// tests/_build/libdevice_motion_nodes_kernels.so (bvh_b200/build_ext.py build_device_motion_nodes_tests) and driven by
// tests/test_device_motion_nodes_gpu.py and scripts/motion_triangle_trace_bench.py.  The shaders are those of
// tests/device_motion_triangle_kernels.cu.  Every array is device-resident unless said otherwise; keys0 / keys1 are the
// count x 9 vertex keys (original order), nodes the node_count + 1 MotionNode records of the handle's tree.
//   dmn_prepare{3f,3d}     prepare_motion_nodes of the handle's view on `stream`.
//   dmn_node_at{3f,3d}     node_at(nodes, s, tau) for every slot s in [1, node_count], 6 values each at out + 6 s.
//   dmn_extent{3f,3d}      per slot, the extent of triangle_at at tau over the finite triangles of the node's subtree (a
//                          traverse_bottom_up pass; +inf / -inf when there are none), 6 values at out + 6 s.
//   dmn_run{3f,3d}         one batch of rays, ray i at times[i], through the motion-node trace_triangles (mode 0), the
//                          motion trace_triangles over the handle's boxes (mode 1), one thread per ray through
//                          traverse_top_down with a node test applying node_at and the slab test (mode 2; inner steps and
//                          triangle tests per ray into inner / tests), or the motion-node call on a copy of the view whose
//                          node bounds are NaN (mode 3).  Filter 0 accepts every hit, 1 rejects odd ids.  Outputs as in
//                          dmt_run; each may be null.
//   dmn_tracer{3f,3d}      the grey diffuse path tracer, path i at times[i], through one motion-node trace_paths call
//                          (mode 0), a wavefront loop of motion-node trace_triangles launches (mode 1, dmn_wavefront_bytes(n)
//                          bytes of scratch) or the motion trace_paths over the handle's boxes (mode 2).
//   dmn_plain3f            float, closest-hit, accept all: 16-byte records through the motion-node trace_triangles: the
//                          benchmark's shader.
// Each returns 0; -1 with a message in dmn_last_error(); -2 when the call threw std::length_error, -3 when it threw
// std::invalid_argument, with its message.
#include <cuda_runtime.h>

#include <bvh/v2/cuda/intersect.cuh>

#include <cstdint>
#include <stdexcept>
#include <string>

namespace {

namespace cu = bvh::v2::cuda;
using cu::DeviceView;
using cu::MotionTriangles;
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

template <int kFilter> __device__ inline bool keep(size_t id) { return kFilter == 0 || (id & 1) == 0; }

template <typename T> struct Outputs {
    uint32_t* ids; T* t; T* u; T* v; uint32_t* calls; uint64_t* hashes; uint32_t* counts;
};
template <typename T> __device__ inline void write(const Outputs<T>& out, size_t i, uint32_t id, T t, T u, T v, uint32_t calls, uint64_t hash) {
    if (out.ids) out.ids[i] = id;
    if (out.t) out.t[i] = t;
    if (out.u) { out.u[i] = u; out.v[i] = v; }
    if (out.calls) out.calls[i] = calls;
    if (out.hashes) out.hashes[i] = hash;
    if (out.counts) atomicAdd(out.counts + i, 1u);
}

// The recording shader, ray i at times[i] (the static form ignores the time)
template <typename T, int kFilter> struct TestShader {
    using Ray = typename DeviceView<T>::Ray;
    struct Payload { uint32_t calls; uint64_t hash; };
    const Ray* rays;
    const T* times;
    Outputs<T> out;
    __device__ Ray start(size_t i, Payload& p, T& time) const { time = times[i]; return start(i, p); }
    __device__ Ray start(size_t i, Payload& p) const { p.calls = 0; p.hash = kHashSeed; return rays[i]; }
    __device__ bool accept(Payload& p, size_t id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(p.hash, id), bits(t)), bits(u)), bits(v));
        return keep<kFilter>(id);
    }
    __device__ void finish(size_t i, const Payload& p, const typename DeviceView<T>::Hit& hit) const {
        write(out, i, (uint32_t)hit.prim_id, hit.t, hit.u, hit.v, p.calls, p.hash);
    }
};

// Triangle `id` of the keys at `time` against the ray, as the motion leaf tests it: PrecomputedTri::intersect of
// precompute_tri(triangle_at(...)) with t in [tmin, tmax]
template <typename T>
__device__ bool test_at(const MotionTriangles<T>& keys, uint32_t id, T time, const typename DeviceView<T>::Ray& ray, T& t, T& u, T& v) {
    T w[9];
    cu::triangle_at(keys, id, time, w);
    const bvhb200::DevTri<T> tri = bvhb200::precompute_tri(w);
    bvhb200::RayCtx<T> r;
    cu::detail::load_ray<T>(ray, r);
    bvhb200::HitState<T> h { bvhb200::kInvalidId, r.tmax, T(0), T(0) };
    if (!bvhb200::tri_test<T>(tri, 0, nullptr, false, r, h)) return false;
    t = h.t; u = h.u; v = h.v;
    return true;
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

// ---------------------------------------------------------------------------------------------------------------------
// The path tracer
// ---------------------------------------------------------------------------------------------------------------------

// A grey diffuse path tracer with a point light and next-event shadow segments (tests/device_path_trace_kernels.cu's
// arithmetic), path i at times[i]; a triangle's normal is taken from triangle_at at the path's time.
template <typename T> struct MotionPathTracer {
    using View = DeviceView<T>;
    using Ray = typename View::Ray;
    using Hit = typename View::Hit;
    struct Payload { T throughput, radiance, pending, time; uint32_t prim, bounce, segments, hash; };
    static constexpr T kAlbedo = T(0.7), kSky = T(0.25), kLight = T(2.0);

    const Ray* primary;
    const T* times;
    T light[3];
    MotionTriangles<T> keys;
    uint32_t max_bounces;
    T* radiance; uint32_t* segments; uint32_t* hashes; uint32_t* counts;

    __device__ void normal(uint32_t prim, bool flip, T time, T n[3]) const {
        T w[9];
        cu::triangle_at(keys, prim, time, w);
        const T e1[3] = { w[3] - w[0], w[4] - w[1], w[5] - w[2] }, e2[3] = { w[6] - w[0], w[7] - w[1], w[8] - w[2] };
        const T c[3] = { e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0] };
        const T len = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
        const T s = len > T(0) ? (flip ? T(-1) / len : T(1) / len) : T(0);
        for (int a = 0; a < 3; ++a) n[a] = c[a] * s;
    }

    __device__ PathStep start(size_t i, Payload& p, Ray& ray, T& time) const {
        const PathStep step = start(i, p, ray);
        time = p.time;
        return step;
    }
    __device__ PathStep start(size_t i, Payload& p, Ray& ray) const {
        ray = primary[i];
        p.throughput = T(1); p.radiance = T(0); p.pending = T(0); p.time = times[i];
        p.prim = kNone; p.bounce = 0; p.segments = 0; p.hash = 2166136261u;
        return PathStep::Closest;
    }
    __device__ bool accept(Payload& p, size_t prim_id, T, T, T) const { return prim_id != p.prim; }

    __device__ PathStep bounce(size_t i, Payload& p, Ray& ray) const {
        if ((p.bounce >> 1) >= max_bounces) return PathStep::End;
        const uint32_t h = hash32((uint32_t)i * 0x9E3779B9u ^ hash32(p.segments));
        const T u1 = T(h >> 16) * T(1.0 / 65536), u2 = T(h & 0xFFFFu) * T(1.0 / 65536);
        const T z = T(1) - T(2) * u1, rr = sqrt(fmax(T(0), T(1) - z * z)), phi = T(6.283185307179586) * u2;
        T d[3] = { rr * cos(phi), rr * sin(phi), z }, n[3];
        normal(p.prim, p.bounce & 1u, p.time, n);
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
        normal(p.prim, false, p.time, n);
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

// The wavefront form: the path state in arrays, one motion trace_triangles pass per segment kind, the path's time
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

// The benchmark's shader: rays and times in, 16-byte records out (the static form ignores the times)
struct PlainShader {
    struct Payload {};
    const bvh_ray3f* rays;
    const float* times;
    bvh_hit3f* hits;
    __device__ bvh_ray3f start(size_t i, Payload&, float& time) const { time = times[i]; return rays[i]; }
    __device__ bvh_ray3f start(size_t i, Payload&) const { return rays[i]; }
    __device__ bool accept(Payload&, size_t, float, float, float) const { return true; }
    __device__ void finish(size_t i, const Payload&, const bvh_hit3f& hit) const { hits[i] = hit; }
};

// ---------------------------------------------------------------------------------------------------------------------
// Motion nodes
// ---------------------------------------------------------------------------------------------------------------------

struct Pick { bool left, right, swap; };

// One ray at `time`, one thread: the view's traverse_top_down from the motion nodes' root with a three-argument node test
// that takes each child's box from node_at at that time and applies the library's slab test (node_test), and a leaf
// that tests each slot's triangle at that time (test_at) with the canonical tie rule (unless kLast) and the filter
// (visit).  Counts inner steps and triangle tests.  Returns the hit's original id (kNone: none); ray.tmax is its t.
template <typename T, bool kAny, bool kRobust, bool kLast, typename Visit>
__device__ uint32_t node_at_ray(const DeviceView<T>& view, const MotionTriangles<T>& keys, const cu::MotionNodes<T>& mn, T time,
                                typename DeviceView<T>::Ray& ray, T& bu, T& bv, uint32_t& steps, uint32_t& tests, Visit&& visit) {
    uint32_t best = kNone;
    bu = T(0); bv = T(0);
    if (ray.tmin != ray.tmin || ray.tmax != ray.tmax) return kNone;      // a NaN interval: a miss, no accept call
    bvhb200::RayCtx<T> r;
    cu::detail::load_ray<T>(ray, r);
    bvhb200::ray_prologue<T, kRobust>(r);
    typename DeviceView<T>::template SmallStack<kStack> stack;
    view.template traverse_top_down<kAny>(mn.nodes[1].index, stack, [&](size_t b, size_t e) {
        for (size_t k = b; k < e; ++k) {
            const uint32_t id = (uint32_t)view.prim_id(k);
            T t, u, v;
            ++tests;
            if (!test_at(keys, id, time, ray, t, u, v)) continue;
            if (!kLast && best != kNone && !(t < ray.tmax) && !(id < best)) continue;      // canonical tie rule
            if (!visit(id, t, u, v)) continue;
            ray.tmax = t; best = id; bu = u; bv = v;
        }
        r.tmax = ray.tmax;
        return best != kNone;
    }, [&](const typename DeviceView<T>::Node&, const typename DeviceView<T>::Node&, size_t left) {
        T lb[6], rb[6], l0, l1, r0, r1;
        cu::node_at(mn, left + 1, time, lb);
        cu::node_at(mn, left + 2, time, rb);
        bvhb200::node_test<T, kRobust>(lb, r, l0, l1);
        bvhb200::node_test<T, kRobust>(rb, r, r0, r1);
        ++steps;
        return Pick { l0 <= l1, r0 <= r1, !kAny && l0 > r0 };
    });
    return best;
}

template <typename T, bool kAny, bool kRobust, bool kLast, int kFilter>
__global__ void __launch_bounds__(kBlock) node_at_kernel(DeviceView<T> view, MotionTriangles<T> keys, cu::MotionNodes<T> mn,
                                                         TestShader<T, kFilter> shader, size_t n, uint32_t* inner, uint32_t* tests) {
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (i >= n) return;
    typename TestShader<T, kFilter>::Payload p;
    T time;
    typename DeviceView<T>::Ray ray = shader.start(i, p, time);
    const T tmax_in = ray.tmax;
    T u, v;
    uint32_t steps = 0, count = 0;
    const uint32_t id = node_at_ray<T, kAny, kRobust, kLast>(view, keys, mn, time, ray, u, v, steps, count, [&](uint32_t pid, T t, T bu, T bv) {
        ++p.calls;
        p.hash = mix(mix(mix(mix(p.hash, pid), bits(t)), bits(bu)), bits(bv));
        return keep<kFilter>(pid);
    });
    write(shader.out, i, id, id == kNone ? tmax_in : ray.tmax, u, v, p.calls, p.hash);
    if (inner) inner[i] = steps;
    if (tests) tests[i] = count;
}

// The view's nodes with every bound NaN and the indices kept
template <typename T> __global__ void nan_nodes_kernel(const bvhb200::DevNode<T>* src, bvhb200::DevNode<T>* dst, size_t slots) {
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= slots) return;
    bvhb200::DevNode<T> node = src[i];
    for (int k = 0; k < 6; ++k) node.bounds[k] = T(NAN);
    dst[i] = node;
}

// node_at of every slot 1 .. node_count at tau, 6 values each (slot 0 left as it is)
template <typename T> __global__ void node_at_all_kernel(cu::MotionNodes<T> mn, T tau, T* out) {
    const size_t s = 1 + (size_t)blockIdx.x * 256 + threadIdx.x;
    if (s <= mn.node_count) cu::node_at(mn, s, tau, out + 6 * s);
}

// The extent of triangle_at at tau over the finite triangles of each node's subtree (+inf / -inf for none), per slot, as a
// bottom-up pass: what node_at's box must hold
template <typename T> struct Extent {
    const uint32_t* prim_ids;
    MotionTriangles<T> keys;
    T tau;
    T* out;
    __device__ void operator()(size_t node, size_t begin, size_t end) const {
        T e[6] = { T(INFINITY), T(-INFINITY), T(INFINITY), T(-INFINITY), T(INFINITY), T(-INFINITY) };
        for (size_t k = begin; k < end; ++k) {
            const uint32_t id = prim_ids[k];
            bool ok = true;
            for (int q = 0; q < 9; ++q) ok = ok && isfinite(keys.vertices[0][9 * id + q]) && isfinite(keys.vertices[1][9 * id + q]);
            if (!ok) continue;
            T v[9];
            cu::triangle_at(keys, id, tau, v);
            for (int q = 0; q < 9; ++q) { e[2 * (q % 3)] = fmin(e[2 * (q % 3)], v[q]); e[2 * (q % 3) + 1] = fmax(e[2 * (q % 3) + 1], v[q]); }
        }
        for (int q = 0; q < 6; ++q) out[6 * (node + 1) + q] = e[q];
    }
    __device__ void operator()(size_t node, size_t left) const {
        const T* l = out + 6 * (left + 1);
        const T* r = out + 6 * (left + 2);
        for (int a = 0; a < 3; ++a) {
            out[6 * (node + 1) + 2 * a] = fmin(__ldcg(l + 2 * a), __ldcg(r + 2 * a));
            out[6 * (node + 1) + 2 * a + 1] = fmax(__ldcg(l + 2 * a + 1), __ldcg(r + 2 * a + 1));
        }
    }
};

template <typename T, bool kAny, bool kRobust, bool kLast, int kFilter>
int run_nodes_filter(const DeviceView<T>& view, const MotionTriangles<T>& keys, const cu::MotionNodes<T>& mn, int mode, size_t n,
                     const void* rays, const T* times, const Outputs<T>& out, uint32_t* inner, uint32_t* tests, void* ws, size_t bytes,
                     cudaStream_t stream) {
    const TestShader<T, kFilter> shader { static_cast<const typename DeviceView<T>::Ray*>(rays), times, out };
    if (mode == 0) {
        view.template trace_triangles<kAny, kRobust, kLast>(n, keys, mn, shader, ws, bytes, stream);
        return 0;
    }
    if (mode == 1) {
        view.template trace_triangles<kAny, kRobust, kLast>(n, keys, shader, ws, bytes, stream);
        return 0;
    }
    if (mode == 3) {                    // the motion nodes through a view whose node bounds are all NaN
        const size_t slots = view.node_count + 1;
        bvhb200::DevNode<T>* copy = nullptr;
        if (cudaMallocAsync(reinterpret_cast<void**>(&copy), slots * sizeof(bvhb200::DevNode<T>), stream) != cudaSuccess) {
            g_error = "nan view: cudaMallocAsync";
            return -1;
        }
        nan_nodes_kernel<T><<<(unsigned)((slots + 255) / 256), 256, 0, stream>>>(view.nodes, copy, slots);
        DeviceView<T> nan_view = view;
        nan_view.nodes = copy;
        int rc = 0;
        try {
            nan_view.template trace_triangles<kAny, kRobust, kLast>(n, keys, mn, shader, ws, bytes, stream);
        } catch (...) {
            cudaFreeAsync(copy, stream);
            throw;
        }
        cudaFreeAsync(copy, stream);
        return rc;
    }
    if (view.depth + 1 > kStack) { g_error = "per-thread kernel: tree too deep"; return -1; }
    if (n == 0) return 0;
    node_at_kernel<T, kAny, kRobust, kLast, kFilter><<<(unsigned)((n + kBlock - 1) / kBlock), kBlock, 0, stream>>>(view, keys, mn, shader, n,
                                                                                                                  inner, tests);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { g_error = std::string("per-thread kernel: ") + cudaGetErrorString(e); return -1; }
    return 0;
}

template <typename T>
int run_nodes(typename Api<T>::Handle* h, const T* keys0, const T* keys1, size_t count, const void* nodes, size_t node_count, int mode,
              int filter, unsigned flags, const void* rays, const T* times, size_t n, Outputs<T> out, uint32_t* inner, uint32_t* tests,
              void* ws, size_t bytes, void* stream) {
    DeviceView<T> view;
    if (!get_view<T>(h, view)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : view.stream);
    const MotionTriangles<T> keys { { keys0, keys1 }, count };
    const cu::MotionNodes<T> mn { static_cast<const cu::MotionNode<T>*>(nodes), node_count };
    return guarded([&] {
        return by_flags(flags, [&]<bool kAny, bool kRobust, bool kLast>() {
            if (filter == 0) return run_nodes_filter<T, kAny, kRobust, kLast, 0>(view, keys, mn, mode, n, rays, times, out, inner, tests, ws, bytes, s);
            return run_nodes_filter<T, kAny, kRobust, kLast, 1>(view, keys, mn, mode, n, rays, times, out, inner, tests, ws, bytes, s);
        });
    });
}

template <typename T>
int tracer(typename Api<T>::Handle* h, const T* keys0, const T* keys1, size_t count, const void* nodes, size_t node_count, int mode,
           unsigned flags, size_t n, const void* primary, const T* times, const T* light, uint32_t max_bounces, T* radiance,
           uint32_t* segments, uint32_t* hashes, uint32_t* counts, void* scratch, void* ws, size_t bytes, void* stream) {
    DeviceView<T> view;
    if (!get_view<T>(h, view)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : view.stream);
    MotionPathTracer<T> shader;
    shader.primary = static_cast<const typename DeviceView<T>::Ray*>(primary);
    shader.times = times;
    for (int a = 0; a < 3; ++a) shader.light[a] = light[a];
    shader.keys = MotionTriangles<T> { { keys0, keys1 }, count };
    shader.max_bounces = max_bounces;
    shader.radiance = radiance; shader.segments = segments; shader.hashes = hashes; shader.counts = counts;
    const cu::MotionNodes<T> mn { static_cast<const cu::MotionNode<T>*>(nodes), node_count };
    return guarded([&] {
        return by_path_flags(flags, [&]<bool kRobust, bool kLast>() {
            if (mode == 0) {
                view.template trace_paths<kRobust, kLast>(n, shader.keys, mn, shader, ws, bytes, s);
                return 0;
            }
            if (mode == 2) {
                view.template trace_paths<kRobust, kLast>(n, shader.keys, shader, ws, bytes, s);
                return 0;
            }
            if (n == 0) return 0;
            using S = MotionPathTracer<T>;
            const WavefrontState<S> st = wavefront_state<S>(scratch, n);
            wavefront_start_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(shader, st, n);
            const cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) throw std::runtime_error(std::string("wavefront start: ") + cudaGetErrorString(e));
            for (uint32_t k = 0; k < max_bounces + 1; ++k) {
                view.template trace_triangles<false, kRobust, kLast>(n, shader.keys, mn, WavefrontPass<S> { shader, st, PathStep::Closest }, ws,
                                                                     bytes, s);
                view.template trace_triangles<true, kRobust, kLast>(n, shader.keys, mn, WavefrontPass<S> { shader, st, PathStep::Occlusion }, ws,
                                                                    bytes, s);
            }
            return 0;
        });
    });
}

template <typename T>
int extent(typename Api<T>::Handle* h, const T* keys0, const T* keys1, size_t count, T tau, T* out, void* ws, size_t bytes, void* stream) {
    DeviceView<T> view;
    if (!get_view<T>(h, view)) return -1;
    return guarded([&] {
        view.traverse_bottom_up(ws, bytes, Extent<T> { view.prim_ids, MotionTriangles<T> { { keys0, keys1 }, count }, tau, out },
                                Extent<T> { view.prim_ids, MotionTriangles<T> { { keys0, keys1 }, count }, tau, out },
                                stream ? stream : view.stream);
        return 0;
    });
}

} // namespace

#define DMN_EXPORT extern "C" __attribute__((visibility("default")))
#define DMN_ENTRY(T, S)                                                                                                   \
    DMN_EXPORT int dmn_prepare##S(bvh##S* h, const T* keys0, const T* keys1, size_t count, void* nodes, void* ws, size_t bytes, \
                                  void* stream) {                                                                        \
        DeviceView<T> view;                                                                                              \
        if (!get_view<T>(h, view)) return -1;                                                                            \
        return guarded([&] {                                                                                             \
            cu::prepare_motion_nodes(view, MotionTriangles<T> { { keys0, keys1 }, count }, static_cast<cu::MotionNode<T>*>(nodes), ws, \
                                     bytes, stream ? stream : view.stream);                                              \
            return 0;                                                                                                    \
        });                                                                                                              \
    }                                                                                                                    \
    DMN_EXPORT int dmn_node_at##S(const void* nodes, size_t node_count, T tau, T* out, void* stream) {                   \
        if (node_count == 0) return 0;                                                                                   \
        node_at_all_kernel<T><<<(unsigned)((node_count + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(      \
            cu::MotionNodes<T> { static_cast<const cu::MotionNode<T>*>(nodes), node_count }, tau, out);                  \
        const cudaError_t e = cudaGetLastError();                                                                        \
        if (e != cudaSuccess) { g_error = cudaGetErrorString(e); return -1; }                                            \
        return 0;                                                                                                        \
    }                                                                                                                    \
    DMN_EXPORT int dmn_extent##S(bvh##S* h, const T* keys0, const T* keys1, size_t count, T tau, T* out, void* ws, size_t bytes, \
                                 void* stream) {                                                                         \
        return extent<T>(h, keys0, keys1, count, tau, out, ws, bytes, stream);                                           \
    }                                                                                                                    \
    DMN_EXPORT int dmn_run##S(bvh##S* h, const T* keys0, const T* keys1, size_t count, const void* nodes, size_t node_count, int mode, \
                              int filter, unsigned flags, const void* rays, const T* times, size_t n, uint32_t* ids, T* t, T* u, \
                              T* v, uint32_t* calls, uint64_t* hashes, uint32_t* counts, uint32_t* inner, uint32_t* tests,  \
                              void* ws, size_t bytes, void* stream) {                                                    \
        return run_nodes<T>(h, keys0, keys1, count, nodes, node_count, mode, filter, flags, rays, times, n,              \
                            Outputs<T> { ids, t, u, v, calls, hashes, counts }, inner, tests, ws, bytes, stream);        \
    }                                                                                                                    \
    DMN_EXPORT int dmn_tracer##S(bvh##S* h, const T* keys0, const T* keys1, size_t count, const void* nodes, size_t node_count, \
                                 int mode, unsigned flags, size_t n, const void* primary, const T* times, const T* light,  \
                                 uint32_t max_bounces, T* radiance, uint32_t* segments, uint32_t* hashes, uint32_t* counts, \
                                 void* scratch, void* ws, size_t bytes, void* stream) {                                  \
        return tracer<T>(h, keys0, keys1, count, nodes, node_count, mode, flags, n, primary, times, light, max_bounces, radiance, \
                         segments, hashes, counts, scratch, ws, bytes, stream);                                          \
    }                                                                                                                    \
    DMN_EXPORT size_t dmn_wavefront_bytes##S(size_t n) { return wavefront_bytes<MotionPathTracer<T>>(n); }

DMN_ENTRY(float, 3f)
DMN_ENTRY(double, 3d)

DMN_EXPORT int dmn_plain3f(bvh3f* h, const float* keys0, const float* keys1, size_t count, const void* nodes, size_t node_count,
                           const void* rays, const float* times, size_t n, void* hits, void* ws, size_t bytes, void* stream) {
    DeviceView<float> view;
    if (!get_view<float>(h, view)) return -1;
    const PlainShader shader { static_cast<const bvh_ray3f*>(rays), times, static_cast<bvh_hit3f*>(hits) };
    return guarded([&] {
        view.trace_triangles<false, false>(n, MotionTriangles<float> { { keys0, keys1 }, count },
                                           cu::MotionNodes<float> { static_cast<const cu::MotionNode<float>*>(nodes), node_count }, shader, ws,
                                           bytes, stream ? stream : view.stream);
        return 0;
    });
}

DMN_EXPORT const char* dmn_last_error() { return g_error.c_str(); }
