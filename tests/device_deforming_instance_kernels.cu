// tests/device_deforming_instance_kernels.cu — test shaders for the deforming forms of DeviceView::trace_instances and
// trace_instance_paths, make_deforming_instance and prepare_deforming_instances (include/bvh/v2/cuda/intersect.cuh).
//
// Compiled for sm_90a with the library's NVCC_FLAGS (--fmad=false among them) into
// tests/_build/libdevice_deforming_instance_kernels.so (bvh_b200/build_ext.py build_device_deforming_instance_tests) and
// driven by tests/test_device_deforming_instance_gpu.py and scripts/deforming_instance_trace_bench.py.  Every array is
// device-resident unless said otherwise.
//   ddi_records{3f,3d}     records from mesh handles (host array), per record its mesh, its kind (0 static, 1 deforming on
//                          shutter boxes, 2 deforming with motion nodes) and two keys (host, count x 12), per mesh its
//                          vertex keys and motion nodes (host arrays of device pointers), through make_deforming_instance,
//                          copied to `records`; the largest bottom depth through *max_depth.
//   ddi_set_keys{3f,3d}    both placement keys of every record from device arrays of count x 12 values.
//   ddi_prepare{3f,3d}     prepare_deforming_instances on `stream`.
//   ddi_bottom{3f,3d}      a deforming bottom's step: prepare_motion_triangles of the keys into boxes / centres and, when
//                          `nodes` is not null, prepare_motion_nodes of the handle's view into nodes.
//   ddi_run{3f,3d}         one batch of rays, ray i at times[i]: mode 0 the deforming trace_instances; mode 1 one thread per
//                          ray that builds instance_at per entered record and nests the bottom traversal by hand (the
//                          view's intersect, or traverse_top_down with node_at boxes, and a triangle_at leaf); mode 2 the
//                          motion trace_instances over MotionInstance copies of the records (in `scratch`); mode 3
//                          trace_triangles of the record 0's bottom: its static, motion or motion-node form by its kind
//                          (the accept hash with instance 0).  Filter 0 accepts every hit, 1 rejects odd instances.
//   ddi_paths{3f,3d}       scripted paths through the deforming trace_instance_paths: path i at times[i] runs the segments
//                          seg_rays[offsets[i] .. offsets[i + 1]) (kind by seg_any), records each as ddi_run does at
//                          that segment's index, and ray_ok = 1 when next received the segment's ray bit for bit.
//   ddi_plain3f            float, closest-hit, accept all: 16-byte records and the instance per ray (a plain shader for timing).
//   ddi_workaround3f       the same scene as two kinds of launch and a merge: the motion trace_instances over the static
//                          copies, then one motion-node trace_triangles per deforming copy (for timing).
// Each returns 0; -1 with a message in ddi_last_error(); -2 when the call threw std::length_error, -3 when it threw
// std::invalid_argument, with its message.
#include <cuda_runtime.h>

#include <bvh/v2/cuda/intersect.cuh>

#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace {

namespace cu = bvh::v2::cuda;
using cu::DeformingInstance;
using cu::DeformingInstances;
using cu::DeviceView;
using cu::Instance;
using cu::MotionInstance;
using cu::MotionInstances;
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

// The recording shader, ray i at times[i]; the triangle calls (mode 3) record instance 0
template <typename T, int kFilter> struct TestShader {
    using Ray = typename DeviceView<T>::Ray;
    using Hit = typename DeviceView<T>::Hit;
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
    __device__ bool accept(Payload& p, size_t id, T t, T u, T v) const { return accept(p, 0u, id, t, u, v); }
    __device__ void finish(size_t i, const Payload& p, const Hit& hit, uint32_t inst) const {
        write(out, i, (uint32_t)hit.prim_id, hit.t, hit.u, hit.v, inst, p.calls, p.hash);
    }
    __device__ void finish(size_t i, const Payload& p, const Hit& hit) const {
        write(out, i, (uint32_t)hit.prim_id, hit.t, hit.u, hit.v, (uint32_t)hit.prim_id == kNone ? kNone : 0u, p.calls, p.hash);
    }
};

// The static form of trace_triangles takes a shader without a time: TestShader with the times dropped
template <typename T, int kFilter> struct NoTime {
    using Payload = typename TestShader<T, kFilter>::Payload;
    TestShader<T, kFilter> s;
    __device__ typename DeviceView<T>::Ray start(size_t i, Payload& p) const { T time; return s.start(i, p, time); }
    __device__ bool accept(Payload& p, size_t id, T t, T u, T v) const { return s.accept(p, id, t, u, v); }
    __device__ void finish(size_t i, const Payload& p, const typename DeviceView<T>::Hit& h) const { s.finish(i, p, h); }
};

// The triangle of slot q of a bottom at `time`, tested against `ray` (static: the view's; deforming: triangle_at)
template <typename T>
__device__ bool test_slot(const DeformingInstance<T>& rec, const DeviceView<T>& bottom, size_t q, T time, const typename DeviceView<T>::Ray& ray,
                          T& t, T& u, T& v) {
    if (!rec.vertices[0]) return bottom.intersect_tri(q, ray, t, u, v);
    T w[9];
    cu::triangle_at(MotionTriangles<T> { { rec.vertices[0], rec.vertices[1] }, 0 }, bottom.prim_id(q), time, w);
    const bvhb200::DevTri<T> tri = bvhb200::precompute_tri(w);
    bvhb200::RayCtx<T> r;
    cu::detail::load_ray<T>(ray, r);
    bvhb200::HitState<T> h { bvhb200::kInvalidId, r.tmax, T(0), T(0) };
    if (!bvhb200::tri_test<T>(tri, 0, nullptr, false, r, h)) return false;
    t = h.t; u = h.u; v = h.v;
    return true;
}

struct Pick { bool left, right, swap; };

// One ray at `time` through the two levels by hand: the top view's intersect, whose leaf builds each record's placement
// with instance_at, transforms the ray (detail::object_ray) and runs the bottom traversal: the view's intersect (static
// and shutter-box bottoms) or traverse_top_down with node_at boxes and the library's slab test (motion-node bottoms),
// with test_slot, the tie rule on (instance, id) and the filter (visit).  Returns the instance of the hit (kNone: none);
// ray.tmax is its t.
template <typename T, bool kAny, bool kRobust, bool kLast, typename Visit>
__device__ uint32_t nested_ray(const DeviceView<T>& top, const DeformingInstance<T>* records, T time, typename DeviceView<T>::Ray& ray,
                               uint32_t& best_id, T& bu, T& bv, Visit&& visit) {
    using View = DeviceView<T>;
    uint32_t best_inst = kNone;
    best_id = kNone; bu = T(0); bv = T(0);
    if (ray.tmin != ray.tmin || ray.tmax != ray.tmax) return kNone;      // a NaN interval: a miss, no accept call
    typename View::template SmallStack<kStack> stack;
    top.template intersect<kAny, kRobust>(ray, top.root_index(), stack, [&](size_t b, size_t e) {
        for (size_t k = b; k < e; ++k) {
            const uint32_t inst = top.prim_id(k);
            const DeformingInstance<T>& drec = records[inst];
            const Instance<T> rec = cu::instance_at(drec, time);
            if (cu::detail::instance_is_singular(rec.world_to_object)) continue;
            View bottom;
            bottom.nodes = rec.nodes; bottom.prim_ids = rec.prim_ids; bottom.tris = rec.tris; bottom.depth = rec.depth;
            bvhb200::RayCtx<T> w, o;
            cu::detail::load_ray<T>(ray, w);
            cu::detail::object_ray(rec.world_to_object, w, o);
            typename View::Ray oray = cu::detail::make_ray<typename View::Ray>(o);
            auto leaf = [&](size_t lb, size_t le) {
                for (size_t q = lb; q < le; ++q) {
                    T t, u, v;
                    if (!test_slot(drec, bottom, q, time, oray, t, u, v)) continue;
                    const uint32_t id = (uint32_t)bottom.prim_id(q);
                    if (!kLast && best_inst != kNone && !(t < oray.tmax) &&
                        !(inst < best_inst || (inst == best_inst && id < best_id))) continue;      // canonical tie rule
                    if (!visit(inst, id, t, u, v)) continue;
                    oray.tmax = t; best_inst = inst; best_id = id; bu = u; bv = v;
                }
                return best_inst != kNone;
            };
            typename View::template SmallStack<kStack> bstack;
            if (drec.vertices[0] && drec.motion_nodes) {
                const cu::MotionNodes<T> mn { drec.motion_nodes, 0 };
                bvhb200::RayCtx<T> r = o;
                bvhb200::ray_prologue<T, kRobust>(r);
                bottom.template traverse_top_down<kAny>(rec.root_index, bstack, [&](size_t lb, size_t le) {
                    const bool hit = leaf(lb, le);
                    r.tmax = oray.tmax;
                    return hit;
                }, [&](const typename View::Node&, const typename View::Node&, size_t left) {
                    T lbx[6], rbx[6], l0, l1, r0, r1;
                    cu::node_at(mn, left + 1, time, lbx);
                    cu::node_at(mn, left + 2, time, rbx);
                    bvhb200::node_test<T, kRobust>(lbx, r, l0, l1);
                    bvhb200::node_test<T, kRobust>(rbx, r, r0, r1);
                    return Pick { l0 <= l1, r0 <= r1, !kAny && l0 > r0 };
                });
            } else {
                bottom.template intersect<kAny, kRobust>(oray, rec.root_index, bstack, leaf);
            }
            ray.tmax = oray.tmax;
            if (kAny && best_inst != kNone) return true;
        }
        return best_inst != kNone;
    });
    return best_inst;
}

template <typename T, bool kAny, bool kRobust, bool kLast, int kFilter>
__global__ void __launch_bounds__(kBlock) per_thread_kernel(DeviceView<T> top, const DeformingInstance<T>* records,
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

template <typename T> __global__ void to_motion_kernel(const DeformingInstance<T>* records, size_t count, MotionInstance<T>* out) {
    const size_t k = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= count) return;
    const DeformingInstance<T>& r = records[k];
    MotionInstance<T> m;
    m.nodes = r.nodes; m.prim_ids = r.prim_ids; m.tris = r.tris; m.root_index = r.root_index; m.depth = r.depth;
    for (int e = 0; e < 2; ++e)
        for (int j = 0; j < 12; ++j) m.object_to_world[e][j] = r.object_to_world[e][j];
    out[k] = m;
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

template <typename T, bool kAny, bool kRobust, bool kLast, int kFilter>
int run_filter(const DeviceView<T>& top, typename Api<T>::Handle* bottom_h, const DeformingInstances<T>& inst, int mode, size_t n,
               const void* rays, const T* times, const Outputs<T>& out, void* scratch, void* ws, size_t bytes, cudaStream_t stream) {
    const TestShader<T, kFilter> shader { static_cast<const typename DeviceView<T>::Ray*>(rays), times, out };
    if (mode == 0) {
        top.template trace_instances<kAny, kRobust, kLast>(n, inst, shader, ws, bytes, stream);
        return 0;
    }
    if (mode == 2) {
        MotionInstance<T>* m = static_cast<MotionInstance<T>*>(scratch);
        if (inst.count) to_motion_kernel<T><<<(unsigned)((inst.count + 255) / 256), 256, 0, stream>>>(inst.records, inst.count, m);
        top.template trace_instances<kAny, kRobust, kLast>(n, MotionInstances<T> { m, inst.count, inst.max_depth }, shader, ws, bytes, stream);
        return 0;
    }
    if (mode == 3) {
        DeviceView<T> bottom;
        if (!get_view<T>(bottom_h, bottom)) return -1;
        DeformingInstance<T> rec;
        cudaError_t e = cudaMemcpyAsync(&rec, inst.records, sizeof rec, cudaMemcpyDeviceToHost, stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) { g_error = cudaGetErrorString(e); return -1; }
        const MotionTriangles<T> keys { { rec.vertices[0], rec.vertices[1] }, bottom.prim_count };
        if (!rec.vertices[0]) {
            bottom.template trace_triangles<kAny, kRobust, kLast>(n, NoTime<T, kFilter> { shader }, ws, bytes, stream);
        } else if (!rec.motion_nodes) {
            bottom.template trace_triangles<kAny, kRobust, kLast>(n, keys, shader, ws, bytes, stream);
        } else {
            bottom.template trace_triangles<kAny, kRobust, kLast>(n, keys, cu::MotionNodes<T> { rec.motion_nodes, bottom.node_count }, shader,
                                                                  ws, bytes, stream);
        }
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
int run(typename Api<T>::Handle* h, typename Api<T>::Handle* bottom, DeformingInstance<T>* recs, size_t count, size_t max_depth, int mode,
        int filter, unsigned flags, const void* rays, const T* times, size_t n, Outputs<T> out, void* scratch, void* ws, size_t bytes,
        void* stream) {
    DeviceView<T> top;
    if (!get_view<T>(h, top)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : top.stream);
    const DeformingInstances<T> inst { recs, count, max_depth };
    return guarded([&] {
        return by_flags(flags, [&]<bool kAny, bool kRobust, bool kLast>() {
            if (filter == 0) return run_filter<T, kAny, kRobust, kLast, 0>(top, bottom, inst, mode, n, rays, times, out, scratch, ws, bytes, s);
            return run_filter<T, kAny, kRobust, kLast, 1>(top, bottom, inst, mode, n, rays, times, out, scratch, ws, bytes, s);
        });
    });
}

template <typename T>
int make_records(typename Api<T>::Handle* const* meshes, const uint32_t* mesh_of, const int* kinds, const T* keys0, const T* keys1,
                 const T* const* vkeys0, const T* const* vkeys1, const void* const* mnodes, size_t count, DeformingInstance<T>* d_records,
                 size_t* max_depth, void* stream) {
    return guarded([&] {
        std::vector<DeformingInstance<T>> recs(count);
        size_t depth = 0;
        for (size_t k = 0; k < count; ++k) {
            DeviceView<T> view;
            if (!get_view<T>(meshes[mesh_of[k]], view)) return -1;
            const uint32_t m = mesh_of[k];
            const MotionTriangles<T> keys { { vkeys0 ? vkeys0[m] : nullptr, vkeys1 ? vkeys1[m] : nullptr }, view.prim_count };
            const cu::MotionNodes<T> mn { mnodes ? static_cast<const cu::MotionNode<T>*>(mnodes[m]) : nullptr, view.node_count };
            if (kinds[k] == 0) recs[k] = cu::make_deforming_instance(view, keys0 + 12 * k, keys1 + 12 * k);
            else if (kinds[k] == 1) recs[k] = cu::make_deforming_instance(view, keys0 + 12 * k, keys1 + 12 * k, keys);
            else recs[k] = cu::make_deforming_instance(view, keys0 + 12 * k, keys1 + 12 * k, keys, mn);
            depth = view.depth > depth ? view.depth : depth;
        }
        *max_depth = depth;
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        cudaError_t e = cudaMemcpyAsync(d_records, recs.data(), count * sizeof(DeformingInstance<T>), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) { g_error = cudaGetErrorString(e); return -1; }
        return 0;
    });
}

template <typename T> __global__ void set_keys_kernel(DeformingInstance<T>* records, const T* keys0, const T* keys1, size_t count) {
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= 12 * count) return;
    records[i / 12].object_to_world[0][i % 12] = keys0[i];
    records[i / 12].object_to_world[1][i % 12] = keys1[i];
}

// Scripted paths: path i at times[i] runs the segments offsets[i] .. offsets[i + 1] of seg_rays
template <typename T, int kFilter> struct PathShader {
    using Ray = typename DeviceView<T>::Ray;
    using Hit = typename DeviceView<T>::Hit;
    struct Payload { uint32_t seg, calls; uint64_t hash; };
    const Ray* seg_rays;
    const uint8_t* seg_any;
    const uint64_t* offsets;
    const T* times;
    Outputs<T> out;                     // per segment (counts: per path)
    uint32_t* ray_ok;

    __device__ PathStep segment(size_t i, uint32_t j, Ray& ray) const {
        const size_t s = offsets[i] + j;
        if (s >= offsets[i + 1]) return PathStep::End;
        ray = seg_rays[s];
        return seg_any[s] ? PathStep::Occlusion : PathStep::Closest;
    }
    __device__ PathStep start(size_t i, Payload& p, Ray& ray, T& time) const {
        p.seg = 0; p.calls = 0; p.hash = kHashSeed;
        time = times[i];
        return segment(i, 0, ray);
    }
    __device__ bool accept(Payload& p, uint32_t inst, size_t id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(mix(p.hash, inst), id), bits(t)), bits(u)), bits(v));
        return keep<kFilter>(inst);
    }
    __device__ PathStep next(size_t i, Payload& p, const Hit& hit, uint32_t inst, Ray& ray) const {
        const size_t s = offsets[i] + p.seg;
        const unsigned char* a = reinterpret_cast<const unsigned char*>(&seg_rays[s]);
        const unsigned char* b = reinterpret_cast<const unsigned char*>(&ray);
        uint32_t same = 1;
        for (size_t k = 0; k < sizeof ray; ++k) same &= a[k] == b[k];
        ray_ok[s] = same;
        Outputs<T> o = out;
        o.counts = nullptr;
        write(o, s, (uint32_t)hit.prim_id, hit.t, hit.u, hit.v, inst, p.calls, p.hash);
        ++p.seg; p.calls = 0; p.hash = kHashSeed;
        return segment(i, p.seg, ray);
    }
    __device__ void finish(size_t i, const Payload&) const { if (out.counts) atomicAdd(out.counts + i, 1u); }
};

template <typename T>
int paths(typename Api<T>::Handle* h, DeformingInstance<T>* recs, size_t count, size_t max_depth, int filter, unsigned flags, size_t n,
          const void* seg_rays, const uint8_t* seg_any, const uint64_t* offsets, const T* times, Outputs<T> out, uint32_t* ray_ok, void* ws,
          size_t bytes, void* stream) {
    DeviceView<T> top;
    if (!get_view<T>(h, top)) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(stream ? stream : top.stream);
    const DeformingInstances<T> inst { recs, count, max_depth };
    using Ray = typename DeviceView<T>::Ray;
    return guarded([&] {
        return by_flags(flags & ~(unsigned)BVH_ANY_HIT, [&]<bool, bool kRobust, bool kLast>() {
            if (filter == 0)
                top.template trace_instance_paths<kRobust, kLast>(
                    n, inst, PathShader<T, 0> { static_cast<const Ray*>(seg_rays), seg_any, offsets, times, out, ray_ok }, ws, bytes, s);
            else
                top.template trace_instance_paths<kRobust, kLast>(
                    n, inst, PathShader<T, 1> { static_cast<const Ray*>(seg_rays), seg_any, offsets, times, out, ray_ok }, ws, bytes, s);
            return 0;
        });
    });
}

// A plain shader for timing: rays and times in, 16-byte records and the instance out
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

// The two-launch workaround the deforming forms replace, for timing: after a motion trace_instances over the static
// copies has written hits / inst, each deforming copy runs the motion-node trace_triangles of its mesh with the ray
// moved into its object space at the ray's time (instance_at) and tmax the best hit so far, and a closer hit replaces
// the record (the closest-hit merge, in finish).
struct MergeShader {
    struct Payload {};
    const bvh_ray3f* rays;
    const float* times;
    const DeformingInstance<float>* rec;
    uint32_t inst_id;
    bvh_hit3f* hits;
    uint32_t* inst;
    __device__ bvh_ray3f start(size_t i, Payload&, float& time) const {
        time = times[i];
        const Instance<float> at = cu::instance_at(*rec, time);
        bvh_ray3f r = rays[i];
        if (cu::detail::instance_is_singular(at.world_to_object)) { r.tmin = r.tmax = NAN; return r; }
        bvhb200::RayCtx<float> w, o;
        cu::detail::load_ray<float>(r, w);
        cu::detail::object_ray(at.world_to_object, w, o);
        r = cu::detail::make_ray<bvh_ray3f>(o);
        const float best = hits[i].t;
        r.tmax = best < r.tmax ? best : r.tmax;
        return r;
    }
    __device__ bool accept(Payload&, size_t, float, float, float) const { return true; }
    __device__ void finish(size_t i, const Payload&, const bvh_hit3f& hit) const {
        if (hit.prim_id != kNone) { hits[i] = hit; inst[i] = inst_id; }
    }
};

} // namespace

#define DDI_EXPORT extern "C" __attribute__((visibility("default")))
#define DDI_ENTRY(T, S)                                                                                                   \
    DDI_EXPORT int ddi_records##S(bvh##S* const* meshes, const uint32_t* mesh_of, const int* kinds, const T* keys0,       \
                                  const T* keys1, const void* vkeys0, const void* vkeys1, const void* mnodes, size_t count, \
                                  void* records, size_t* max_depth, void* stream) {                                      \
        return make_records<T>(meshes, mesh_of, kinds, keys0, keys1, static_cast<const T* const*>(vkeys0),               \
                               static_cast<const T* const*>(vkeys1), static_cast<const void* const*>(mnodes), count,     \
                               static_cast<DeformingInstance<T>*>(records), max_depth, stream);                           \
    }                                                                                                                    \
    DDI_EXPORT int ddi_set_keys##S(void* records, const T* keys0, const T* keys1, size_t count, void* stream) {          \
        if (count == 0) return 0;                                                                                        \
        set_keys_kernel<T><<<(unsigned)((12 * count + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(          \
            static_cast<DeformingInstance<T>*>(records), keys0, keys1, count);                                            \
        const cudaError_t e = cudaGetLastError();                                                                        \
        if (e != cudaSuccess) { g_error = cudaGetErrorString(e); return -1; }                                            \
        return 0;                                                                                                        \
    }                                                                                                                    \
    DDI_EXPORT int ddi_prepare##S(void* records, size_t count, size_t max_depth, void* bboxes, void* centers, void* stream) { \
        const DeformingInstances<T> inst { static_cast<DeformingInstance<T>*>(records), count, max_depth };               \
        return guarded([&] {                                                                                             \
            cu::prepare_deforming_instances(inst, static_cast<bvh_bbox##S*>(bboxes), static_cast<bvh_vec##S*>(centers), stream); \
            return 0;                                                                                                    \
        });                                                                                                              \
    }                                                                                                                    \
    DDI_EXPORT int ddi_bottom##S(bvh##S* h, const T* k0, const T* k1, size_t count, void* bboxes, void* centers,          \
                                 void* nodes, void* ws, size_t bytes, void* stream) {                                    \
        return guarded([&] {                                                                                             \
            const MotionTriangles<T> keys { { k0, k1 }, count };                                                         \
            if (bboxes) cu::prepare_motion_triangles(keys, static_cast<bvh_bbox##S*>(bboxes), static_cast<bvh_vec##S*>(centers), stream); \
            if (nodes) {                                                                                                 \
                DeviceView<T> view;                                                                                      \
                if (!get_view<T>(h, view)) return -1;                                                                    \
                cu::prepare_motion_nodes(view, keys, static_cast<cu::MotionNode<T>*>(nodes), ws, bytes, stream);         \
            }                                                                                                            \
            return 0;                                                                                                    \
        });                                                                                                              \
    }                                                                                                                    \
    DDI_EXPORT int ddi_run##S(bvh##S* top, bvh##S* bottom, void* records, size_t count, size_t max_depth, int mode,       \
                              int filter, unsigned flags, const void* rays, const T* times, size_t n, uint32_t* ids, T* t, \
                              T* u, T* v, uint32_t* inst, uint32_t* calls, uint64_t* hashes, uint32_t* counts, void* scratch, \
                              void* ws, size_t bytes, void* stream) {                                                    \
        return run<T>(top, bottom, static_cast<DeformingInstance<T>*>(records), count, max_depth, mode, filter, flags, rays, \
                      times, n, Outputs<T> { ids, t, u, v, inst, calls, hashes, counts }, scratch, ws, bytes, stream);    \
    }                                                                                                                    \
    DDI_EXPORT int ddi_paths##S(bvh##S* top, void* records, size_t count, size_t max_depth, int filter, unsigned flags,  \
                                size_t n, const void* seg_rays, const uint8_t* seg_any, const uint64_t* offsets,         \
                                const T* times, uint32_t* ids, T* t, T* u, T* v, uint32_t* inst, uint32_t* calls,         \
                                uint64_t* hashes, uint32_t* counts, uint32_t* ray_ok, void* ws, size_t bytes, void* stream) { \
        return paths<T>(top, static_cast<DeformingInstance<T>*>(records), count, max_depth, filter, flags, n, seg_rays,  \
                        seg_any, offsets, times, Outputs<T> { ids, t, u, v, inst, calls, hashes, counts }, ray_ok, ws,    \
                        bytes, stream);                                                                                  \
    }                                                                                                                    \
    DDI_EXPORT size_t ddi_record_bytes##S() { return sizeof(DeformingInstance<T>); }                                     \
    DDI_EXPORT size_t ddi_motion_record_bytes##S() { return sizeof(MotionInstance<T>); }                                 \
    DDI_EXPORT size_t ddi_motion_node_bytes##S() { return sizeof(cu::MotionNode<T>); }

DDI_ENTRY(float, 3f)
DDI_ENTRY(double, 3d)

DDI_EXPORT int ddi_plain3f(bvh3f* top, void* records, size_t count, size_t max_depth, const void* rays, const float* times, size_t n,
                           void* hits, uint32_t* inst, void* ws, size_t bytes, void* stream) {
    DeviceView<float> view;
    if (!get_view<float>(top, view)) return -1;
    const DeformingInstances<float> instances { static_cast<DeformingInstance<float>*>(records), count, max_depth };
    return guarded([&] {
        view.trace_instances<false, false>(n, instances, PlainShader { static_cast<const bvh_ray3f*>(rays), times,
                                                                       static_cast<bvh_hit3f*>(hits), inst },
                                           ws, bytes, stream ? stream : view.stream);
        return 0;
    });
}

// The workaround (see MergeShader): `static_records` (MotionInstance<float>, static copies only) under `top`, then for
// each record deforming_ids[k] (host ids) of `deforming` (device DeformingInstance<float>, the whole scene) one motion-node
// trace_triangles launch of `bottom`.
DDI_EXPORT int ddi_workaround3f(bvh3f* top, void* static_records, size_t count, size_t max_depth, bvh3f* bottom, const float* k0,
                                const float* k1, const void* motion_nodes, const void* deforming, const uint32_t* deforming_ids,
                                size_t deforming_count, const void* rays, const float* times, size_t n, void* hits, uint32_t* inst,
                                void* ws, size_t bytes, void* stream) {
    DeviceView<float> view, mesh;
    if (!get_view<float>(top, view) || !get_view<float>(bottom, mesh)) return -1;
    const MotionInstances<float> instances { static_cast<MotionInstance<float>*>(static_records), count, max_depth };
    const MotionTriangles<float> keys { { k0, k1 }, mesh.prim_count };
    const cu::MotionNodes<float> nodes { static_cast<const cu::MotionNode<float>*>(motion_nodes), mesh.node_count };
    return guarded([&] {
        const bvh_ray3f* r = static_cast<const bvh_ray3f*>(rays);
        view.trace_instances<false, false>(n, instances, PlainShader { r, times, static_cast<bvh_hit3f*>(hits), inst }, ws, bytes, stream);
        for (size_t k = 0; k < deforming_count; ++k)
            mesh.trace_triangles<false, false>(n, keys, nodes,
                                               MergeShader { r, times, static_cast<const DeformingInstance<float>*>(deforming) + deforming_ids[k],
                                                             deforming_ids[k], static_cast<bvh_hit3f*>(hits), inst },
                                               ws, bytes, stream);
        return 0;
    });
}

DDI_EXPORT const char* ddi_last_error() { return g_error.c_str(); }
