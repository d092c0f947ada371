// tests/device_instance_trace_host_test.cpp — DeviceView::trace_instances and prepare_instances
// (include/bvh/v2/cuda/intersect.cuh) compiled as plain host C++, against a nested loop over the C++ surface
// (include/bvh/v2/b200_surface.h): Bvh<Node>::intersect on the top tree, whose leaf runs each instance's
// Bvh<Node>::intersect with a PrecomputedTri::intersect leaf on the object-space ray.
//
//   device_instance_trace_host_test <case file> f|d    input: u64 mesh count; per mesh u64 node_count, prim_count, the
//                                                       reference nodes (bounds[6], index), u64 prim_ids and the
//                                                       triangles (9 values each, original order); then u64 ray_count
//                                                       and the rays (org, dir, tmin, tmax), written by
//                                                       tests/test_device_instance_trace_host.py.
// Scenes, each placed with make_instance, prepared with prepare_instances and topped by a tree built here over the
// prepared boxes (median splits, up to 3 instances per leaf):
//   identity   mesh 0 unmoved: also equal to trace_triangles on mesh 0, bit for bit
//   translate  mesh 0 moved;   scale: mesh 0 scaled by 2 about its centre;   permute: its axes permuted
//   pair       two identical copies of mesh 0 at the same place: every hit ties, the canonical rule takes instance 0
//   many       20 copies of every mesh: identity, translations, power-of-two scales, axis permutations, general rotations
//              and two singular matrices (which get empty boxes and no hits)
// For the four IsAnyHit x IsRobust combinations, both tie rules and three filters (accept all, reject odd ids, reject odd
// instances) it compares per ray the accept-call count, a hash of the accept sequence (instance, original id and the
// bits of t, u, v), the record (id, bits of t, u, v) and its instance, and checks one start and one finish per ray.
#include <bvh/v2/bvh.h>
#include <bvh/v2/cuda/intersect.cuh>
#include <bvh/v2/stack.h>
#include <bvh/v2/tri.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <numeric>
#include <stdexcept>
#include <string>
#include <vector>

namespace {

namespace cu = bvh::v2::cuda;

uint64_t mix(uint64_t h, uint64_t x) { return (h ^ x) * 1099511628211ull; }
constexpr uint64_t kSeed = 1469598103934665603ull;
constexpr uint32_t kNone = 0xFFFFFFFFu;

template <typename T> uint64_t bits(T x) {
    if constexpr (sizeof(T) == 4) { uint32_t b; std::memcpy(&b, &x, 4); return b; }
    else { uint64_t b; std::memcpy(&b, &x, 8); return b; }
}

enum Filter : int { kAll = 0, kEvenIds, kEvenInstances, kFilters };
bool keep(int filter, uint32_t inst, size_t id) {
    if (filter == kEvenIds) return (id & 1) == 0;
    if (filter == kEvenInstances) return (inst & 1) == 0;
    return true;
}

template <typename T> constexpr uint64_t kMissId = sizeof(T) == 4 ? 0xFFFFFFFFull : ~0ull;

struct Out { uint64_t id, t, u, v; uint32_t inst, calls, starts, finishes; uint64_t hash; };

// One mesh: the reference tree, its triangles, and the device layout a DeviceView points at.
template <typename T> struct Mesh {
    using Node = bvh::v2::Node<T, 3>;
    bvh::v2::Bvh<Node> bvh;
    std::vector<bvh::v2::PrecomputedTri<T>> tris;       // BVH order
    std::vector<bvhb200::DevNode<T>> dev_nodes;
    std::vector<uint32_t> ids32;
    std::vector<bvhb200::DevTri<T>> dev_tris;
    std::vector<T> verts;                               // original order
    cu::DeviceView<T> view;
};

template <typename T> size_t tree_depth(const bvh::v2::Bvh<bvh::v2::Node<T, 3>>& bvh) {
    size_t depth = 0;
    std::vector<std::pair<size_t, size_t>> todo { { 0, 0 } };
    while (!todo.empty()) {
        auto [i, d] = todo.back(); todo.pop_back();
        if (bvh.nodes[i].is_leaf()) continue;
        depth = d > depth ? d : depth;
        todo.push_back({ bvh.nodes[i].index.first_id(), d + 1 });
        todo.push_back({ bvh.nodes[i].index.first_id() + 1, d + 1 });
    }
    return depth;
}

// The device layout of a reference tree, as bvhNN_get_device_view reports it.
template <typename T> void device_layout(const bvh::v2::Bvh<bvh::v2::Node<T, 3>>& bvh, std::vector<bvhb200::DevNode<T>>& nodes,
                                         std::vector<uint32_t>& ids32, cu::DeviceView<T>& view) {
    nodes.assign(bvh.nodes.size() + 1, bvhb200::DevNode<T> {});
    for (size_t i = 0; i < bvh.nodes.size(); ++i) {
        for (int k = 0; k < 6; ++k) nodes[i + 1].bounds[k] = bvh.nodes[i].bounds[k];
        nodes[i + 1].index = bvh.nodes[i].index.value;
    }
    ids32.assign(bvh.prim_ids.begin(), bvh.prim_ids.end());
    view = cu::DeviceView<T> {};
    view.nodes = nodes.data(); view.prim_ids = ids32.data();
    view.node_count = bvh.nodes.size(); view.prim_count = bvh.prim_ids.size(); view.depth = tree_depth<T>(bvh);
}

// A top tree over instance boxes: median splits on the widest axis of the centres, leaves of up to 3 instances.  Empty
// boxes do not widen their parents.
template <typename T> bvh::v2::Bvh<bvh::v2::Node<T, 3>> build_top(const std::vector<typename cu::detail::ViewTypes<T>::BBox>& boxes,
                                                                   const std::vector<typename cu::detail::ViewTypes<T>::Vec>& centres) {
    using Node = bvh::v2::Node<T, 3>;
    bvh::v2::Bvh<Node> bvh;
    const size_t n = boxes.size();
    bvh.prim_ids.resize(n);
    std::iota(bvh.prim_ids.begin(), bvh.prim_ids.end(), size_t(0));
    auto box_of = [&](size_t b, size_t e, Node& node) {
        const T inf = std::numeric_limits<T>::infinity();
        for (int a = 0; a < 3; ++a) { node.bounds[2 * a] = inf; node.bounds[2 * a + 1] = -inf; }
        for (size_t k = b; k < e; ++k) {
            const auto& x = boxes[bvh.prim_ids[k]];
            const T lo[3] = { x.min.x, x.min.y, x.min.z }, hi[3] = { x.max.x, x.max.y, x.max.z };
            for (int a = 0; a < 3; ++a) {
                node.bounds[2 * a] = std::min(node.bounds[2 * a], lo[a]);
                node.bounds[2 * a + 1] = std::max(node.bounds[2 * a + 1], hi[a]);
            }
        }
    };
    auto c = [&](size_t id, int a) { return a == 0 ? centres[id].x : a == 1 ? centres[id].y : centres[id].z; };
    bvh.nodes.resize(1);
    struct Todo { size_t node, b, e; };
    std::vector<Todo> todo { { 0, 0, n } };
    while (!todo.empty()) {
        const Todo w = todo.back(); todo.pop_back();
        box_of(w.b, w.e, bvh.nodes[w.node]);
        if (w.e - w.b <= 3) { bvh.nodes[w.node].index = Node::Index::make_leaf(w.b, w.e - w.b); continue; }
        int axis = 0;
        T best = -1;
        for (int a = 0; a < 3; ++a) {
            T lo = c(bvh.prim_ids[w.b], a), hi = lo;
            for (size_t k = w.b; k < w.e; ++k) { lo = std::min(lo, c(bvh.prim_ids[k], a)); hi = std::max(hi, c(bvh.prim_ids[k], a)); }
            if (hi - lo > best) { best = hi - lo; axis = a; }
        }
        const size_t mid = (w.b + w.e) / 2;
        std::nth_element(bvh.prim_ids.begin() + w.b, bvh.prim_ids.begin() + mid, bvh.prim_ids.begin() + w.e,
                         [&](size_t x, size_t y) { return c(x, axis) < c(y, axis) || (c(x, axis) == c(y, axis) && x < y); });
        const size_t first = bvh.nodes.size();
        bvh.nodes.resize(first + 2);
        bvh.nodes[w.node].index = Node::Index::make_inner(first);
        todo.push_back({ first, w.b, mid });
        todo.push_back({ first + 1, mid, w.e });
    }
    return bvh;
}

// The matrices of the scenes: 3 x 4 row-major, about the centre `c` of the mesh.
template <typename T> struct Placement { size_t mesh; T m[12]; };
template <typename T> Placement<T> linear_about(size_t mesh, const T (&a)[9], const T c[3], const T (&shift)[3]) {
    // x -> A (x - c) + c + shift
    Placement<T> p { mesh, {} };
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) p.m[4 * i + j] = a[3 * i + j];
        T b = c[i] + shift[i];
        for (int j = 0; j < 3; ++j) b -= a[3 * i + j] * c[j];
        p.m[4 * i + 3] = b;
    }
    return p;
}
template <typename T> void rotation(T angle, T ax, T ay, T az, T (&r)[9]) {
    const T n = std::sqrt(ax * ax + ay * ay + az * az);
    ax /= n; ay /= n; az /= n;
    const T s = std::sin(angle), k = std::cos(angle), v = 1 - k;
    const T m[9] = { k + ax * ax * v, ax * ay * v - az * s, ax * az * v + ay * s,
                     ay * ax * v + az * s, k + ay * ay * v, ay * az * v - ax * s,
                     az * ax * v - ay * s, az * ay * v + ax * s, k + az * az * v };
    std::copy(m, m + 9, r);
}

template <typename T> struct RayPod;
template <> struct RayPod<float> { using Type = bvh_ray3f; };
template <> struct RayPod<double> { using Type = bvh_ray3d; };

// The recording shader of trace_instances
template <typename T> struct InstanceShader {
    using Ray = typename RayPod<T>::Type;
    struct Payload { uint32_t calls; uint64_t hash; };
    const T* rays;
    int filter;
    Out* out;
    size_t* order;
    size_t* started;
    Ray start(size_t i, Payload& p) const {
        const T* r = rays + 8 * i;
        Ray ray;
        ray.org.x = r[0]; ray.org.y = r[1]; ray.org.z = r[2]; ray.dir.x = r[3]; ray.dir.y = r[4]; ray.dir.z = r[5];
        ray.tmin = r[6]; ray.tmax = r[7];
        p.calls = 0; p.hash = kSeed;
        out[i].starts += 1;
        order[(*started)++] = i;
        return ray;
    }
    bool accept(Payload& p, uint32_t inst, size_t id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(mix(p.hash, inst), id), bits(t)), bits(u)), bits(v));
        return keep(filter, inst, id);
    }
    template <typename Hit> void finish(size_t i, const Payload& p, const Hit& hit, uint32_t inst) const {
        out[i].id = hit.prim_id; out[i].t = bits(hit.t); out[i].u = bits(hit.u); out[i].v = bits(hit.v);
        out[i].inst = inst; out[i].calls = p.calls; out[i].hash = p.hash; out[i].finishes += 1;
    }
};
// The same, through trace_triangles on one mesh (instance 0 in the hash)
template <typename T> struct TriangleShader {
    InstanceShader<T> s;
    using Payload = typename InstanceShader<T>::Payload;
    typename InstanceShader<T>::Ray start(size_t i, Payload& p) const { return s.start(i, p); }
    bool accept(Payload& p, size_t id, T t, T u, T v) const { return s.accept(p, 0, id, t, u, v); }
    template <typename Hit> void finish(size_t i, const Payload& p, const Hit& hit) const { s.finish(i, p, hit, hit.prim_id == (decltype(hit.prim_id))~0ull ? kNone : 0); }
};

template <typename T, bool Any, bool Robust, bool Last>
void trace(const cu::DeviceView<T>& top, size_t n, const cu::Instances<T>& inst, const InstanceShader<T>& shader, unsigned long long& cursor) {
    top.template trace_instances<Any, Robust, Last>(n, inst, shader, &cursor, sizeof cursor);
}
template <typename T, bool Any, bool Robust, bool Last>
void trace_tri(const cu::DeviceView<T>& view, size_t n, const TriangleShader<T>& shader, unsigned long long& cursor) {
    view.template trace_triangles<Any, Robust, Last>(n, shader, &cursor, sizeof cursor);
}
template <typename T, typename F> void by_mode(int mode, F&& f) {
    switch (mode) {
    case 0: f(std::integral_constant<bool, false>(), std::integral_constant<bool, false>(), std::integral_constant<bool, false>()); break;
    case 1: f(std::integral_constant<bool, true>(), std::integral_constant<bool, false>(), std::integral_constant<bool, false>()); break;
    case 2: f(std::integral_constant<bool, false>(), std::integral_constant<bool, true>(), std::integral_constant<bool, false>()); break;
    case 3: f(std::integral_constant<bool, true>(), std::integral_constant<bool, true>(), std::integral_constant<bool, false>()); break;
    case 4: f(std::integral_constant<bool, false>(), std::integral_constant<bool, false>(), std::integral_constant<bool, true>()); break;
    case 5: f(std::integral_constant<bool, true>(), std::integral_constant<bool, false>(), std::integral_constant<bool, true>()); break;
    case 6: f(std::integral_constant<bool, false>(), std::integral_constant<bool, true>(), std::integral_constant<bool, true>()); break;
    default: f(std::integral_constant<bool, true>(), std::integral_constant<bool, true>(), std::integral_constant<bool, true>()); break;
    }
}

template <typename T>
int run(std::ifstream& in) {
    using Node = bvh::v2::Node<T, 3>;
    using Vec3 = bvh::v2::Vec<T, 3>;
    using BBox = typename cu::detail::ViewTypes<T>::BBox;
    using VecC = typename cu::detail::ViewTypes<T>::Vec;
    uint64_t mesh_count = 0;
    in.read((char*)&mesh_count, 8);
    std::vector<Mesh<T>> meshes(mesh_count);
    for (auto& mesh : meshes) {
        uint64_t node_count, prim_count;
        in.read((char*)&node_count, 8); in.read((char*)&prim_count, 8);
        mesh.bvh.nodes.resize(node_count);
        in.read((char*)mesh.bvh.nodes.data(), node_count * sizeof(Node));
        std::vector<uint64_t> ids(prim_count);
        in.read((char*)ids.data(), prim_count * 8);
        mesh.bvh.prim_ids.assign(ids.begin(), ids.end());
        mesh.verts.resize(9 * prim_count);
        in.read((char*)mesh.verts.data(), mesh.verts.size() * sizeof(T));
        device_layout<T>(mesh.bvh, mesh.dev_nodes, mesh.ids32, mesh.view);
        mesh.dev_tris.resize(prim_count);
        mesh.tris.resize(prim_count);
        for (size_t k = 0; k < prim_count; ++k) {
            const T* v = &mesh.verts[9 * ids[k]];
            mesh.dev_tris[k] = bvhb200::precompute_tri(v);
            mesh.tris[k] = bvh::v2::PrecomputedTri<T>(Vec3(v[0], v[1], v[2]), Vec3(v[3], v[4], v[5]), Vec3(v[6], v[7], v[8]));
        }
        mesh.view.tris = mesh.dev_tris.data();
    }
    uint64_t ray_count = 0;
    in.read((char*)&ray_count, 8);
    std::vector<T> rays(8 * ray_count);
    in.read((char*)rays.data(), rays.size() * sizeof(T));
    if (!in) { std::puts("short input"); return 2; }

    // the scenes, about the centre of mesh 0's root box
    const auto& rb = meshes[0].bvh.nodes[0].bounds;
    const T c[3] = { (rb[0] + rb[1]) / 2, (rb[2] + rb[3]) / 2, (rb[4] + rb[5]) / 2 };
    const T size = std::max({ rb[1] - rb[0], rb[3] - rb[2], rb[5] - rb[4] });
    const T id9[9] = { 1, 0, 0, 0, 1, 0, 0, 0, 1 }, two9[9] = { 2, 0, 0, 0, 2, 0, 0, 0, 2 }, half9[9] = { 0.5, 0, 0, 0, 0.5, 0, 0, 0, 0.5 };
    const T perm9[9] = { 0, 0, 1, 1, 0, 0, 0, 1, 0 }, zero3[3] = { 0, 0, 0 };
    const T flat9[9] = { 1, 0, 0, 0, 0, 0, 0, 0, 1 };                               // singular: y collapses
    struct Scene { const char* name; std::vector<Placement<T>> place; };
    std::vector<Scene> scenes;
    const Placement<T> ident { 0, { 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0 } };
    scenes.push_back({ "identity", { ident } });
    const T shift[3] = { size / 4, -size / 8, size / 2 };
    scenes.push_back({ "translate", { linear_about<T>(0, id9, c, shift) } });
    scenes.push_back({ "scale", { linear_about<T>(0, two9, c, zero3) } });
    scenes.push_back({ "permute", { linear_about<T>(0, perm9, c, zero3) } });
    scenes.push_back({ "pair", { ident, ident } });
    {
        std::vector<Placement<T>> many;
        uint64_t s = 12345;
        auto rnd = [&] { s = s * 6364136223846793005ull + 1442695040888963407ull; return T((s >> 11) * (1.0 / 9007199254740992.0)); };
        for (size_t k = 0; k < 20; ++k) {
            const size_t mesh = k % meshes.size();
            const T sh[3] = { (rnd() - T(0.5)) * size, (rnd() - T(0.5)) * size, (rnd() - T(0.5)) * size / 2 };
            T a[9];
            switch (k % 7) {
            case 0: std::copy(id9, id9 + 9, a); break;
            case 1: std::copy(half9, half9 + 9, a); break;
            case 2: std::copy(perm9, perm9 + 9, a); break;
            case 6: std::copy(flat9, flat9 + 9, a); break;
            default: rotation<T>(rnd() * T(6.283185307179586), rnd() - T(0.5), rnd() - T(0.5), rnd() - T(0.5), a); break;
            }
            many.push_back(k == 0 ? ident : linear_about<T>(mesh, a, c, k % 7 == 0 ? zero3 : sh));
        }
        scenes.push_back({ "many", many });
    }

    unsigned long long cursor = 0;
    int failures = 0;
    for (const Scene& scene : scenes) {
        const size_t count = scene.place.size();
        std::vector<cu::Instance<T>> records(count);
        std::vector<size_t> mesh_of(count);
        size_t max_depth = 0;
        for (size_t k = 0; k < count; ++k) {
            records[k] = cu::make_instance(meshes[scene.place[k].mesh].view, scene.place[k].m);
            mesh_of[k] = scene.place[k].mesh;
            max_depth = std::max(max_depth, meshes[mesh_of[k]].view.depth);
        }
        const cu::Instances<T> inst { records.data(), count, max_depth };
        std::vector<BBox> boxes(count);
        std::vector<VecC> centres(count);
        cu::prepare_instances(inst, boxes.data(), centres.data());
        size_t singular = 0;
        for (size_t k = 0; k < count; ++k) {
            const bool empty = !(boxes[k].min.x <= boxes[k].max.x);
            singular += empty;
            if (empty != cu::detail::instance_is_singular(records[k].world_to_object)) ++failures;
        }
        const bvh::v2::Bvh<Node> top_bvh = build_top<T>(boxes, centres);
        std::vector<bvhb200::DevNode<T>> top_nodes;
        std::vector<uint32_t> top_ids;
        cu::DeviceView<T> top;
        device_layout<T>(top_bvh, top_nodes, top_ids, top);

        for (int filter = 0; filter < kFilters; ++filter) {
            for (int mode = 0; mode < 8; ++mode) {       // bit 0 any-hit, bit 1 robust, bit 2 last visited
                const bool last = mode & 4;
                std::vector<Out> got(ray_count);
                std::memset(got.data(), 0, got.size() * sizeof(got[0]));
                std::vector<size_t> order(ray_count + 1);
                size_t started = 0;
                const InstanceShader<T> shader { rays.data(), filter, got.data(), order.data(), &started };
                by_mode<T>(mode, [&](auto any, auto robust, auto lst) {
                    trace<T, decltype(any)::value, decltype(robust)::value, decltype(lst)::value>(top, ray_count, inst, shader, cursor);
                });
                int bad = 0, hits = 0, ties = 0, lower = 0;
                uint64_t calls = 0;
                for (size_t i = 0; i < ray_count; ++i) {
                    const T* r = &rays[8 * i];
                    bvh::v2::Ray<T, 3> wray(Vec3(r[0], r[1], r[2]), Vec3(r[3], r[4], r[5]), r[6], r[7]);
                    const T tmax_in = r[7];
                    uint32_t best_inst = kNone, best_id = kNone;
                    T bt = tmax_in, bu = T(0), bv = T(0);
                    uint32_t want_calls = 0;
                    uint64_t want_hash = kSeed;
                    bool tied = false;
                    auto top_leaf = [&](size_t b, size_t e, auto any, auto robust) {
                        for (size_t k = b; k < e; ++k) {
                            const uint32_t id_inst = (uint32_t)top_bvh.prim_ids[k];
                            const cu::Instance<T>& rec = records[id_inst];
                            if (cu::detail::instance_is_singular(rec.world_to_object)) continue;
                            const Mesh<T>& mesh = meshes[mesh_of[id_inst]];
                            bvhb200::RayCtx<T> w, o;
                            for (int a = 0; a < 3; ++a) { w.org[a] = wray.org[a]; w.dir[a] = wray.dir[a]; }
                            w.tmin = wray.tmin; w.tmax = wray.tmax;
                            cu::detail::object_ray(rec.world_to_object, w, o);
                            bvh::v2::Ray<T, 3> oray(Vec3(o.org[0], o.org[1], o.org[2]), Vec3(o.dir[0], o.dir[1], o.dir[2]), o.tmin, o.tmax);
                            bvh::v2::GrowingStack<typename Node::Index> stack;
                            mesh.bvh.template intersect<decltype(any)::value, decltype(robust)::value>(
                                oray, mesh.bvh.get_root().index, stack, [&](size_t lb, size_t le) {
                                    for (size_t q = lb; q < le; ++q) {
                                        const auto h = mesh.tris[q].intersect(oray);
                                        if (!h) continue;
                                        const auto [t, u, v] = *h;
                                        const uint32_t id = (uint32_t)mesh.bvh.prim_ids[q];
                                        if (best_inst != kNone && !(t < oray.tmax)) {
                                            // canonical: an exact tie is taken only from a lower (instance, id)
                                            tied = true;
                                            if (!last && !(id_inst < best_inst || (id_inst == best_inst && id < best_id))) continue;
                                        }
                                        ++want_calls;
                                        want_hash = mix(mix(mix(mix(mix(want_hash, id_inst), id), bits(t)), bits(u)), bits(v));
                                        if (!keep(filter, id_inst, id)) continue;
                                        oray.tmax = t; best_inst = id_inst; best_id = id; bt = t; bu = u; bv = v;
                                    }
                                    return best_inst != kNone;
                                });
                            wray.tmax = oray.tmax;
                            if (decltype(any)::value && best_inst != kNone) return true;
                        }
                        return best_inst != kNone;
                    };
                    bvh::v2::GrowingStack<typename Node::Index> stack;
                    by_mode<T>(mode & 3, [&](auto any, auto robust, auto) {
                        top_bvh.template intersect<decltype(any)::value, decltype(robust)::value>(
                            wray, top_bvh.get_root().index, stack, [&](size_t b, size_t e) { return top_leaf(b, e, any, robust); });
                    });
                    const uint64_t want_id = best_inst == kNone ? kMissId<T> : best_id;
                    const Out& g = got[i];
                    calls += g.calls;
                    hits += g.id != kMissId<T>;
                    ties += tied;
                    lower += tied && g.inst == 0;
                    if (g.id != want_id || g.t != bits(bt) || g.u != bits(bu) || g.v != bits(bv) || g.inst != best_inst ||
                        g.calls != want_calls || g.hash != want_hash || g.starts != 1 || g.finishes != 1 || order[i] != i) {
                        if (bad < 3) std::printf("  %s ray %zu: calls %u/%u id %llu/%llu inst %u/%u starts %u finishes %u\n", scene.name, i, g.calls,
                                                 want_calls, (unsigned long long)g.id, (unsigned long long)want_id, g.inst, best_inst, g.starts, g.finishes);
                        ++bad;
                    }
                }
                // with the identity, trace_triangles on mesh 0 gives the same calls and records
                int tri_bad = 0;
                if (std::string(scene.name) == "identity" && filter != kEvenInstances) {
                    std::vector<Out> tri(ray_count);
                    std::memset(tri.data(), 0, tri.size() * sizeof(tri[0]));
                    size_t tri_started = 0;
                    const TriangleShader<T> ts { { rays.data(), filter, tri.data(), order.data(), &tri_started } };
                    by_mode<T>(mode, [&](auto any, auto robust, auto lst) {
                        trace_tri<T, decltype(any)::value, decltype(robust)::value, decltype(lst)::value>(meshes[0].view, ray_count, ts, cursor);
                    });
                    for (size_t i = 0; i < ray_count; ++i)
                        if (std::memcmp(&tri[i], &got[i], sizeof(Out)) != 0) ++tri_bad;
                }
                std::printf("scene %s filter %d mode %d mismatches %d triangle mismatches %d singular %zu ties %d lower %d hits %d accept calls %llu\n",
                            scene.name, filter, mode, bad, tri_bad, singular, ties, lower, hits, (unsigned long long)calls);
                failures += bad + tri_bad;
            }
        }

        if (std::string(scene.name) == "many") {
            // n = 0 calls nothing; a record count other than the top tree's, a small workspace or a stack beyond 200 KB throw
            std::vector<Out> got(1);
            std::memset(got.data(), 0, sizeof(got[0]));
            size_t order[1], started = 0;
            const InstanceShader<T> shader { rays.data(), 0, got.data(), order, &started };
            top.template trace_instances<false, false>(0, inst, shader, &cursor, sizeof cursor);
            const bool empty_ok = started == 0 && got[0].finishes == 0;
            bool count_threw = false, ws_threw = false, deep_threw = false;
            cu::Instances<T> fewer = inst;
            fewer.count -= 1;
            try { top.template trace_instances<false, false>(1, fewer, shader, &cursor, sizeof cursor); } catch (const std::invalid_argument&) { count_threw = true; }
            try { top.template trace_instances<false, false>(1, inst, shader, &cursor, sizeof cursor - 1); } catch (const std::length_error&) { ws_threw = true; }
            cu::Instances<T> deep = inst;
            deep.max_depth = 400;
            try { top.template trace_instances<false, false>(1, deep, shader, &cursor, sizeof cursor); } catch (const std::length_error&) { deep_threw = true; }
            std::printf("empty batch %s, record count %s, small workspace %s, deep stack %s\n", empty_ok ? "ok" : "CALLED",
                        count_threw ? "throws" : "DID NOT THROW", ws_threw ? "throws" : "DID NOT THROW", deep_threw ? "throws" : "DID NOT THROW");
            if (!empty_ok || !count_threw || !ws_threw || !deep_threw || started != 0) ++failures;
        }
    }
    return failures;
}

} // namespace

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    std::ifstream in(argv[1], std::ios::binary);
    if (!in) return 2;
    const int failures = argv[2][0] == 'd' ? run<double>(in) : run<float>(in);
    std::printf("failures %d\n", failures);
    return failures ? 1 : 0;
}
