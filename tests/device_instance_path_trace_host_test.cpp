// tests/device_instance_path_trace_host_test.cpp — DeviceView::trace_instance_paths (include/bvh/v2/cuda/intersect.cuh)
// compiled as plain host C++, against the nested loop over the C++ surface (include/bvh/v2/b200_surface.h) that
// tests/device_instance_trace_host_test.cpp checks trace_instances with: Bvh<Node>::intersect on the top tree, whose leaf
// runs each instance's Bvh<Node>::intersect with a PrecomputedTri::intersect leaf on the object-space ray.
//
//   device_instance_path_trace_host_test <case file> f|d    input as tests/device_instance_trace_host_test.cpp reads it
//                                                            (written by tests/test_device_instance_path_trace_host.py).
// Scenes (placed with make_instance, prepared with prepare_instances, topped by a tree built here over the prepared
// boxes): identity, translate, scale (power of two), permute, pair (two copies at one place) and many (20 copies of every
// mesh: identity, translations, scales, permutations, rotations and two singular matrices).  A recording shader runs
// scripted paths: path i has length(i) segments (0 to 64; path 0 has none, path 1 has 64), segment j traces ray
// hash(i, j) of the case as a Closest or an Occlusion segment by another bit of the hash.  For both robust settings, both
// tie rules and three filters (accept all, reject odd ids, reject odd instances) it compares per segment the accept-call
// count, a hash of the accept sequence (instance, original id, bits of t, u, v), the record and its instance with the
// nested loop run as Bvh::intersect<IsAnyHit = Occlusion, IsRobust>, checks that next receives the scripted world ray
// bit for bit, and that start and finish are called once per path, in index order.  Under the identity scene the
// results equal trace_paths on mesh 0.
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
using cu::PathStep;

uint64_t mix(uint64_t h, uint64_t x) { return (h ^ x) * 1099511628211ull; }
constexpr uint64_t kSeed = 1469598103934665603ull;
constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr size_t kPaths = 160;

template <typename T> uint64_t bits(T x) {
    if constexpr (sizeof(T) == 4) { uint32_t b; std::memcpy(&b, &x, 4); return b; }
    else { uint64_t b; std::memcpy(&b, &x, 8); return b; }
}
uint32_t hash32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
size_t path_length(size_t i) { return i == 0 ? 0 : i == 1 ? 64 : hash32((uint32_t)i) % 65; }
uint32_t segment_hash(size_t i, size_t j) { return hash32((uint32_t)(i * 977 + j) ^ 0x5bd1e995u); }

enum Filter : int { kAll = 0, kEvenIds, kEvenInstances, kFilters };
bool keep(int filter, uint32_t inst, size_t id) {
    if (filter == kEvenIds) return (id & 1) == 0;
    if (filter == kEvenInstances) return (inst & 1) == 0;
    return true;
}
template <typename T> constexpr uint64_t kMissId = sizeof(T) == 4 ? 0xFFFFFFFFull : ~0ull;

struct Seg { uint64_t id, t, u, v; uint32_t inst, calls; uint64_t hash; uint32_t ray_ok; };
struct PathOut { uint32_t starts, finishes, segments, finish_order; };

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

// A top tree over instance boxes: median splits on the widest axis of the centres, leaves of up to 3 instances
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

template <typename T> struct Placement { size_t mesh; T m[12]; };
template <typename T> Placement<T> linear_about(size_t mesh, const T (&a)[9], const T c[3], const T (&shift)[3]) {
    Placement<T> p { mesh, {} };                        // x -> A (x - c) + c + shift
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

// The recording shader of trace_instance_paths
template <typename T> struct Recorder {
    using View = cu::DeviceView<T>;
    using Ray = typename View::Ray;
    using Hit = typename View::Hit;
    struct Payload { size_t seg; uint32_t calls; uint64_t hash; };
    const T* rays;
    size_t ray_count;
    int filter;
    const size_t* offsets;
    Seg* segs;
    PathOut* paths;
    std::vector<size_t>* order;        // the index sequence of start calls
    uint32_t* finished;

    PathStep segment(size_t i, size_t j, Ray& ray) const {
        const uint32_t h = segment_hash(i, j);
        const T* r = rays + 8 * (h % ray_count);
        ray.org.x = r[0]; ray.org.y = r[1]; ray.org.z = r[2];
        ray.dir.x = r[3]; ray.dir.y = r[4]; ray.dir.z = r[5];
        ray.tmin = r[6]; ray.tmax = r[7];
        return (h >> 31) ? PathStep::Occlusion : PathStep::Closest;
    }
    PathStep start(size_t i, Payload& p, Ray& ray) const {
        paths[i].starts += 1;
        order->push_back(i);
        p.seg = 0; p.calls = 0; p.hash = kSeed;
        return path_length(i) ? segment(i, 0, ray) : PathStep::End;
    }
    bool accept(Payload& p, uint32_t inst, size_t id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(mix(p.hash, inst), id), bits(t)), bits(u)), bits(v));
        return keep(filter, inst, id);
    }
    PathStep next(size_t i, Payload& p, const Hit& hit, uint32_t inst, Ray& ray) const {
        Ray want;
        segment(i, p.seg, want);
        Seg& s = segs[offsets[i] + p.seg];
        s.ray_ok = std::memcmp(&want, &ray, sizeof ray) == 0;
        s.id = hit.prim_id; s.t = bits(hit.t); s.u = bits(hit.u); s.v = bits(hit.v);
        s.inst = inst; s.calls = p.calls; s.hash = p.hash;
        ++p.seg; p.calls = 0; p.hash = kSeed;
        return p.seg < path_length(i) ? segment(i, p.seg, ray) : PathStep::End;
    }
    void finish(size_t i, const Payload& p) const {
        paths[i].finishes += 1;
        paths[i].segments = (uint32_t)p.seg;
        paths[i].finish_order = (*finished)++;
    }
};
// The same through trace_paths on one mesh (instance 0 in the hash, and for every hit)
template <typename T> struct MeshRecorder {
    Recorder<T> s;
    using Payload = typename Recorder<T>::Payload;
    using Ray = typename Recorder<T>::Ray;
    using Hit = typename Recorder<T>::Hit;
    PathStep start(size_t i, Payload& p, Ray& ray) const { return s.start(i, p, ray); }
    bool accept(Payload& p, size_t id, T t, T u, T v) const { return s.accept(p, 0, id, t, u, v); }
    PathStep next(size_t i, Payload& p, const Hit& hit, Ray& ray) const {
        return s.next(i, p, hit, hit.prim_id == (decltype(hit.prim_id))~0ull ? kNone : 0, ray);
    }
    void finish(size_t i, const Payload& p) const { s.finish(i, p); }
};

template <typename F> void by_mode(int mode, F&& f) {      // bit 0 robust, bit 1 last visited
    switch (mode) {
    case 0: f(std::integral_constant<bool, false>(), std::integral_constant<bool, false>()); break;
    case 1: f(std::integral_constant<bool, true>(), std::integral_constant<bool, false>()); break;
    case 2: f(std::integral_constant<bool, false>(), std::integral_constant<bool, true>()); break;
    default: f(std::integral_constant<bool, true>(), std::integral_constant<bool, true>()); break;
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

    std::vector<size_t> offsets(kPaths + 1, 0);
    for (size_t i = 0; i < kPaths; ++i) offsets[i + 1] = offsets[i] + path_length(i);
    const size_t seg_count = offsets[kPaths];

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
        const bvh::v2::Bvh<Node> top_bvh = build_top<T>(boxes, centres);
        std::vector<bvhb200::DevNode<T>> top_nodes;
        std::vector<uint32_t> top_ids;
        cu::DeviceView<T> top;
        device_layout<T>(top_bvh, top_nodes, top_ids, top);

        for (int filter = 0; filter < kFilters; ++filter) {
            for (int mode = 0; mode < 4; ++mode) {
                const bool robust = mode & 1, last = mode & 2;
                std::vector<Seg> segs(seg_count + 1);
                std::vector<PathOut> paths(kPaths);
                std::memset(segs.data(), 0, segs.size() * sizeof(segs[0]));
                std::memset(paths.data(), 0, paths.size() * sizeof(paths[0]));
                std::vector<size_t> order;
                uint32_t finished = 0;
                const Recorder<T> shader { rays.data(), ray_count, filter, offsets.data(), segs.data(), paths.data(), &order, &finished };
                by_mode(mode, [&](auto rob, auto lst) {
                    top.template trace_instance_paths<decltype(rob)::value, decltype(lst)::value>(kPaths, inst, shader, &cursor, sizeof cursor);
                });
                int bad = 0, path_bad = 0, hits = 0, occlusion = 0, nan = 0;
                uint64_t calls = 0;
                for (size_t i = 0; i < kPaths; ++i) {
                    const PathOut& po = paths[i];
                    if (po.starts != 1 || po.finishes != 1 || po.segments != path_length(i) || po.finish_order != i || order[i] != i) {
                        if (path_bad < 3) std::printf("  %s path %zu: starts %u finishes %u segments %u/%zu\n", scene.name, i, po.starts,
                                                      po.finishes, po.segments, path_length(i));
                        ++path_bad;
                    }
                    for (size_t j = 0; j < path_length(i); ++j) {
                        const uint32_t h = segment_hash(i, j);
                        const bool any = h >> 31;
                        const T* r = &rays[8 * (h % ray_count)];
                        bvh::v2::Ray<T, 3> wray(Vec3(r[0], r[1], r[2]), Vec3(r[3], r[4], r[5]), r[6], r[7]);
                        uint32_t best_inst = kNone, best_id = kNone;
                        T bt = r[7], bu = T(0), bv = T(0);
                        uint32_t want_calls = 0;
                        uint64_t want_hash = kSeed;
                        auto top_leaf = [&](size_t b, size_t e, auto any_c, auto robust_c) {
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
                                mesh.bvh.template intersect<decltype(any_c)::value, decltype(robust_c)::value>(
                                    oray, mesh.bvh.get_root().index, stack, [&](size_t lb, size_t le) {
                                        for (size_t q = lb; q < le; ++q) {
                                            const auto hq = mesh.tris[q].intersect(oray);
                                            if (!hq) continue;
                                            const auto [t, u, v] = *hq;
                                            const uint32_t id = (uint32_t)mesh.bvh.prim_ids[q];
                                            if (!last && best_inst != kNone && !(t < oray.tmax) &&
                                                !(id_inst < best_inst || (id_inst == best_inst && id < best_id)))
                                                continue;              // canonical: an exact tie only from a lower (instance, id)
                                            ++want_calls;
                                            want_hash = mix(mix(mix(mix(mix(want_hash, id_inst), id), bits(t)), bits(u)), bits(v));
                                            if (!keep(filter, id_inst, id)) continue;
                                            oray.tmax = t; best_inst = id_inst; best_id = id; bt = t; bu = u; bv = v;
                                        }
                                        return best_inst != kNone;
                                    });
                                wray.tmax = oray.tmax;
                                if (decltype(any_c)::value && best_inst != kNone) return true;
                            }
                            return best_inst != kNone;
                        };
                        bvh::v2::GrowingStack<typename Node::Index> stack;
                        auto nest = [&](auto any_c, auto robust_c) {
                            top_bvh.template intersect<decltype(any_c)::value, decltype(robust_c)::value>(
                                wray, top_bvh.get_root().index, stack, [&](size_t b, size_t e) { return top_leaf(b, e, any_c, robust_c); });
                        };
                        switch ((any ? 1 : 0) | (robust ? 2 : 0)) {
                        case 0: nest(std::false_type(), std::false_type()); break;
                        case 1: nest(std::true_type(), std::false_type()); break;
                        case 2: nest(std::false_type(), std::true_type()); break;
                        default: nest(std::true_type(), std::true_type()); break;
                        }
                        const uint64_t want_id = best_inst == kNone ? kMissId<T> : best_id;
                        const Seg& g = segs[offsets[i] + j];
                        calls += g.calls;
                        hits += g.id != kMissId<T>;
                        occlusion += any;
                        nan += r[6] != r[6] || r[7] != r[7];
                        if (g.id != want_id || g.t != bits(bt) || g.u != bits(bu) || g.v != bits(bv) || g.inst != best_inst ||
                            g.calls != want_calls || g.hash != want_hash || !g.ray_ok) {
                            if (bad < 3) std::printf("  %s path %zu segment %zu: calls %u/%u id %llu/%llu inst %u/%u ray %s\n", scene.name, i, j,
                                                     g.calls, want_calls, (unsigned long long)g.id, (unsigned long long)want_id, g.inst,
                                                     best_inst, g.ray_ok ? "ok" : "CHANGED");
                            ++bad;
                        }
                    }
                }
                // with the identity, trace_paths on mesh 0 gives the same calls and records
                int mesh_bad = 0;
                if (std::string(scene.name) == "identity" && filter != kEvenInstances) {
                    std::vector<Seg> msegs(seg_count + 1);
                    std::vector<PathOut> mpaths(kPaths);
                    std::memset(msegs.data(), 0, msegs.size() * sizeof(msegs[0]));
                    std::memset(mpaths.data(), 0, mpaths.size() * sizeof(mpaths[0]));
                    std::vector<size_t> morder;
                    uint32_t mfinished = 0;
                    const MeshRecorder<T> ms { { rays.data(), ray_count, filter, offsets.data(), msegs.data(), mpaths.data(), &morder, &mfinished } };
                    by_mode(mode, [&](auto rob, auto lst) {
                        meshes[0].view.template trace_paths<decltype(rob)::value, decltype(lst)::value>(kPaths, ms, &cursor, sizeof cursor);
                    });
                    for (size_t k = 0; k < seg_count; ++k) mesh_bad += std::memcmp(&msegs[k], &segs[k], sizeof(Seg)) != 0;
                    for (size_t k = 0; k < kPaths; ++k) mesh_bad += std::memcmp(&mpaths[k], &paths[k], sizeof(PathOut)) != 0;
                }
                std::printf("scene %s filter %d mode %d segments %zu occlusion %d nan %d mismatches %d path mismatches %d mesh mismatches %d "
                            "hits %d accept calls %llu\n", scene.name, filter, mode, seg_count, occlusion, nan, bad, path_bad, mesh_bad, hits,
                            (unsigned long long)calls);
                failures += bad + path_bad + mesh_bad;
            }
        }

        if (std::string(scene.name) == "many") {
            // n = 0 calls nothing; a record count other than the top tree's, a small workspace or a stack beyond 200 KB throw
            std::vector<Seg> segs(seg_count + 1);
            std::vector<PathOut> paths(kPaths);
            std::vector<size_t> order;
            uint32_t finished = 0;
            const Recorder<T> shader { rays.data(), ray_count, 0, offsets.data(), segs.data(), paths.data(), &order, &finished };
            top.template trace_instance_paths<false>(0, inst, shader, &cursor, sizeof cursor);
            const bool empty_ok = order.empty() && finished == 0;
            bool count_threw = false, ws_threw = false, deep_threw = false;
            cu::Instances<T> fewer = inst;
            fewer.count -= 1;
            try { top.template trace_instance_paths<false>(1, fewer, shader, &cursor, sizeof cursor); } catch (const std::invalid_argument&) { count_threw = true; }
            try { top.template trace_instance_paths<false>(1, inst, shader, &cursor, sizeof cursor - 1); } catch (const std::length_error&) { ws_threw = true; }
            cu::Instances<T> deep = inst;
            deep.max_depth = 400;
            try { top.template trace_instance_paths<false>(1, deep, shader, &cursor, sizeof cursor); } catch (const std::length_error&) { deep_threw = true; }
            std::printf("empty batch %s, record count %s, small workspace %s, deep stack %s\n", empty_ok ? "ok" : "CALLED",
                        count_threw ? "throws" : "DID NOT THROW", ws_threw ? "throws" : "DID NOT THROW", deep_threw ? "throws" : "DID NOT THROW");
            if (!empty_ok || !count_threw || !ws_threw || !deep_threw || !order.empty()) ++failures;
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
