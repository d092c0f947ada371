// tests/device_motion_instance_host_test.cpp — the motion forms of DeviceView::trace_instances and trace_instance_paths,
// prepare_motion_instances and instance_at (include/bvh/v2/cuda/intersect.cuh) compiled as plain host C++, against the
// static calls over instance_at(records[k], time) on the same top tree.
//
//   device_motion_instance_host_test <case file> f|d    input as tests/device_instance_trace_host_test.cpp reads it
//                                                        (written by tests/test_device_motion_instance_host.py).
// Scenes (placed with make_motion_instance, prepared with prepare_motion_instances, topped by a tree built here over the
// prepared boxes), each a set of key pairs: equal (20 copies of every mesh at identity, scale, permutation, rotation and
// singular matrices, key1 = key0), translate, rotscale (rotation plus scale), singular_end (scale 0 at time 0),
// both_singular (two flattening keys) and non_finite (a NaN and an infinite key next to a moving copy).  Ray i has time
// time_of(i): 0, 1, 0.5, 0.3, a random time, -1, 2 and NaN.  Per scene it checks:
//   * instance_at at 0 and 1 gives the keys bit for bit and prepare_instance's inverse of them;
//   * every box contains every bottom vertex moved in long double by the rounded A(tau) of instance_at, at 65 tau; a
//     non-finite key gives the empty box;
//   * for any-hit and closest-hit, both robust settings, both tie rules and three filters (accept all, reject odd ids,
//     reject odd instances), per ray: the accept-call count, a hash of the accept sequence (instance, original id, bits
//     of t, u, v), the record and its instance equal a static trace_instances of that ray over instance_at(records[k],
//     time_i);
//   * for both robust settings, both tie rules and the three filters, scripted paths of 0 to 16 mixed segments at
//     time_of(i): per segment the same equality against the static trace_instances of the segment's world ray, and
//     next receives that ray bit for bit;
//   * n = 0 calls nothing; a wrong record count, a small workspace and a too-deep stack throw, naming the motion call.
#include <bvh/v2/bvh.h>
#include <bvh/v2/cuda/intersect.cuh>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <limits>
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
constexpr size_t kPaths = 96;

template <typename T> uint64_t bits(T x) {
    if constexpr (sizeof(T) == 4) { uint32_t b; std::memcpy(&b, &x, 4); return b; }
    else { uint64_t b; std::memcpy(&b, &x, 8); return b; }
}
uint32_t hash32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
template <typename T> T time_of(size_t i) {
    switch (i % 8) {
    case 0: return T(0);
    case 1: return T(1);
    case 2: return T(0.5);
    case 3: return T(0.3);
    case 4: return T(hash32((uint32_t)i) >> 8) * T(1.0 / 16777216);
    case 5: return T(-1);
    case 6: return T(2);
    default: return std::numeric_limits<T>::quiet_NaN();
    }
}
size_t path_length(size_t i) { return i == 0 ? 0 : i == 1 ? 16 : hash32((uint32_t)i) % 17; }
uint32_t segment_hash(size_t i, size_t j) { return hash32((uint32_t)(i * 977 + j) ^ 0x5bd1e995u); }

enum Filter : int { kAll = 0, kEvenIds, kEvenInstances, kFilters };
bool keep(int filter, uint32_t inst, size_t id) {
    if (filter == kEvenIds) return (id & 1) == 0;
    if (filter == kEvenInstances) return (inst & 1) == 0;
    return true;
}

struct Out { uint64_t id, t, u, v; uint32_t inst, calls; uint64_t hash; uint32_t ray_ok, pad; };

template <typename T> struct Mesh {
    using Node = bvh::v2::Node<T, 3>;
    bvh::v2::Bvh<Node> bvh;
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

// A top tree over record boxes: median splits on the widest axis of the centres, leaves of up to 3 records.  An empty
// box (a non-finite key) still takes a slot; its centre is 0.
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

template <typename T> struct Key { T m[12]; };
template <typename T> Key<T> linear_about(const T (&a)[9], const T c[3], const T (&shift)[3]) {
    Key<T> p {};                        // x -> A (x - c) + c + shift
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) p.m[4 * i + j] = a[3 * i + j];
        T b = c[i] + shift[i];
        for (int j = 0; j < 3; ++j) b -= a[3 * i + j] * c[j];
        p.m[4 * i + 3] = b;
    }
    return p;
}
template <typename T> void rotation(T angle, T ax, T ay, T az, T s, T (&r)[9]) {
    const T n = std::sqrt(ax * ax + ay * ay + az * az);
    ax /= n; ay /= n; az /= n;
    const T si = std::sin(angle), k = std::cos(angle), v = 1 - k;
    const T m[9] = { k + ax * ax * v, ax * ay * v - az * si, ax * az * v + ay * si,
                     ay * ax * v + az * si, k + ay * ay * v, ay * az * v - ax * si,
                     az * ax * v - ay * si, az * ay * v + ax * si, k + az * az * v };
    for (int q = 0; q < 9; ++q) r[q] = m[q] * s;
}
template <typename T> struct Placement { size_t mesh; Key<T> k0, k1; };

// The recording shader: the motion form (start with a time) and the static oracle (start without), same records
template <typename T> struct Recorder {
    using View = cu::DeviceView<T>;
    using Ray = typename View::Ray;
    using Hit = typename View::Hit;
    struct Payload { uint32_t calls; uint64_t hash; };
    const T* rays;
    int filter;
    Out* out;
    size_t first;                       // the static oracle: ray `first`, written to out[0]

    Ray ray(size_t i) const {
        const T* r = rays + 8 * i;
        Ray x;
        x.org.x = r[0]; x.org.y = r[1]; x.org.z = r[2];
        x.dir.x = r[3]; x.dir.y = r[4]; x.dir.z = r[5];
        x.tmin = r[6]; x.tmax = r[7];
        return x;
    }
    Ray start(size_t i, Payload& p, T& time) const { p.calls = 0; p.hash = kSeed; time = time_of<T>(i); return ray(i); }
    Ray start(size_t i, Payload& p) const { p.calls = 0; p.hash = kSeed; return ray(first + i); }
    bool accept(Payload& p, uint32_t inst, size_t id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(mix(p.hash, inst), id), bits(t)), bits(u)), bits(v));
        return keep(filter, inst, id);
    }
    void finish(size_t i, const Payload& p, const Hit& hit, uint32_t inst) const {
        Out& o = out[i];
        o.id = hit.prim_id; o.t = bits(hit.t); o.u = bits(hit.u); o.v = bits(hit.v);
        o.inst = inst; o.calls = p.calls; o.hash = p.hash; o.ray_ok = 1;
    }
};

// The path shader: scripted segments, path i at time_of(i); per segment its record in segs[offsets[i] + j]
template <typename T> struct PathRecorder {
    using Ray = typename cu::DeviceView<T>::Ray;
    using Hit = typename cu::DeviceView<T>::Hit;
    struct Payload { size_t seg; uint32_t calls; uint64_t hash; };
    const T* rays;
    size_t ray_count;
    int filter;
    const size_t* offsets;
    Out* segs;
    uint32_t* starts;
    uint32_t* finishes;

    PathStep segment(size_t i, size_t j, Ray& ray) const {
        const uint32_t h = segment_hash(i, j);
        const T* r = rays + 8 * (h % ray_count);
        ray.org.x = r[0]; ray.org.y = r[1]; ray.org.z = r[2];
        ray.dir.x = r[3]; ray.dir.y = r[4]; ray.dir.z = r[5];
        ray.tmin = r[6]; ray.tmax = r[7];
        return (h >> 31) ? PathStep::Occlusion : PathStep::Closest;
    }
    PathStep start(size_t i, Payload& p, Ray& ray, T& time) const {
        starts[i] += 1;
        p.seg = 0; p.calls = 0; p.hash = kSeed;
        time = time_of<T>(i);
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
        Out& s = segs[offsets[i] + p.seg];
        s.ray_ok = std::memcmp(&want, &ray, sizeof ray) == 0;
        s.id = hit.prim_id; s.t = bits(hit.t); s.u = bits(hit.u); s.v = bits(hit.v);
        s.inst = inst; s.calls = p.calls; s.hash = p.hash;
        ++p.seg; p.calls = 0; p.hash = kSeed;
        return p.seg < path_length(i) ? segment(i, p.seg, ray) : PathStep::End;
    }
    void finish(size_t i, const Payload& p) const { finishes[i] += 1 + (p.seg != path_length(i) ? 100 : 0); }
};

template <typename F> void by_mode(int mode, F&& f) {      // bit 0 any-hit, bit 1 robust, bit 2 last visited
    using B0 = std::false_type; using B1 = std::true_type;
    switch (mode) {
    case 0: f(B0(), B0(), B0()); break;
    case 1: f(B1(), B0(), B0()); break;
    case 2: f(B0(), B1(), B0()); break;
    case 3: f(B1(), B1(), B0()); break;
    case 4: f(B0(), B0(), B1()); break;
    case 5: f(B1(), B0(), B1()); break;
    case 6: f(B0(), B1(), B1()); break;
    default: f(B1(), B1(), B1()); break;
    }
}

template <typename T>
int run(std::ifstream& in) {
    using Node = bvh::v2::Node<T, 3>;
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
        for (size_t k = 0; k < prim_count; ++k) mesh.dev_tris[k] = bvhb200::precompute_tri(&mesh.verts[9 * ids[k]]);
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
    const T id9[9] = { 1, 0, 0, 0, 1, 0, 0, 0, 1 }, half9[9] = { 0.5, 0, 0, 0, 0.5, 0, 0, 0, 0.5 };
    const T perm9[9] = { 0, 0, 1, 1, 0, 0, 0, 1, 0 }, zero3[3] = { 0, 0, 0 }, zero9[9] = {};
    const T flat_y[9] = { 1, 0, 0, 0, 0, 0, 0, 0, 1 }, flat_x[9] = { 0, 0, 0, 0, 1, 0, 0, 0, 1 };
    const T step[3] = { size / 3, -size / 5, size / 7 };
    uint64_t seed = 12345;
    auto rnd = [&] { seed = seed * 6364136223846793005ull + 1442695040888963407ull; return T((seed >> 11) * (1.0 / 9007199254740992.0)); };
    auto rot = [&](T scale, T (&a)[9]) { rotation<T>(rnd() * T(6.283185307179586), rnd() - T(0.5), rnd() - T(0.5), rnd() - T(0.5), scale, a); };
    struct Scene { const char* name; std::vector<Placement<T>> place; };
    std::vector<Scene> scenes;
    {
        std::vector<Placement<T>> p;
        for (size_t k = 0; k < 20; ++k) {
            const T sh[3] = { (rnd() - T(0.5)) * size, (rnd() - T(0.5)) * size, (rnd() - T(0.5)) * size / 2 };
            T a[9];
            switch (k % 7) {
            case 0: std::copy(id9, id9 + 9, a); break;
            case 1: std::copy(half9, half9 + 9, a); break;
            case 2: std::copy(perm9, perm9 + 9, a); break;
            case 6: std::copy(flat_y, flat_y + 9, a); break;
            default: rot(T(1), a); break;
            }
            const Key<T> key = linear_about<T>(a, c, k == 0 ? zero3 : sh);
            p.push_back({ k % meshes.size(), key, key });
        }
        scenes.push_back({ "equal", p });
    }
    {
        std::vector<Placement<T>> p;
        for (size_t k = 0; k < 6; ++k) {
            const T sh[3] = { (T(k) - T(2.5)) * size / 2, (rnd() - T(0.5)) * size / 4, 0 };
            const T sh1[3] = { sh[0] + step[0], sh[1] + step[1], sh[2] + step[2] };
            p.push_back({ k % meshes.size(), linear_about<T>(id9, c, sh), linear_about<T>(id9, c, sh1) });
        }
        scenes.push_back({ "translate", p });
    }
    {
        std::vector<Placement<T>> p;
        for (size_t k = 0; k < 6; ++k) {
            T a0[9], a1[9];
            rot(T(1), a0);
            rot(T(1.5), a1);
            const T sh[3] = { (T(k) - T(2.5)) * size / 2, 0, 0 };
            const T sh1[3] = { sh[0] + step[0], sh[1] + step[1], sh[2] };
            p.push_back({ k % meshes.size(), linear_about<T>(a0, c, sh), linear_about<T>(a1, c, sh1) });
        }
        scenes.push_back({ "rotscale", p });
    }
    {
        std::vector<Placement<T>> p;
        for (size_t k = 0; k < 4; ++k) {
            T a1[9];
            rot(T(1), a1);
            const T sh[3] = { (T(k) - T(1.5)) * size / 2, 0, 0 };
            p.push_back({ k % meshes.size(), linear_about<T>(zero9, c, sh), linear_about<T>(a1, c, sh) });
        }
        scenes.push_back({ "singular_end", p });
    }
    {
        std::vector<Placement<T>> p;
        p.push_back({ 0, linear_about<T>(flat_y, c, zero3), linear_about<T>(flat_x, c, step) });
        p.push_back({ meshes.size() - 1, linear_about<T>(flat_x, c, zero3), linear_about<T>(flat_y, c, zero3) });
        p.push_back({ 0, linear_about<T>(id9, c, zero3), linear_about<T>(half9, c, step) });
        scenes.push_back({ "both_singular", p });
    }
    {
        std::vector<Placement<T>> p;
        Key<T> bad0 = linear_about<T>(id9, c, zero3), bad1 = bad0;
        bad0.m[5] = std::numeric_limits<T>::quiet_NaN();
        bad1.m[3] = std::numeric_limits<T>::infinity();
        const Key<T> ok = linear_about<T>(id9, c, zero3);
        p.push_back({ 0, bad0, ok });
        p.push_back({ 0, linear_about<T>(id9, c, zero3), linear_about<T>(id9, c, step) });
        p.push_back({ 0, ok, bad1 });
        scenes.push_back({ "non_finite", p });
    }

    std::vector<size_t> offsets(kPaths + 1, 0);
    for (size_t i = 0; i < kPaths; ++i) offsets[i + 1] = offsets[i] + path_length(i);
    const size_t seg_count = offsets[kPaths];

    unsigned long long cursor = 0;
    int failures = 0;
    for (const Scene& scene : scenes) {
        const size_t count = scene.place.size();
        std::vector<cu::MotionInstance<T>> records(count);
        size_t max_depth = 0;
        for (size_t k = 0; k < count; ++k) {
            const Placement<T>& pl = scene.place[k];
            records[k] = cu::make_motion_instance(meshes[pl.mesh].view, pl.k0.m, pl.k1.m);
            max_depth = std::max(max_depth, meshes[pl.mesh].view.depth);
        }
        const cu::MotionInstances<T> inst { records.data(), count, max_depth };
        std::vector<BBox> boxes(count);
        std::vector<VecC> centres(count);
        cu::prepare_motion_instances(inst, boxes.data(), centres.data());
        const bvh::v2::Bvh<Node> top_bvh = build_top<T>(boxes, centres);
        std::vector<bvhb200::DevNode<T>> top_nodes;
        std::vector<uint32_t> top_ids;
        cu::DeviceView<T> top;
        device_layout<T>(top_bvh, top_nodes, top_ids, top);

        // instance_at at the keys, and the boxes over the shutter
        int key_bad = 0, box_bad = 0, empty = 0;
        for (size_t k = 0; k < count; ++k) {
            const Placement<T>& pl = scene.place[k];
            bool finite = true;
            for (int q = 0; q < 12; ++q) finite = finite && std::isfinite(pl.k0.m[q]) && std::isfinite(pl.k1.m[q]);
            for (int e = 0; e < 2; ++e) {
                const Key<T>& key = e ? pl.k1 : pl.k0;
                const cu::Instance<T> at = cu::instance_at(records[k], T(e));
                cu::Instance<T> st = cu::make_instance(meshes[pl.mesh].view, key.m);
                BBox b; VecC m;
                cu::detail::prepare_instance(st, b, m);
                key_bad += std::memcmp(at.object_to_world, key.m, sizeof key.m) != 0;
                key_bad += std::memcmp(at.world_to_object, st.world_to_object, sizeof key.m) != 0;
                key_bad += at.root_index != records[k].root_index || at.nodes != records[k].nodes || at.depth != records[k].depth;
            }
            const BBox& b = boxes[k];
            if (!finite) {
                empty += b.min.x == std::numeric_limits<T>::infinity() && b.max.x == -std::numeric_limits<T>::infinity();
                continue;
            }
            const std::vector<T>& v = meshes[pl.mesh].verts;
            const T lo[3] = { b.min.x, b.min.y, b.min.z }, hi[3] = { b.max.x, b.max.y, b.max.z };
            for (int s = 0; s <= 64; ++s) {
                const cu::Instance<T> at = cu::instance_at(records[k], T(s) / T(64));
                for (size_t p = 0; p < v.size(); p += 3)
                    for (int a = 0; a < 3; ++a) {
                        const T* row = at.object_to_world + 4 * a;
                        const long double x = (long double)row[0] * v[p] + (long double)row[1] * v[p + 1] + (long double)row[2] * v[p + 2] + row[3];
                        box_bad += !((long double)lo[a] <= x && x <= (long double)hi[a]);
                    }
            }
        }
        std::printf("scene %s keys mismatches %d box misses %d empty boxes %d\n", scene.name, key_bad, box_bad, empty);
        failures += key_bad + box_bad;

        // rays: the motion call against the static call over instance_at at each ray's time
        for (int filter = 0; filter < kFilters; ++filter) {
            for (int mode = 0; mode < 8; ++mode) {
                std::vector<Out> got(ray_count), want(ray_count);
                std::memset(got.data(), 0, got.size() * sizeof(Out));
                std::memset(want.data(), 0, want.size() * sizeof(Out));
                by_mode(mode, [&](auto any, auto rob, auto lst) {
                    constexpr bool A = decltype(any)::value, Rb = decltype(rob)::value, L = decltype(lst)::value;
                    top.template trace_instances<A, Rb, L>(ray_count, inst, Recorder<T> { rays.data(), filter, got.data(), 0 }, &cursor,
                                                           sizeof cursor);
                    std::vector<cu::Instance<T>> at(count);
                    for (size_t i = 0; i < ray_count; ++i) {
                        for (size_t k = 0; k < count; ++k) at[k] = cu::instance_at(records[k], time_of<T>(i));
                        const cu::Instances<T> st { at.data(), count, max_depth };
                        top.template trace_instances<A, Rb, L>(1, st, Recorder<T> { rays.data(), filter, want.data() + i, i }, &cursor,
                                                               sizeof cursor);
                    }
                });
                int bad = 0, hits = 0;
                uint64_t calls = 0;
                for (size_t i = 0; i < ray_count; ++i) {
                    hits += got[i].inst != kNone;
                    calls += got[i].calls;
                    if (std::memcmp(&got[i], &want[i], sizeof(Out)) != 0) {
                        if (bad < 3) std::printf("  %s ray %zu: calls %u/%u id %llu/%llu inst %u/%u\n", scene.name, i, got[i].calls, want[i].calls,
                                                 (unsigned long long)got[i].id, (unsigned long long)want[i].id, got[i].inst, want[i].inst);
                        ++bad;
                    }
                }
                std::printf("rays %s filter %d mode %d mismatches %d hits %d accept calls %llu\n", scene.name, filter, mode, bad, hits,
                            (unsigned long long)calls);
                failures += bad;
            }
        }

        // paths: each segment against the static call of its world ray at the path's time
        for (int filter = 0; filter < kFilters; ++filter) {
            for (int mode = 0; mode < 4; ++mode) {
                std::vector<Out> segs(seg_count + 1), want(seg_count + 1);
                std::memset(segs.data(), 0, segs.size() * sizeof(Out));
                std::memset(want.data(), 0, want.size() * sizeof(Out));
                std::vector<uint32_t> starts(kPaths), finishes(kPaths);
                const PathRecorder<T> shader { rays.data(), ray_count, filter, offsets.data(), segs.data(), starts.data(), finishes.data() };
                by_mode(mode << 1, [&](auto, auto rob, auto lst) {
                    constexpr bool Rb = decltype(rob)::value, L = decltype(lst)::value;
                    top.template trace_instance_paths<Rb, L>(kPaths, inst, shader, &cursor, sizeof cursor);
                    std::vector<cu::Instance<T>> at(count);
                    for (size_t i = 0; i < kPaths; ++i) {
                        for (size_t k = 0; k < count; ++k) at[k] = cu::instance_at(records[k], time_of<T>(i));
                        const cu::Instances<T> st { at.data(), count, max_depth };
                        for (size_t j = 0; j < path_length(i); ++j) {
                            const uint32_t h = segment_hash(i, j);
                            const Recorder<T> r { rays.data(), filter, want.data() + offsets[i] + j, h % ray_count };
                            if (h >> 31) top.template trace_instances<true, Rb, L>(1, st, r, &cursor, sizeof cursor);
                            else top.template trace_instances<false, Rb, L>(1, st, r, &cursor, sizeof cursor);
                        }
                    }
                });
                int bad = 0, path_bad = 0, hits = 0;
                for (size_t i = 0; i < kPaths; ++i) path_bad += starts[i] != 1 || finishes[i] != 1;
                for (size_t k = 0; k < seg_count; ++k) {
                    hits += segs[k].inst != kNone;
                    if (std::memcmp(&segs[k], &want[k], sizeof(Out)) != 0) {
                        if (bad < 3) std::printf("  %s segment %zu: calls %u/%u id %llu/%llu inst %u/%u ray %s\n", scene.name, k, segs[k].calls,
                                                 want[k].calls, (unsigned long long)segs[k].id, (unsigned long long)want[k].id, segs[k].inst,
                                                 want[k].inst, segs[k].ray_ok ? "ok" : "CHANGED");
                        ++bad;
                    }
                }
                std::printf("paths %s filter %d mode %d segments %zu mismatches %d path mismatches %d hits %d\n", scene.name, filter, mode,
                            seg_count, bad, path_bad, hits);
                failures += bad + path_bad;
            }
        }

        if (std::string(scene.name) == "rotscale") {
            // n = 0 calls nothing; a record count other than the top tree's, a small workspace or a stack beyond 200 KB throw
            std::vector<Out> out(ray_count);
            const Recorder<T> rec { rays.data(), 0, out.data(), 0 };
            std::vector<uint32_t> starts(kPaths), finishes(kPaths);
            const PathRecorder<T> paths { rays.data(), ray_count, 0, offsets.data(), out.data(), starts.data(), finishes.data() };
            top.template trace_instances<false, false>(0, inst, rec, &cursor, sizeof cursor);
            top.template trace_instance_paths<false>(0, inst, paths, &cursor, sizeof cursor);
            const bool empty_ok = starts[0] == 0 && finishes[0] == 0;
            cu::MotionInstances<T> fewer = inst, deep = inst;
            fewer.count -= 1;
            deep.max_depth = 400;
            int threw = 0;
            auto expect = [&](auto&& f, const char* name, bool length) {
                try { f(); } catch (const std::length_error& e) {
                    threw += length && std::string(e.what()).find(name) != std::string::npos;
                } catch (const std::invalid_argument& e) {
                    threw += !length && std::string(e.what()).find(name) != std::string::npos;
                }
            };
            const char* ti = "DeviceView::trace_instances (motion):";
            const char* tp = "DeviceView::trace_instance_paths (motion):";
            expect([&] { top.template trace_instances<false, false>(1, fewer, rec, &cursor, sizeof cursor); }, ti, false);
            expect([&] { top.template trace_instances<false, false>(1, inst, rec, &cursor, sizeof cursor - 1); }, ti, true);
            expect([&] { top.template trace_instances<false, false>(1, deep, rec, &cursor, sizeof cursor); }, ti, true);
            expect([&] { top.template trace_instance_paths<false>(1, fewer, paths, &cursor, sizeof cursor); }, tp, false);
            expect([&] { top.template trace_instance_paths<false>(1, inst, paths, &cursor, sizeof cursor - 1); }, tp, true);
            expect([&] { top.template trace_instance_paths<false>(1, deep, paths, &cursor, sizeof cursor); }, tp, true);
            std::printf("empty batch %s, errors thrown %d of 6\n", empty_ok ? "ok" : "CALLED", threw);
            if (!empty_ok || threw != 6) ++failures;
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
