// tests/device_motion_nodes_host_test.cpp — prepare_motion_nodes, node_at and the motion-node forms of
// DeviceView::trace_triangles and trace_paths (include/bvh/v2/cuda/intersect.cuh) compiled as plain host C++, against the
// motion forms without motion nodes and the C++ surface's Bvh<Node>::intersect with a triangle_at leaf, both on a copy
// of the tree whose node bounds are node_at at the ray's time.
//
//   device_motion_nodes_host_test <case file> f|d    one mesh and its rays, as tests/device_instance_trace_host_test.cpp
//                                                     reads them (written by tests/test_device_motion_nodes_host.py).
// The tree keeps the mesh's topology, refitted here from prepare_motion_triangles' boxes (the shutter-box tree), and its
// motion nodes come from prepare_motion_nodes.  The key pairs are those of tests/device_motion_triangle_host_test.cpp:
// equal (one pointer twice), translate, rotscale, jitter, collapse, flip, offset (at 1e4), ulps (at 1e4, keys one to
// three ulps apart), non_finite and partial (the triangles below the median x static, the others moving onto the mesh at
// time 1, with rays at the edge midpoints of the static triangles nearest the moving part).  Ray i has time time_of(i): 0, 1, 0.5, 0.3, a random time, -1, 2 and NaN.  Per key
// pair it checks:
//   * every record's index is the view's; with equal keys both keys of every record are the shutter-box tree's bounds
//     bit for bit;
//   * containment: at 65 uniform times, at adversarial ones (around 0.5, just below 1, the smallest positive times) and
//     at 1024 full-mantissa random times, every node_at box holds triangle_at of every finite triangle of its subtree;
//     a node that holds nothing is +-max at every time.  It counts the coordinates the blend of the unwidened key
//     boxes would miss ("plain misses": the rounding the widening is there for; the ulps pair has them);
//   * for any-hit and closest-hit, both robust settings, both tie rules and three filters (accept all, reject odd ids, an
//     alpha cut-out), per ray: the accept-call count, a hash of the accept sequence (original id, bits of t, u, v) and the
//     record equal the motion form without motion nodes, and the surface's Bvh::intersect, on the tree at the ray's
//     time; with equal keys they also equal the motion form on the shutter-box tree, and robust closest-hit records with
//     canonical ties equal its records for every key pair;
//   * for both robust settings, both tie rules and the three filters, scripted paths of 0 to 16 mixed segments at
//     time_of(i): per segment the same equality, and next receives the segment's ray bit for bit;
//   * n = 0 calls nothing; a wrong node count, a null motion-node pointer, a small workspace and a too-deep stack throw,
//     naming the motion-node call; prepare_motion_nodes throws on a wrong triangle count, a null pointer and a small
//     workspace, naming itself.
#include <bvh/v2/bvh.h>
#include <bvh/v2/cuda/intersect.cuh>
#include <bvh/v2/stack.h>
#include <bvh/v2/tri.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <functional>
#include <limits>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

namespace {

namespace cu = bvh::v2::cuda;
using cu::PathStep;

uint64_t mix(uint64_t h, uint64_t x) { return (h ^ x) * 1099511628211ull; }
constexpr uint64_t kSeed = 1469598103934665603ull;
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

enum Filter : int { kAll = 0, kEvenIds, kAlpha, kFilters };
template <typename T> bool keep(int filter, size_t id, T u, T v) {
    if (filter == kEvenIds) return (id & 1) == 0;
    if (filter == kAlpha) return u < T(0.5) || v < T(0.25);
    return true;
}

struct Out { uint64_t id, t, u, v; uint32_t calls, ray_ok; uint64_t hash; };

template <typename T> using RayOf = typename cu::DeviceView<T>::Ray;
template <typename T> RayOf<T> load_ray(const T* r) {
    RayOf<T> x;
    x.org.x = r[0]; x.org.y = r[1]; x.org.z = r[2];
    x.dir.x = r[3]; x.dir.y = r[4]; x.dir.z = r[5];
    x.tmin = r[6]; x.tmax = r[7];
    return x;
}

// The recording shader: ray first + i at time_of(first + i); `time_index`, when not SIZE_MAX, overrides the time's index
// (a path segment at its path's time)
template <typename T> struct Recorder {
    using Hit = typename cu::DeviceView<T>::Hit;
    struct Payload { uint32_t calls; uint64_t hash; };
    const T* rays;
    int filter;
    Out* out;
    size_t first;
    size_t time_index = SIZE_MAX;

    RayOf<T> start(size_t i, Payload& p, T& time) const {
        p.calls = 0; p.hash = kSeed;
        time = time_of<T>(time_index != SIZE_MAX ? time_index : first + i);
        return load_ray(rays + 8 * (first + i));
    }
    bool accept(Payload& p, size_t id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(p.hash, id), bits(t)), bits(u)), bits(v));
        return keep<T>(filter, id, u, v);
    }
    void finish(size_t i, const Payload& p, const Hit& hit) const {
        Out& o = out[i];
        o.id = hit.prim_id; o.t = bits(hit.t); o.u = bits(hit.u); o.v = bits(hit.v);
        o.calls = p.calls; o.hash = p.hash; o.ray_ok = 1;
    }
};

// The path shader: scripted segments, path i at time_of(i); per segment its record in segs[offsets[i] + j]
template <typename T> struct PathRecorder {
    using Hit = typename cu::DeviceView<T>::Hit;
    struct Payload { size_t seg; uint32_t calls; uint64_t hash; };
    const T* rays;
    size_t ray_count;
    int filter;
    const size_t* offsets;
    Out* segs;
    uint32_t* starts;
    uint32_t* finishes;

    PathStep segment(size_t i, size_t j, RayOf<T>& ray) const {
        const uint32_t h = segment_hash(i, j);
        ray = load_ray(rays + 8 * (h % ray_count));
        return (h >> 31) ? PathStep::Occlusion : PathStep::Closest;
    }
    PathStep start(size_t i, Payload& p, RayOf<T>& ray, T& time) const {
        starts[i] += 1;
        p.seg = 0; p.calls = 0; p.hash = kSeed;
        time = time_of<T>(i);
        return path_length(i) ? segment(i, 0, ray) : PathStep::End;
    }
    bool accept(Payload& p, size_t id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(p.hash, id), bits(t)), bits(u)), bits(v));
        return keep<T>(filter, id, u, v);
    }
    PathStep next(size_t i, Payload& p, const Hit& hit, RayOf<T>& ray) const {
        RayOf<T> want;
        segment(i, p.seg, want);
        Out& s = segs[offsets[i] + p.seg];
        s.ray_ok = std::memcmp(&want, &ray, sizeof ray) == 0;
        s.id = hit.prim_id; s.t = bits(hit.t); s.u = bits(hit.u); s.v = bits(hit.v);
        s.calls = p.calls; s.hash = p.hash;
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

// A static part meeting a moving one (both builds of the bound's case): a root over an inner node and a far leaf C; the
// inner node over leaf A, one static triangle with an edge on x = L, and leaf B, one triangle whose lowest x moves from
// L + 10 at time 0 to exactly L at time 1.  The inner node's lower x keys then differ (L, L - d) over A's equal keys
// (L, L).  For `meshes` values of L in [1e3, 1e5] and `times` full-mantissa times in (0, 0.1) it counts the node_at boxes
// (inner node and root) whose lower x lies above L, and the rays down the edge x = L (robust, closest-hit) whose record
// differs from the motion call on the shutter-box tree.
struct MeetShader {
    template <typename T> struct S {
        using Hit = typename cu::DeviceView<T>::Hit;
        struct Payload {};
        T x;
        const T* times;
        uint32_t* ids;
        RayOf<T> start(size_t i, Payload&, T& time) const {
            time = times[i];
            RayOf<T> r;
            r.org.x = x; r.org.y = T(0.5); r.org.z = T(1); r.dir.x = T(0); r.dir.y = T(0); r.dir.z = T(-1);
            r.tmin = T(0); r.tmax = std::numeric_limits<T>::infinity();
            return r;
        }
        bool accept(Payload&, size_t, T, T, T) const { return true; }
        void finish(size_t i, const Payload&, const Hit& h) const { ids[i] = (uint32_t)h.prim_id; }
    };
};
template <typename T> void meet(size_t meshes, size_t times_per_mesh, int& box_misses, int& lost_hits) {
    using View = cu::DeviceView<T>;
    using U = typename bvhb200::Real<T>::UInt;
    box_misses = lost_hits = 0;
    const U index[5] = { bvhb200::make_index<U>(1, 0), bvhb200::make_index<U>(3, 0), bvhb200::make_index<U>(2, 1),
                         bvhb200::make_index<U>(0, 1), bvhb200::make_index<U>(1, 1) };
    const uint32_t ids[3] = { 0, 1, 2 };
    uint64_t seed = 99;
    auto rnd = [&] { seed = seed * 6364136223846793005ull + 1442695040888963407ull; return (double)((seed >> 11) * (1.0 / 9007199254740992.0)); };
    std::vector<T> times(times_per_mesh);
    std::vector<uint32_t> got(times_per_mesh), want(times_per_mesh);
    for (size_t m = 0; m < meshes; ++m) {
        const T L = T(1e3 + rnd() * (1e5 - 1e3));
        const T k0[27] = { L, 0, 0, L, 1, 0, L + 1, 0, 0,   L + 10, 2, 0, L + 11, 2, 0, L + 10, 3, 0,   L + 100, 0, 0, L + 101, 0, 0, L + 100, 1, 0 };
        T k1[27];
        std::memcpy(k1, k0, sizeof k1);
        for (int q = 9; q < 18; q += 3) k1[q] -= T(10);                     // B: lowest x exactly L at time 1
        const cu::MotionTriangles<T> motion { { k0, k1 }, 3 };
        typename cu::detail::ViewTypes<T>::BBox boxes[3];
        typename cu::detail::ViewTypes<T>::Vec centres[3];
        cu::prepare_motion_triangles(motion, boxes, centres);
        bvhb200::DevNode<T> nodes[6];
        std::memset(nodes, 0, sizeof nodes);
        for (int i = 0; i < 5; ++i) nodes[i + 1].index = index[i];
        uint32_t parent[6] = {};
        int flags[6] = {};
        for (size_t i = 1; i < 6; ++i) bvhb200::refit_link(nodes, 6, i, parent, flags);
        for (size_t i = 6; i-- > 1;)
            bvhb200::refit_from_leaf<T>(nodes, i, parent, flags, ids, bvhb200::BoxSource<T> { reinterpret_cast<const T*>(boxes) });
        View view;
        view.nodes = nodes; view.prim_ids = ids; view.node_count = 5; view.prim_count = 3; view.depth = 2;
        cu::MotionNode<T> records[6];
        std::memset(records, 0, sizeof records);
        uint32_t workspace[12];
        cu::prepare_motion_nodes(view, motion, records, workspace, sizeof workspace);
        const cu::MotionNodes<T> mn { records, 5 };
        for (T& t : times) t = T(T(rnd() * 0.1) / T(1.0009765625));
        for (T tau : times)
            for (size_t slot : { 1, 2 }) {                              // the root and the inner node over A and B
                T b[6];
                cu::node_at(mn, slot, tau, b);
                box_misses += !(b[0] <= L);
            }
        unsigned long long cursor = 0;
        const typename MeetShader::template S<T> shader_got { L, times.data(), got.data() }, shader_want { L, times.data(), want.data() };
        view.template trace_triangles<false, true>(times.size(), motion, mn, shader_got, &cursor, sizeof cursor);
        view.template trace_triangles<false, true>(times.size(), motion, shader_want, &cursor, sizeof cursor);
        for (size_t i = 0; i < times.size(); ++i) lost_hits += got[i] != want[i];
    }
}

template <typename T>
int run(std::ifstream& in) {
    using Node = bvh::v2::Node<T, 3>;
    using Bvh = bvh::v2::Bvh<Node>;
    using Vec3 = bvh::v2::Vec<T, 3>;
    using View = cu::DeviceView<T>;
    using BBox = typename cu::detail::ViewTypes<T>::BBox;
    using VecC = typename cu::detail::ViewTypes<T>::Vec;
    uint64_t mesh_count = 0, node_count = 0, prim_count = 0, ray_count = 0;
    in.read((char*)&mesh_count, 8);
    in.read((char*)&node_count, 8); in.read((char*)&prim_count, 8);
    Bvh bvh;
    bvh.nodes.resize(node_count);
    in.read((char*)bvh.nodes.data(), node_count * sizeof(Node));
    std::vector<uint64_t> ids(prim_count);
    in.read((char*)ids.data(), prim_count * 8);
    bvh.prim_ids.assign(ids.begin(), ids.end());
    std::vector<T> mesh(9 * prim_count);
    in.read((char*)mesh.data(), mesh.size() * sizeof(T));
    in.read((char*)&ray_count, 8);
    std::vector<T> base_rays(8 * ray_count);
    in.read((char*)base_rays.data(), base_rays.size() * sizeof(T));
    if (!in || mesh_count != 1) { std::puts("short input"); return 2; }
    const std::vector<uint32_t> ids32(ids.begin(), ids.end());
    const size_t depth = tree_depth<T>(bvh);

    // the key pairs
    T lo[3], hi[3];
    for (int a = 0; a < 3; ++a) { lo[a] = hi[a] = mesh[a]; }
    for (size_t k = 0; k < mesh.size(); ++k) { lo[k % 3] = std::min(lo[k % 3], mesh[k]); hi[k % 3] = std::max(hi[k % 3], mesh[k]); }
    const T c[3] = { (lo[0] + hi[0]) / 2, (lo[1] + hi[1]) / 2, (lo[2] + hi[2]) / 2 };
    const T size = std::max({ hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2], T(1e-3) });
    const T step = size / T(2 * std::cbrt((double)prim_count + 1));      // about a triangle's size
    uint64_t seed = 12345;
    auto rnd = [&] { seed = seed * 6364136223846793005ull + 1442695040888963407ull; return T((seed >> 11) * (1.0 / 9007199254740992.0)); };
    struct Scene { const char* name; std::vector<T> k0, k1; T offset; bool same; };
    std::vector<Scene> scenes;
    auto moved = [&](auto&& f) {
        std::vector<T> out(mesh);
        for (size_t t = 0; t < prim_count; ++t) f(t, &out[9 * t]);
        return out;
    };
    scenes.push_back({ "equal", mesh, mesh, T(0), true });
    scenes.push_back({ "translate", mesh, moved([&](size_t, T* v) {
        for (int q = 0; q < 9; ++q) v[q] += (q % 3 == 0 ? step : q % 3 == 1 ? -step / 2 : step / 3);
    }), T(0), false });
    {
        const T ang = T(0.3), s = T(1.25), co = std::cos(ang), si = std::sin(ang);
        scenes.push_back({ "rotscale", mesh, moved([&](size_t, T* v) {
            for (int q = 0; q < 9; q += 3) {
                const T x = v[q] - c[0], y = v[q + 1] - c[1], z = v[q + 2] - c[2];
                v[q] = c[0] + s * (co * x - si * y); v[q + 1] = c[1] + s * (si * x + co * y); v[q + 2] = c[2] + s * z;
            }
        }), T(0), false });
    }
    scenes.push_back({ "jitter", mesh, moved([&](size_t, T* v) { for (int q = 0; q < 9; ++q) v[q] += (rnd() - T(0.5)) * step; }), T(0), false });
    scenes.push_back({ "collapse", mesh, moved([&](size_t t, T* v) {
        if (t % 3 == 0) for (int q = 0; q < 3; ++q) v[6 + q] = v[3 + q];                  // p2 onto p1: a segment
        else for (int q = 0; q < 9; ++q) v[q] += (rnd() - T(0.5)) * step;
    }), T(0), false });
    scenes.push_back({ "flip", mesh, moved([&](size_t, T* v) { for (int q = 0; q < 3; ++q) std::swap(v[3 + q], v[6 + q]); }), T(0), false });
    {
        const T off = T(1e4);
        std::vector<T> k0(mesh), k1;
        for (T& x : k0) x += off;
        k1 = k0;
        for (size_t q = 0; q < k1.size(); ++q) k1[q] += (q % 3 == 0 ? step : T(0)) + (rnd() - T(0.5)) * step / 4;
        scenes.push_back({ "offset", k0, k1, off, false });
        // the same place, each coordinate moved by 1 to 3 ulps either way: the blend's rounding can leave the keys'
        // interval, and the extreme coordinate of an axis is one whose keys are that close
        // (here key 0 also moves each coordinate by 0 to 2 ulps, so that vertices shared by neighbouring triangles of a
        // grid differ at both keys: a leaf's extreme coordinate then comes from different vertices at the two keys, in
        // double as in float, and the blend of the unwidened key boxes can miss the blended vertices)
        std::vector<T> u0(k0);
        for (T& x : u0) {
            const uint32_t h = hash32((uint32_t)(&x - u0.data()) ^ 0x9E3779B9u);
            for (uint32_t q = 0; q < h % 3; ++q) x = std::nextafter(x, (h >> 8) & 1 ? std::numeric_limits<T>::infinity() : -std::numeric_limits<T>::infinity());
        }
        std::vector<T> u1(u0);
        for (T& x : u1) {
            const uint32_t h = hash32((uint32_t)(&x - u1.data()) ^ 0x2545F491u);
            for (uint32_t q = 0; q < 1 + h % 3; ++q) x = std::nextafter(x, (h >> 8) & 1 ? std::numeric_limits<T>::infinity() : -std::numeric_limits<T>::infinity());
        }
        scenes.push_back({ "ulps", u0, u1, off, false });
    }
    {
        std::vector<T> k1 = moved([&](size_t, T* v) { for (int q = 0; q < 9; ++q) v[q] += (q % 3 == 1 ? step : T(0)); }), k0(mesh);
        for (size_t t = 0; t < prim_count; t += 7) {
            if ((t / 7) % 2 == 0) k0[9 * t + 4] = std::numeric_limits<T>::quiet_NaN();
            else k1[9 * t + 2] = std::numeric_limits<T>::infinity();
        }
        scenes.push_back({ "non_finite", k0, k1, T(0), false });
    }
    // part of the mesh static: the triangles whose centre lies below the median x stay, the others move from the mesh
    // moved by a triangle's size at time 0 to the mesh itself at time 1.  Where a static and a moving leaf meet (a grid's
    // shared vertices) a bound of the moving one reaches the static one's exactly at key 1, so their parent's keys differ
    // over a child whose keys are equal
    std::vector<T> centre_x(prim_count);
    for (size_t t = 0; t < prim_count; ++t) centre_x[t] = (mesh[9 * t] + mesh[9 * t + 3] + mesh[9 * t + 6]) / T(3);
    std::vector<T> sorted_x(centre_x);
    std::nth_element(sorted_x.begin(), sorted_x.begin() + prim_count / 2, sorted_x.end());
    const T median_x = sorted_x[prim_count / 2];
    auto is_static = [&](size_t t) { return centre_x[t] < median_x; };
    scenes.push_back({ "partial", moved([&](size_t t, T* v) {
        if (!is_static(t)) for (int q = 0; q < 9; ++q) v[q] += (q % 3 == 0 ? step : q % 3 == 1 ? -step / 2 : step / 3);
    }), mesh, T(0), false });

    int meet_misses = 0, meet_lost = 0;
    meet<T>(500, 1000, meet_misses, meet_lost);
    std::printf("meet box misses %d lost hits %d\n", meet_misses, meet_lost);
    int failures = meet_misses + meet_lost;

    std::vector<size_t> offsets(kPaths + 1, 0);
    for (size_t i = 0; i < kPaths; ++i) offsets[i + 1] = offsets[i] + path_length(i);
    const size_t seg_count = offsets[kPaths];

    unsigned long long cursor = 0;
    for (const Scene& scene : scenes) {
        std::vector<T> rays(base_rays);
        for (size_t i = 0; i < ray_count; ++i)
            for (int a = 0; a < 3; ++a) rays[8 * i + a] += scene.offset;
        if (std::string(scene.name) == "partial") {
            // the last rays aimed at the edge midpoints of the static triangles nearest the moving part, along the
            // triangle's normal: an edge on which a coordinate is constant is where a node box one ulp short loses the hit
            std::vector<size_t> near;
            for (size_t t = 0; t < prim_count; ++t)
                if (is_static(t)) near.push_back(t);
            std::sort(near.begin(), near.end(), [&](size_t a, size_t b) { return centre_x[a] > centre_x[b] || (centre_x[a] == centre_x[b] && a < b); });
            size_t r = ray_count;
            for (size_t j = 0; j < near.size() && r > ray_count / 2; ++j)
                for (int e = 0; e < 3 && r > ray_count / 2; ++e) {
                    const T* p = &mesh[9 * near[j]];
                    const T e1[3] = { p[3] - p[0], p[4] - p[1], p[5] - p[2] }, e2[3] = { p[6] - p[0], p[7] - p[1], p[8] - p[2] };
                    const T n[3] = { e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0] };
                    T* ray = &rays[8 * --r];
                    for (int a = 0; a < 3; ++a) {
                        const T mid = (p[3 * e + a] + p[3 * ((e + 1) % 3) + a]) / T(2);
                        ray[a] = mid + n[a];
                        ray[3 + a] = -n[a];
                    }
                    ray[6] = T(0); ray[7] = std::numeric_limits<T>::infinity();
                }
        }
        const cu::MotionTriangles<T> motion { { scene.k0.data(), scene.same ? scene.k0.data() : scene.k1.data() }, prim_count };
        std::vector<BBox> boxes(prim_count);
        std::vector<VecC> centres(prim_count);
        cu::prepare_motion_triangles(motion, boxes.data(), centres.data());
        // the shutter-box tree: the library's refit (refit_from_leaf) of the topology over prepare_motion_triangles' boxes
        const size_t slots = node_count + 1;
        std::vector<bvhb200::DevNode<T>> dev_nodes(slots);
        std::memset(dev_nodes.data(), 0, dev_nodes.size() * sizeof(dev_nodes[0]));
        for (size_t i = 0; i < node_count; ++i) dev_nodes[i + 1].index = bvh.nodes[i].index.value;
        {
            std::vector<uint32_t> parent(slots, 0);
            std::vector<int> flags(slots, 0);
            for (size_t i = 1; i < slots; ++i) bvhb200::refit_link(dev_nodes.data(), slots, i, parent.data(), flags.data());
            for (size_t i = slots; i-- > 1;)
                bvhb200::refit_from_leaf<T>(dev_nodes.data(), i, parent.data(), flags.data(), ids32.data(),
                                            bvhb200::BoxSource<T> { reinterpret_cast<const T*>(boxes.data()) });
        }
        View view;                                      // no triangles: a tree over boxes
        view.nodes = dev_nodes.data(); view.prim_ids = ids32.data();
        view.node_count = node_count; view.prim_count = prim_count; view.depth = depth;

        // the motion nodes
        std::vector<cu::MotionNode<T>> mnodes(slots);
        std::memset(mnodes.data(), 0, mnodes.size() * sizeof(mnodes[0]));
        std::vector<unsigned char> workspace(view.bottom_up_workspace_bytes());
        cu::prepare_motion_nodes(view, motion, mnodes.data(), workspace.data(), workspace.size());
        const cu::MotionNodes<T> mn { mnodes.data(), node_count };
        auto key_bounds = [&](size_t s, int k, T b[6]) {
            for (int q = 0; q < 4; ++q) b[q] = mnodes[s].xy[k][q];
            b[4] = mnodes[s].z[k][0]; b[5] = mnodes[s].z[k][1];
        };
        int index_bad = 0, equal_bad = 0;
        for (size_t s = 1; s < slots; ++s) {
            index_bad += mnodes[s].index != dev_nodes[s].index;
            for (int k = 0; k < 2 && scene.same; ++k) {
                T b[6];
                key_bounds(s, k, b);
                equal_bad += std::memcmp(b, dev_nodes[s].bounds, sizeof b) != 0;
            }
        }

        // containment: per time, every node_at box against the extent of triangle_at over its subtree's finite triangles,
        // and the blend of the unwidened key boxes (the per-key unions without the widening) against the same extent
        std::vector<char> finite(prim_count);
        for (size_t t = 0; t < prim_count; ++t) {
            bool ok = true;
            for (int q = 0; q < 9; ++q) ok = ok && std::isfinite(motion.vertices[0][9 * t + q]) && std::isfinite(motion.vertices[1][9 * t + q]);
            finite[t] = ok;
        }
        const bool all_finite = std::all_of(finite.begin(), finite.end(), [](char f) { return f != 0; });
        const T inf = std::numeric_limits<T>::infinity(), big = std::numeric_limits<T>::max();
        std::vector<T> plain(12 * slots);             // [slot][key][6]
        std::function<void(size_t)> plain_of = [&](size_t i) {
            T* p = &plain[12 * (i + 1)];
            for (int k = 0; k < 2; ++k)
                for (int a = 0; a < 3; ++a) { p[6 * k + 2 * a] = inf; p[6 * k + 2 * a + 1] = -inf; }
            const auto& node = bvh.nodes[i];
            auto grow = [&](int k, const T* lo, const T* hi, int stride) {
                for (int a = 0; a < 3; ++a) {
                    p[6 * k + 2 * a] = std::min(p[6 * k + 2 * a], lo[stride * a]);
                    p[6 * k + 2 * a + 1] = std::max(p[6 * k + 2 * a + 1], hi[stride * a]);
                }
            };
            if (node.is_leaf()) {
                for (size_t s = node.index.first_id(); s < node.index.first_id() + node.index.prim_count(); ++s) {
                    const size_t id = ids32[s];
                    if (!finite[id]) continue;
                    for (int k = 0; k < 2; ++k) {
                        T lo[3], hi[3], c[3];
                        bvhb200::tri_bounds_center(motion.vertices[k] + 9 * id, lo, hi, c);
                        grow(k, lo, hi, 1);
                    }
                }
                return;
            }
            for (size_t c = node.index.first_id(); c < node.index.first_id() + 2; ++c) {
                plain_of(c);
                for (int k = 0; k < 2; ++k) grow(k, &plain[12 * (c + 1) + 6 * k], &plain[12 * (c + 1) + 6 * k + 1], 2);
            }
        };
        plain_of(0);
        std::vector<T> times;
        for (int s = 0; s <= 64; ++s) times.push_back(T(s) / T(64));
        const T half = T(0.5), one = T(1), zero = T(0);
        for (T x : { std::nextafter(half, zero), std::nextafter(half, one), std::nextafter(one, zero), std::numeric_limits<T>::denorm_min(),
                     std::numeric_limits<T>::min(), std::numeric_limits<T>::epsilon(), T(1) / T(3), T(2) / T(3), T(-1), T(2),
                     std::numeric_limits<T>::quiet_NaN() })
            times.push_back(x);
        for (uint32_t s = 0; s < 1024; ++s)            // full-mantissa random times, as the deforming-mesh host test draws them
            times.push_back(T(T((((uint64_t)hash32(s ^ 0x68E31DA4u) << 32 | hash32(s)) >> 11) * T(1.0 / 9007199254740992.0)) / T(1.0009765625)));
        int box_bad = 0, empty_bad = 0, nan_bad = 0, plain_misses = 0, empty_nodes = 0;
        std::vector<T> at_box(6 * slots), ext(6 * slots);
        for (T tau : times) {
            for (size_t s = 1; s < slots; ++s) cu::node_at(mn, s, tau, &at_box[6 * s]);
            const T ptau = cu::detail::shutter_time(tau), prest = T(1) - ptau;
            std::function<void(size_t)> extent = [&](size_t i) {
                T* e = &ext[6 * (i + 1)];
                for (int a = 0; a < 3; ++a) { e[2 * a] = inf; e[2 * a + 1] = -inf; }
                const auto& node = bvh.nodes[i];
                if (node.is_leaf()) {
                    for (size_t s = node.index.first_id(); s < node.index.first_id() + node.index.prim_count(); ++s) {
                        if (!finite[ids32[s]]) continue;
                        T v[9];
                        cu::triangle_at(motion, ids32[s], tau, v);
                        for (int q = 0; q < 9; ++q) { e[2 * (q % 3)] = std::min(e[2 * (q % 3)], v[q]); e[2 * (q % 3) + 1] = std::max(e[2 * (q % 3) + 1], v[q]); }
                    }
                } else {
                    for (size_t c = node.index.first_id(); c < node.index.first_id() + 2; ++c) {
                        extent(c);
                        const T* ce = &ext[6 * (c + 1)];
                        for (int a = 0; a < 3; ++a) { e[2 * a] = std::min(e[2 * a], ce[2 * a]); e[2 * a + 1] = std::max(e[2 * a + 1], ce[2 * a + 1]); }
                    }
                }
            };
            extent(0);
            for (size_t s = 1; s < slots; ++s) {
                const T* b = &at_box[6 * s];
                const T* e = &ext[6 * s];
                for (int q = 0; q < 6; ++q) nan_bad += b[q] != b[q];
                if (e[0] > e[1]) {                       // holds nothing: +-max at every time
                    ++empty_nodes;
                    for (int a = 0; a < 3; ++a) empty_bad += b[2 * a] != big || b[2 * a + 1] != -big;
                    continue;
                }
                const T* p = &plain[12 * s];
                for (int a = 0; a < 3; ++a) {
                    box_bad += !(b[2 * a] <= e[2 * a] && e[2 * a + 1] <= b[2 * a + 1]);
                    const T plo = cu::detail::blend_key(p[2 * a], p[6 + 2 * a], ptau, prest);
                    const T phi = cu::detail::blend_key(p[2 * a + 1], p[6 + 2 * a + 1], ptau, prest);
                    plain_misses += !(plo <= e[2 * a]) + !(e[2 * a + 1] <= phi);
                }
            }
        }
        std::printf("scene %s index mismatches %d equal-key mismatches %d box misses %d empty misses %d nan bounds %d empty nodes %d plain misses %d\n",
                    scene.name, index_bad, equal_bad, box_bad, empty_bad, nan_bad, empty_nodes, plain_misses);
        failures += index_bad + equal_bad + box_bad + empty_bad + nan_bad;

        // the tree at each time the rays and paths use: the shutter-box tree's topology with node_at's boxes, as device
        // nodes (for the motion form without motion nodes) and as the surface's Bvh
        struct AtTime { std::vector<bvhb200::DevNode<T>> dev; Bvh tree; };
        std::map<uint64_t, AtTime> at;
        auto tree_at = [&](T time) -> const AtTime& {
            AtTime& a = at[bits(time)];
            if (a.dev.empty()) {
                a.dev = dev_nodes;
                a.tree.nodes = bvh.nodes;
                a.tree.prim_ids = bvh.prim_ids;
                for (size_t s = 1; s < slots; ++s) {
                    cu::node_at(mn, s, time, a.dev[s].bounds);
                    for (int q = 0; q < 6; ++q) a.tree.nodes[s - 1].bounds[q] = a.dev[s].bounds[q];
                }
            }
            return a;
        };
        // the shutter-box tree's view with NaN node bounds: the motion-node forms must not read them
        std::vector<bvhb200::DevNode<T>> nan_nodes(dev_nodes);
        for (size_t s = 1; s < slots; ++s)
            for (int q = 0; q < 6; ++q) nan_nodes[s].bounds[q] = std::numeric_limits<T>::quiet_NaN();
        View nan_view = view;
        nan_view.nodes = nan_nodes.data();
        // one ray through the surface's Bvh::intersect on `tree`, whose leaf tests PrecomputedTri(triangle_at(...)) with
        // the tie rule and the filter
        auto surface = [&](const Bvh& tree, int mode, int filter, const T* r, T time) {
            const bool last = mode & 4;
            bvh::v2::Ray<T, 3> ray(Vec3(r[0], r[1], r[2]), Vec3(r[3], r[4], r[5]), r[6], r[7]);
            const T tmax_in = r[7];
            bvh::v2::GrowingStack<typename Node::Index> stack;
            size_t best = SIZE_MAX;
            T bu = T(0), bv = T(0);
            Out o {};
            o.hash = kSeed;
            auto leaf_fn = [&](size_t b, size_t e) {
                for (size_t k = b; k < e; ++k) {
                    const size_t id = tree.prim_ids[k];
                    T v[9];
                    cu::triangle_at(motion, id, time, v);
                    const bvh::v2::PrecomputedTri<T> tri(Vec3(v[0], v[1], v[2]), Vec3(v[3], v[4], v[5]), Vec3(v[6], v[7], v[8]));
                    const auto h = tri.intersect(ray);
                    if (!h) continue;
                    const auto [t, u, w] = *h;
                    if (!last && best != SIZE_MAX && !(t < ray.tmax) && !(id < tree.prim_ids[best])) continue;
                    ++o.calls;
                    o.hash = mix(mix(mix(mix(o.hash, id), bits(t)), bits(u)), bits(w));
                    if (!keep<T>(filter, id, u, w)) continue;
                    ray.tmax = t; best = k; bu = u; bv = w;
                }
                return best != SIZE_MAX;
            };
            if (!(r[6] != r[6] || r[7] != r[7])) {
                const auto root = tree.get_root().index;
                switch (mode & 3) {
                case 0: tree.template intersect<false, false>(ray, root, stack, leaf_fn); break;
                case 1: tree.template intersect<true, false>(ray, root, stack, leaf_fn); break;
                case 2: tree.template intersect<false, true>(ray, root, stack, leaf_fn); break;
                default: tree.template intersect<true, true>(ray, root, stack, leaf_fn); break;
                }
            }
            const bool hit = best != SIZE_MAX;
            o.id = hit ? (uint64_t)tree.prim_ids[best] : (sizeof(T) == 4 ? 0xFFFFFFFFull : ~0ull);
            o.t = bits(hit ? ray.tmax : tmax_in); o.u = bits(bu); o.v = bits(bv);
            o.ray_ok = 1;
            return o;
        };

        // rays: the motion-node call against the motion call and the surface on the tree at each ray's time
        for (int filter = 0; filter < kFilters; ++filter) {
            for (int mode = 0; mode < 8; ++mode) {
                std::vector<Out> got(ray_count), want(ray_count), shutter(ray_count), nan_got(ray_count);
                std::memset(got.data(), 0, got.size() * sizeof(Out));
                std::memset(want.data(), 0, want.size() * sizeof(Out));
                std::memset(shutter.data(), 0, shutter.size() * sizeof(Out));
                std::memset(nan_got.data(), 0, nan_got.size() * sizeof(Out));
                by_mode(mode, [&](auto any, auto rob, auto lst) {
                    constexpr bool A = decltype(any)::value, Rb = decltype(rob)::value, L = decltype(lst)::value;
                    view.template trace_triangles<A, Rb, L>(ray_count, motion, mn, Recorder<T> { rays.data(), filter, got.data(), 0 }, &cursor,
                                                            sizeof cursor);
                    nan_view.template trace_triangles<A, Rb, L>(ray_count, motion, mn, Recorder<T> { rays.data(), filter, nan_got.data(), 0 },
                                                                &cursor, sizeof cursor);
                    if (scene.same || (Rb && !A && !L))
                        view.template trace_triangles<A, Rb, L>(ray_count, motion, Recorder<T> { rays.data(), filter, shutter.data(), 0 }, &cursor,
                                                                sizeof cursor);
                    for (size_t i = 0; i < ray_count; ++i) {
                        View st = view;
                        st.nodes = tree_at(time_of<T>(i)).dev.data();
                        st.template trace_triangles<A, Rb, L>(1, motion, Recorder<T> { rays.data(), filter, want.data() + i, i }, &cursor,
                                                              sizeof cursor);
                    }
                });
                int bad = 0, surf_bad = 0, other_bad = 0, hits = 0;
                uint64_t calls = 0;
                for (size_t i = 0; i < ray_count; ++i) {
                    hits += got[i].id != (sizeof(T) == 4 ? 0xFFFFFFFFull : ~0ull);
                    calls += got[i].calls;
                    const Out s = surface(tree_at(time_of<T>(i)).tree, mode, filter, &rays[8 * i], time_of<T>(i));
                    const bool b1 = std::memcmp(&got[i], &want[i], sizeof(Out)) != 0, b2 = std::memcmp(&got[i], &s, sizeof(Out)) != 0;
                    // with equal keys the shutter-box call bit for bit; with robust closest-hit rays and canonical ties its
                    // record (both trees hold the closest triangle: not so for a triangle with a non-finite key, which
                    // neither tree's boxes hold, but whose leaf a ray may reach for a triangle beside it)
                    const bool b3 = std::memcmp(&got[i], &nan_got[i], sizeof(Out)) != 0 ||
                                    (scene.same && std::memcmp(&got[i], &shutter[i], sizeof(Out)) != 0) ||
                                    (mode == 2 && all_finite && std::memcmp(&got[i], &shutter[i], 4 * sizeof(uint64_t)) != 0);
                    if ((b1 || b2 || b3) && bad + surf_bad + other_bad < 3)
                        std::printf("  %s ray %zu: calls %u/%u/%u id %llu/%llu/%llu\n", scene.name, i, got[i].calls, want[i].calls, s.calls,
                                    (unsigned long long)got[i].id, (unsigned long long)want[i].id, (unsigned long long)s.id);
                    bad += b1;
                    surf_bad += b2;
                    other_bad += b3;
                }
                std::printf("rays %s filter %d mode %d mismatches %d surface mismatches %d shutter/nan mismatches %d hits %d accept calls %llu\n",
                            scene.name, filter, mode, bad, surf_bad, other_bad, hits, (unsigned long long)calls);
                failures += bad + surf_bad + other_bad;
            }
        }

        // paths: each segment against the motion call and the surface on the tree at the path's time
        for (int filter = 0; filter < kFilters; ++filter) {
            for (int mode = 0; mode < 4; ++mode) {
                std::vector<Out> segs(seg_count + 1), want(seg_count + 1);
                std::memset(segs.data(), 0, segs.size() * sizeof(Out));
                std::memset(want.data(), 0, want.size() * sizeof(Out));
                std::vector<uint32_t> starts(kPaths), finishes(kPaths);
                const PathRecorder<T> shader { rays.data(), ray_count, filter, offsets.data(), segs.data(), starts.data(), finishes.data() };
                int surf_bad = 0;
                by_mode(mode << 1, [&](auto, auto rob, auto lst) {
                    constexpr bool Rb = decltype(rob)::value, L = decltype(lst)::value;
                    view.template trace_paths<Rb, L>(kPaths, motion, mn, shader, &cursor, sizeof cursor);
                    for (size_t i = 0; i < kPaths; ++i) {
                        const AtTime& a = tree_at(time_of<T>(i));
                        View st = view;
                        st.nodes = a.dev.data();
                        for (size_t j = 0; j < path_length(i); ++j) {
                            const uint32_t h = segment_hash(i, j);
                            Out* w = want.data() + offsets[i] + j;
                            const Recorder<T> r { rays.data(), filter, w, h % ray_count, i };
                            if (h >> 31) st.template trace_triangles<true, Rb, L>(1, motion, r, &cursor, sizeof cursor);
                            else st.template trace_triangles<false, Rb, L>(1, motion, r, &cursor, sizeof cursor);
                            const Out s = surface(a.tree, ((h >> 31) ? 1 : 0) | (mode << 1), filter, &rays[8 * (h % ray_count)], time_of<T>(i));
                            surf_bad += std::memcmp(w, &s, sizeof(Out)) != 0;
                        }
                    }
                });
                int bad = 0, path_bad = 0, hits = 0;
                for (size_t i = 0; i < kPaths; ++i) path_bad += starts[i] != 1 || finishes[i] != 1;
                for (size_t k = 0; k < seg_count; ++k) {
                    hits += segs[k].id != (sizeof(T) == 4 ? 0xFFFFFFFFull : ~0ull);
                    if (std::memcmp(&segs[k], &want[k], sizeof(Out)) != 0) {
                        if (bad < 3) std::printf("  %s segment %zu: calls %u/%u id %llu/%llu ray %s\n", scene.name, k, segs[k].calls, want[k].calls,
                                                 (unsigned long long)segs[k].id, (unsigned long long)want[k].id, segs[k].ray_ok ? "ok" : "CHANGED");
                        ++bad;
                    }
                }
                std::printf("paths %s filter %d mode %d segments %zu mismatches %d surface mismatches %d path mismatches %d hits %d\n",
                            scene.name, filter, mode, seg_count, bad, surf_bad, path_bad, hits);
                failures += bad + surf_bad + path_bad;
            }
        }

        if (std::string(scene.name) == "jitter") {
            // n = 0 calls nothing; a node count other than the tree's, a null motion-node pointer, a small workspace or a
            // stack beyond 200 KB throw; so does prepare_motion_nodes on a wrong triangle count, a null pointer or a small
            // workspace
            std::vector<Out> out(ray_count);
            const Recorder<T> rec { rays.data(), 0, out.data(), 0 };
            std::vector<uint32_t> starts(kPaths), finishes(kPaths);
            const PathRecorder<T> paths { rays.data(), ray_count, 0, offsets.data(), out.data(), starts.data(), finishes.data() };
            view.template trace_triangles<false, false>(0, motion, mn, rec, &cursor, sizeof cursor);
            view.template trace_paths<false>(0, motion, mn, paths, &cursor, sizeof cursor);
            const bool empty_ok = starts[0] == 0 && finishes[0] == 0 && out[0].ray_ok == 0;
            cu::MotionNodes<T> fewer = mn, null_nodes = mn;
            fewer.node_count -= 1;
            null_nodes.nodes = nullptr;
            cu::MotionTriangles<T> fewer_tris = motion;
            fewer_tris.count -= 1;
            View deep = view;
            deep.depth = 100000;
            int threw = 0;
            auto expect = [&](auto&& f, const char* name, bool length) {
                try { f(); } catch (const std::length_error& e) {
                    threw += length && std::string(e.what()).find(name) != std::string::npos;
                } catch (const std::invalid_argument& e) {
                    threw += !length && std::string(e.what()).find(name) != std::string::npos;
                }
            };
            const char* tt = "DeviceView::trace_triangles (motion nodes):";
            const char* tp = "DeviceView::trace_paths (motion nodes):";
            const char* pm = "prepare_motion_nodes:";
            expect([&] { view.template trace_triangles<false, false>(1, motion, fewer, rec, &cursor, sizeof cursor); }, tt, false);
            expect([&] { view.template trace_triangles<false, false>(1, motion, null_nodes, rec, &cursor, sizeof cursor); }, tt, false);
            expect([&] { view.template trace_triangles<false, false>(1, motion, mn, rec, &cursor, sizeof cursor - 1); }, tt, true);
            expect([&] { deep.template trace_triangles<false, false>(1, motion, mn, rec, &cursor, sizeof cursor); }, tt, true);
            expect([&] { view.template trace_paths<false>(1, motion, fewer, paths, &cursor, sizeof cursor); }, tp, false);
            expect([&] { view.template trace_paths<false>(1, motion, null_nodes, paths, &cursor, sizeof cursor); }, tp, false);
            expect([&] { view.template trace_paths<false>(1, motion, mn, paths, &cursor, sizeof cursor - 1); }, tp, true);
            expect([&] { deep.template trace_paths<false>(1, motion, mn, paths, &cursor, sizeof cursor); }, tp, true);
            std::vector<cu::MotionNode<T>> scratch(slots);
            expect([&] { cu::prepare_motion_nodes(view, fewer_tris, scratch.data(), workspace.data(), workspace.size()); }, pm, false);
            expect([&] { cu::prepare_motion_nodes(view, motion, (cu::MotionNode<T>*)nullptr, workspace.data(), workspace.size()); }, pm, false);
            expect([&] { cu::prepare_motion_nodes(view, motion, scratch.data(), workspace.data(), workspace.size() - 1); }, pm, true);
            std::printf("empty batch %s, errors thrown %d of 11\n", empty_ok ? "ok" : "CALLED", threw);
            if (!empty_ok || threw != 11) ++failures;
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
