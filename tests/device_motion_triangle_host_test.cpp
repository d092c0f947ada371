// tests/device_motion_triangle_host_test.cpp — the motion forms of DeviceView::trace_triangles and trace_paths,
// prepare_motion_triangles and triangle_at (include/bvh/v2/cuda/intersect.cuh) compiled as plain host C++, against the
// static trace_triangles on the same tree with the triangles set to triangle_at at the ray's time, and against the C++
// surface's Bvh<Node>::intersect with a PrecomputedTri(triangle_at(...))::intersect leaf.
//
//   device_motion_triangle_host_test <case file> f|d    one mesh and its rays, as tests/device_instance_trace_host_test.cpp
//                                                        reads them (written by tests/test_device_motion_triangle_host.py).
// The tree keeps the mesh's topology; its boxes are refitted here from prepare_motion_triangles' boxes.  Key pairs (key 0
// is the mesh): equal (one pointer twice), translate, rotscale (a turn and a scale about the mesh's centre), jitter (each
// vertex moved on its own), collapse (every third triangle degenerate at time 1), flip (p1 and p2 swapped at time 1, so
// the triangle turns over mid-shutter), offset (both keys moved to 1e4, with the rays), ulps (at 1e4, each coordinate
// of key 1 one to three ulps from key 0's) and non_finite (a NaN in key 0 and an infinity in key 1 of some triangles).
// Ray i has time time_of(i): 0, 1, 0.5, 0.3, a random time, -1, 2 and NaN.  Per key pair it checks:
//   * triangle_at at 0 and 1 gives the keys bit for bit;
//   * every box holds triangle_at at 65 uniform times, at adversarial ones (around 0.5, just below 1, the smallest
//     positive times) and at 1024 random times; it counts the vertices the union of the key boxes alone would miss
//     ("union misses": the rounding the widening is there for; the ulps pair has them, at random times only); a
//     non-finite key gives the empty box; every centre is tri_bounds_center's of triangle_at at 0.5; with equal keys box
//     and centre are tri_bounds_center's of the key bit for bit;
//   * for any-hit and closest-hit, both robust settings, both tie rules and three filters (accept all, reject odd ids, an
//     alpha cut-out), per ray: the accept-call count, a hash of the accept sequence (original id, bits of t, u, v) and the
//     record equal the static trace_triangles of that ray with the triangles at its time, and the surface's nested loop;
//   * for both robust settings, both tie rules and the three filters, scripted paths of 0 to 16 mixed segments at
//     time_of(i): per segment the same equality, and next receives the segment's ray bit for bit;
//   * n = 0 calls nothing; a wrong triangle count, a null key, a small workspace and a too-deep stack throw, naming the
//     motion call.
#include <bvh/v2/bvh.h>
#include <bvh/v2/cuda/intersect.cuh>
#include <bvh/v2/stack.h>
#include <bvh/v2/tri.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
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

// The recording shader: the motion form (start with a time) and the static oracle (start without: ray `first`, into
// out[0]), same records
template <typename T> struct Recorder {
    using Hit = typename cu::DeviceView<T>::Hit;
    struct Payload { uint32_t calls; uint64_t hash; };
    const T* rays;
    int filter;
    Out* out;
    size_t first;

    RayOf<T> start(size_t i, Payload& p, T& time) const { p.calls = 0; p.hash = kSeed; time = time_of<T>(i); return load_ray(rays + 8 * i); }
    RayOf<T> start(size_t i, Payload& p) const { p.calls = 0; p.hash = kSeed; return load_ray(rays + 8 * (first + i)); }
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

// The tree's boxes from per-primitive boxes (original order), children before parents: the same topology
template <typename T>
void refit(bvh::v2::Bvh<bvh::v2::Node<T, 3>>& bvh, const std::vector<typename cu::detail::ViewTypes<T>::BBox>& boxes, size_t i = 0) {
    auto& node = bvh.nodes[i];
    const T inf = std::numeric_limits<T>::infinity();
    for (int a = 0; a < 3; ++a) { node.bounds[2 * a] = inf; node.bounds[2 * a + 1] = -inf; }
    auto grow = [&](const T lo[3], const T hi[3]) {
        for (int a = 0; a < 3; ++a) {
            node.bounds[2 * a] = std::min(node.bounds[2 * a], lo[a]);
            node.bounds[2 * a + 1] = std::max(node.bounds[2 * a + 1], hi[a]);
        }
    };
    if (node.is_leaf()) {
        for (size_t k = node.index.first_id(); k < node.index.first_id() + node.index.prim_count(); ++k) {
            const auto& b = boxes[bvh.prim_ids[k]];
            const T lo[3] = { b.min.x, b.min.y, b.min.z }, hi[3] = { b.max.x, b.max.y, b.max.z };
            grow(lo, hi);
        }
        return;
    }
    for (size_t c = node.index.first_id(); c < node.index.first_id() + 2; ++c) {
        refit<T>(bvh, boxes, c);
        const auto& cb = bvh.nodes[c].bounds;
        const T lo[3] = { cb[0], cb[2], cb[4] }, hi[3] = { cb[1], cb[3], cb[5] };
        grow(lo, hi);
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
        std::vector<T> u1(k0);
        for (T& x : u1) {
            const uint32_t h = hash32((uint32_t)(&x - u1.data()) ^ 0x2545F491u);
            for (uint32_t q = 0; q < 1 + h % 3; ++q) x = std::nextafter(x, (h >> 8) & 1 ? std::numeric_limits<T>::infinity() : -std::numeric_limits<T>::infinity());
        }
        scenes.push_back({ "ulps", k0, u1, off, false });
    }
    {
        std::vector<T> k1 = moved([&](size_t, T* v) { for (int q = 0; q < 9; ++q) v[q] += (q % 3 == 1 ? step : T(0)); }), k0(mesh);
        for (size_t t = 0; t < prim_count; t += 7) {
            if ((t / 7) % 2 == 0) k0[9 * t + 4] = std::numeric_limits<T>::quiet_NaN();
            else k1[9 * t + 2] = std::numeric_limits<T>::infinity();
        }
        scenes.push_back({ "non_finite", k0, k1, T(0), false });
    }

    std::vector<size_t> offsets(kPaths + 1, 0);
    for (size_t i = 0; i < kPaths; ++i) offsets[i + 1] = offsets[i] + path_length(i);
    const size_t seg_count = offsets[kPaths];

    unsigned long long cursor = 0;
    int failures = 0;
    for (const Scene& scene : scenes) {
        std::vector<T> rays(base_rays);
        for (size_t i = 0; i < ray_count; ++i)
            for (int a = 0; a < 3; ++a) rays[8 * i + a] += scene.offset;
        const cu::MotionTriangles<T> motion { { scene.k0.data(), scene.same ? scene.k0.data() : scene.k1.data() }, prim_count };
        std::vector<BBox> boxes(prim_count);
        std::vector<VecC> centres(prim_count);
        cu::prepare_motion_triangles(motion, boxes.data(), centres.data());
        Bvh tree;
        tree.nodes = bvh.nodes;
        tree.prim_ids = bvh.prim_ids;
        refit<T>(tree, boxes);
        std::vector<bvhb200::DevNode<T>> dev_nodes(node_count + 1);
        std::memset(dev_nodes.data(), 0, dev_nodes.size() * sizeof(dev_nodes[0]));
        for (size_t i = 0; i < node_count; ++i) {
            for (int k = 0; k < 6; ++k) dev_nodes[i + 1].bounds[k] = tree.nodes[i].bounds[k];
            dev_nodes[i + 1].index = tree.nodes[i].index.value;
        }
        View view;                                      // no triangles: a tree over boxes
        view.nodes = dev_nodes.data(); view.prim_ids = ids32.data();
        view.node_count = node_count; view.prim_count = prim_count; view.depth = depth;

        // triangle_at at the keys, and the boxes over the shutter
        int key_bad = 0, box_bad = 0, empty = 0, static_bad = 0, centre_bad = 0, union_misses = 0;
        std::vector<T> times;
        for (int s = 0; s <= 64; ++s) times.push_back(T(s) / T(64));
        const T half = T(0.5), one = T(1), zero = T(0);
        for (T x : { std::nextafter(half, zero), std::nextafter(half, one), std::nextafter(one, zero), std::numeric_limits<T>::denorm_min(),
                     std::numeric_limits<T>::min(), std::numeric_limits<T>::epsilon(), T(1) / T(3), T(2) / T(3) })
            times.push_back(x);
        for (uint32_t s = 0; s < 1024; ++s)            // random times: the dyadic ones above blend without leaving the keys
            // (the division fills the mantissa below 2^-53 too, so that 1 - tau rounds in double as well as in float)
            times.push_back(T(T((((uint64_t)hash32(s ^ 0x68E31DA4u) << 32 | hash32(s)) >> 11) * T(1.0 / 9007199254740992.0)) / T(1.0009765625)));
        for (size_t t = 0; t < prim_count; ++t) {
            const T* k0 = &scene.k0[9 * t];
            const T* k1 = scene.same ? k0 : &scene.k1[9 * t];
            bool finite = true;
            for (int q = 0; q < 9; ++q) finite = finite && std::isfinite(k0[q]) && std::isfinite(k1[q]);
            T v[9];
            cu::triangle_at(motion, t, T(0), v);
            key_bad += std::memcmp(v, k0, sizeof v) != 0;
            cu::triangle_at(motion, t, T(1), v);
            key_bad += std::memcmp(v, k1, sizeof v) != 0;
            const BBox& b = boxes[t];
            if (!finite) {
                empty += b.min.x == std::numeric_limits<T>::infinity() && b.max.x == -std::numeric_limits<T>::infinity() &&
                         b.min.y == std::numeric_limits<T>::infinity() && b.max.z == -std::numeric_limits<T>::infinity();
                continue;
            }
            const T blo[3] = { b.min.x, b.min.y, b.min.z }, bhi[3] = { b.max.x, b.max.y, b.max.z };
            // the union of the key boxes without the widening: what the blend's rounding can leave
            T lo0[3], hi0[3], c0[3], lo1[3], hi1[3], c1[3], ulo[3], uhi[3];
            bvhb200::tri_bounds_center(k0, lo0, hi0, c0);
            bvhb200::tri_bounds_center(k1, lo1, hi1, c1);
            for (int a = 0; a < 3; ++a) { ulo[a] = std::min(lo0[a], lo1[a]); uhi[a] = std::max(hi0[a], hi1[a]); }
            for (T tau : times) {
                cu::triangle_at(motion, t, tau, v);
                for (int q = 0; q < 9; ++q) {
                    box_bad += !(blo[q % 3] <= v[q] && v[q] <= bhi[q % 3]);
                    union_misses += !(ulo[q % 3] <= v[q] && v[q] <= uhi[q % 3]);
                }
            }
            {   // the centre is tri_bounds_center's of the triangle at 0.5
                T mlo[3], mhi[3], mc[3];
                cu::triangle_at(motion, t, half, v);
                bvhb200::tri_bounds_center(v, mlo, mhi, mc);
                const T gc[3] = { centres[t].x, centres[t].y, centres[t].z };
                centre_bad += std::memcmp(mc, gc, sizeof mc) != 0;
            }
            if (scene.same) {
                T slo[3], shi[3], sc[3];
                bvhb200::tri_bounds_center(k0, slo, shi, sc);
                const T glo[3] = { b.min.x, b.min.y, b.min.z }, ghi[3] = { b.max.x, b.max.y, b.max.z };
                const T gc[3] = { centres[t].x, centres[t].y, centres[t].z };
                static_bad += std::memcmp(slo, glo, sizeof slo) != 0 || std::memcmp(shi, ghi, sizeof shi) != 0 || std::memcmp(sc, gc, sizeof sc) != 0;
            }
        }
        std::printf("scene %s keys mismatches %d box misses %d static box mismatches %d centre mismatches %d empty boxes %d union misses %d\n",
                    scene.name, key_bad, box_bad, static_bad, centre_bad, empty, union_misses);
        failures += key_bad + box_bad + static_bad + centre_bad;

        // the static triangles at each time the rays and paths use, BVH order
        std::map<uint64_t, std::vector<bvhb200::DevTri<T>>> at;
        auto tris_at = [&](T time) -> const bvhb200::DevTri<T>* {
            auto& tri = at[bits(time)];
            if (tri.empty()) {
                tri.resize(prim_count);
                for (size_t k = 0; k < prim_count; ++k) {
                    T v[9];
                    cu::triangle_at(motion, ids32[k], time, v);
                    tri[k] = bvhb200::precompute_tri(v);
                }
            }
            return tri.data();
        };
        // one ray through the surface's Bvh::intersect, whose leaf tests PrecomputedTri(triangle_at(...)) with the tie
        // rule and the filter
        auto surface = [&](int mode, int filter, const T* r, T time) {
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

        // rays: the motion call against the static call at each ray's time and the surface's nested loop
        for (int filter = 0; filter < kFilters; ++filter) {
            for (int mode = 0; mode < 8; ++mode) {
                std::vector<Out> got(ray_count), want(ray_count);
                std::memset(got.data(), 0, got.size() * sizeof(Out));
                std::memset(want.data(), 0, want.size() * sizeof(Out));
                by_mode(mode, [&](auto any, auto rob, auto lst) {
                    constexpr bool A = decltype(any)::value, Rb = decltype(rob)::value, L = decltype(lst)::value;
                    view.template trace_triangles<A, Rb, L>(ray_count, motion, Recorder<T> { rays.data(), filter, got.data(), 0 }, &cursor,
                                                            sizeof cursor);
                    for (size_t i = 0; i < ray_count; ++i) {
                        View st = view;
                        st.tris = tris_at(time_of<T>(i));
                        st.template trace_triangles<A, Rb, L>(1, Recorder<T> { rays.data(), filter, want.data() + i, i }, &cursor, sizeof cursor);
                    }
                });
                int bad = 0, surf_bad = 0, hits = 0;
                uint64_t calls = 0;
                for (size_t i = 0; i < ray_count; ++i) {
                    hits += got[i].id != (sizeof(T) == 4 ? 0xFFFFFFFFull : ~0ull);
                    calls += got[i].calls;
                    const Out s = surface(mode, filter, &rays[8 * i], time_of<T>(i));
                    const bool b1 = std::memcmp(&got[i], &want[i], sizeof(Out)) != 0, b2 = std::memcmp(&got[i], &s, sizeof(Out)) != 0;
                    if ((b1 || b2) && bad + surf_bad < 3)
                        std::printf("  %s ray %zu: calls %u/%u/%u id %llu/%llu/%llu\n", scene.name, i, got[i].calls, want[i].calls, s.calls,
                                    (unsigned long long)got[i].id, (unsigned long long)want[i].id, (unsigned long long)s.id);
                    bad += b1;
                    surf_bad += b2;
                }
                std::printf("rays %s filter %d mode %d mismatches %d surface mismatches %d hits %d accept calls %llu\n", scene.name, filter,
                            mode, bad, surf_bad, hits, (unsigned long long)calls);
                failures += bad + surf_bad;
            }
        }

        // paths: each segment against the static call and the surface's loop for its ray at the path's time
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
                    view.template trace_paths<Rb, L>(kPaths, motion, shader, &cursor, sizeof cursor);
                    for (size_t i = 0; i < kPaths; ++i) {
                        View st = view;
                        st.tris = tris_at(time_of<T>(i));
                        for (size_t j = 0; j < path_length(i); ++j) {
                            const uint32_t h = segment_hash(i, j);
                            Out* w = want.data() + offsets[i] + j;
                            const Recorder<T> r { rays.data(), filter, w, h % ray_count };
                            if (h >> 31) st.template trace_triangles<true, Rb, L>(1, r, &cursor, sizeof cursor);
                            else st.template trace_triangles<false, Rb, L>(1, r, &cursor, sizeof cursor);
                            const Out s = surface(((h >> 31) ? 1 : 0) | (mode << 1), filter, &rays[8 * (h % ray_count)], time_of<T>(i));
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
            // n = 0 calls nothing; a triangle count other than the tree's, a null key, a small workspace or a stack beyond
            // 200 KB throw
            std::vector<Out> out(ray_count);
            const Recorder<T> rec { rays.data(), 0, out.data(), 0 };
            std::vector<uint32_t> starts(kPaths), finishes(kPaths);
            const PathRecorder<T> paths { rays.data(), ray_count, 0, offsets.data(), out.data(), starts.data(), finishes.data() };
            view.template trace_triangles<false, false>(0, motion, rec, &cursor, sizeof cursor);
            view.template trace_paths<false>(0, motion, paths, &cursor, sizeof cursor);
            const bool empty_ok = starts[0] == 0 && finishes[0] == 0 && out[0].ray_ok == 0;
            cu::MotionTriangles<T> fewer = motion, null_key = motion;
            fewer.count -= 1;
            null_key.vertices[1] = nullptr;
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
            const char* tt = "DeviceView::trace_triangles (motion):";
            const char* tp = "DeviceView::trace_paths (motion):";
            expect([&] { view.template trace_triangles<false, false>(1, fewer, rec, &cursor, sizeof cursor); }, tt, false);
            expect([&] { view.template trace_triangles<false, false>(1, null_key, rec, &cursor, sizeof cursor); }, tt, false);
            expect([&] { view.template trace_triangles<false, false>(1, motion, rec, &cursor, sizeof cursor - 1); }, tt, true);
            expect([&] { deep.template trace_triangles<false, false>(1, motion, rec, &cursor, sizeof cursor); }, tt, true);
            expect([&] { view.template trace_paths<false>(1, fewer, paths, &cursor, sizeof cursor); }, tp, false);
            expect([&] { view.template trace_paths<false>(1, null_key, paths, &cursor, sizeof cursor); }, tp, false);
            expect([&] { view.template trace_paths<false>(1, motion, paths, &cursor, sizeof cursor - 1); }, tp, true);
            expect([&] { deep.template trace_paths<false>(1, motion, paths, &cursor, sizeof cursor); }, tp, true);
            std::printf("empty batch %s, errors thrown %d of 8\n", empty_ok ? "ok" : "CALLED", threw);
            if (!empty_ok || threw != 8) ++failures;
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
