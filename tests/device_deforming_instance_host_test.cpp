// tests/device_deforming_instance_host_test.cpp — the deforming forms of DeviceView::trace_instances and
// trace_instance_paths, make_deforming_instance and prepare_deforming_instances (include/bvh/v2/cuda/intersect.cuh)
// compiled as plain host C++.
//
//   device_deforming_instance_host_test <case file> f|d    one mesh and its rays, as tests/device_instance_trace_host_test.cpp
//                                                           reads them (written by tests/test_device_deforming_instance_host.py).
// The mesh's golden tree is the static bottom; the same topology refitted over prepare_motion_triangles' boxes is the
// shutter-box bottom, and prepare_motion_nodes gives its motion nodes.  Key pairs: equal, jitter (about a triangle's
// size), ulps (the mesh at 1e4, keys one to three ulps apart), non_finite (a NaN and an infinite key) and partial (half
// the mesh static).  Ray i has time time_of(i): 0, 1, 0.5, 0.3, a random time, -1, 2 and NaN.  Per key pair it checks,
// for any-hit and closest-hit, both robust settings, both tie rules and three filters, per ray (accept-call count, a
// hash of the accept sequence, the record and its instance):
//   * a scene of every bottom kind under moving placements (one singular at time 0): the static bottoms only equal the
//     motion trace_instances over the same fields;
//   * one identity record with equal placement keys equals the motion trace_triangles (shutter boxes) or the
//     motion-node trace_triangles on the mesh, and for equal vertex keys every kind equals the static bottom;
//   * scripted paths at time_of(i): each segment equals trace_instances of its world ray, and next gets that ray;
//   * two copies of a deforming mesh at one place tie to the lower instance (closest-hit, canonical rule);
//   * containment at 65 uniform, adversarial and 1024 full-mantissa random times: every world box holds every finite
//     vertex blended by triangle_at and moved by instance_at's rounded placement (in long double); and, in object
//     space, every blended finite vertex lies in its leaf's motion-node keys unioned and in the root's two key boxes
//     unioned (the bottom box B of prepare_deforming_instance), while for the ulps pair some lie outside the same leaf
//     boxes recomputed without the widening ("unwidened misses"), so a removed widening fails the leaf check;
//   * make_deforming_instance (counts, null pointers, a static bottom without triangles) and the calls throw as documented, naming "trace_instances (deforming)" and
//     "trace_instance_paths (deforming)".
#include <bvh/v2/bvh.h>
#include <bvh/v2/cuda/intersect.cuh>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <limits>
#include <stdexcept>
#include <string>
#include <vector>

namespace {

namespace cu = bvh::v2::cuda;
using cu::PathStep;

uint64_t mix(uint64_t h, uint64_t x) { return (h ^ x) * 1099511628211ull; }
constexpr uint64_t kSeed = 1469598103934665603ull;
constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr size_t kPaths = 64;

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
size_t path_length(size_t i) { return i == 0 ? 0 : hash32((uint32_t)i) % 9; }
uint32_t segment_hash(size_t i, size_t j) { return hash32((uint32_t)(i * 977 + j) ^ 0x5bd1e995u); }

bool keep(int filter, uint32_t inst, size_t id) {
    if (filter == 1) return (id & 1) == 0;
    if (filter == 2) return (inst & 1) == 0;
    return true;
}

struct Out { uint64_t id, t, u, v; uint32_t inst, calls; uint64_t hash; uint32_t ray_ok, pad; };

template <typename T> struct Recorder {
    using Ray = typename cu::DeviceView<T>::Ray;
    using Hit = typename cu::DeviceView<T>::Hit;
    struct Payload { uint32_t calls; uint64_t hash; };
    const T* rays;
    int filter;
    Out* out;
    size_t first;                       // ray first + i
    size_t time_index;                  // SIZE_MAX: the ray's own

    Ray start(size_t i, Payload& p, T& time) const {
        p.calls = 0; p.hash = kSeed;
        time = time_of<T>(time_index != SIZE_MAX ? time_index : first + i);
        const T* r = rays + 8 * (first + i);
        Ray x;
        x.org.x = r[0]; x.org.y = r[1]; x.org.z = r[2]; x.dir.x = r[3]; x.dir.y = r[4]; x.dir.z = r[5]; x.tmin = r[6]; x.tmax = r[7];
        return x;
    }
    bool accept(Payload& p, uint32_t inst, size_t id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(mix(p.hash, inst), id), bits(t)), bits(u)), bits(v));
        return keep(filter, inst, id);
    }
    bool accept(Payload& p, size_t id, T t, T u, T v) const { return accept(p, 0u, id, t, u, v); }
    void finish(size_t i, const Payload& p, const Hit& hit, uint32_t inst) const {
        Out& o = out[i];
        o.id = hit.prim_id; o.t = bits(hit.t); o.u = bits(hit.u); o.v = bits(hit.v);
        o.inst = inst; o.calls = p.calls; o.hash = p.hash; o.ray_ok = 1;
    }
    void finish(size_t i, const Payload& p, const Hit& hit) const { finish(i, p, hit, (uint32_t)hit.prim_id == kNone ? kNone : 0u); }
};

template <typename T> struct PathRecorder {
    using Ray = typename cu::DeviceView<T>::Ray;
    using Hit = typename cu::DeviceView<T>::Hit;
    struct Payload { size_t seg; uint32_t calls; uint64_t hash; };
    const T* rays;
    size_t ray_count;
    int filter;
    const size_t* offsets;
    Out* segs;
    uint32_t* finishes;

    PathStep segment(size_t i, size_t j, Ray& ray) const {
        const uint32_t h = segment_hash(i, j);
        const T* r = rays + 8 * (h % ray_count);
        ray.org.x = r[0]; ray.org.y = r[1]; ray.org.z = r[2]; ray.dir.x = r[3]; ray.dir.y = r[4]; ray.dir.z = r[5];
        ray.tmin = r[6]; ray.tmax = r[7];
        return (h >> 31) ? PathStep::Occlusion : PathStep::Closest;
    }
    PathStep start(size_t i, Payload& p, Ray& ray, T& time) const {
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

template <typename T> struct Key { T m[12]; };
template <typename T> Key<T> place(T angle, T scale, T sx, T sy, T sz) {      // rotation about z, scale, shift
    const T c = std::cos(angle) * scale, s = std::sin(angle) * scale;
    return Key<T> { { c, -s, 0, sx, s, c, 0, sy, 0, 0, scale, sz } };
}

int compare(const std::vector<Out>& got, const std::vector<Out>& want) {
    int bad = 0;
    for (size_t i = 0; i < got.size(); ++i) bad += std::memcmp(&got[i], &want[i], sizeof(Out)) != 0;
    return bad;
}

template <typename T>
int run(std::ifstream& in) {
    using Node = bvh::v2::Node<T, 3>;
    using View = cu::DeviceView<T>;
    using BBox = typename cu::detail::ViewTypes<T>::BBox;
    using VecC = typename cu::detail::ViewTypes<T>::Vec;
    uint64_t mesh_count = 0, node_count = 0, prim_count = 0, ray_count = 0;
    in.read((char*)&mesh_count, 8);
    in.read((char*)&node_count, 8); in.read((char*)&prim_count, 8);
    bvh::v2::Bvh<Node> bvh;
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

    T lo[3], hi[3];
    for (int a = 0; a < 3; ++a) lo[a] = hi[a] = mesh[a];
    for (size_t k = 0; k < mesh.size(); ++k) { lo[k % 3] = std::min(lo[k % 3], mesh[k]); hi[k % 3] = std::max(hi[k % 3], mesh[k]); }
    const T size = std::max({ hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2], T(1e-3) });
    const T step = size / T(2 * std::cbrt((double)prim_count + 1));
    uint64_t seed = 777;
    auto rnd = [&] { seed = seed * 6364136223846793005ull + 1442695040888963407ull; return T((seed >> 11) * (1.0 / 9007199254740992.0)); };

    struct Pair { const char* name; std::vector<T> k0, k1; T offset; };
    std::vector<Pair> pairs;
    pairs.push_back({ "equal", mesh, mesh, T(0) });
    {
        std::vector<T> k1(mesh);
        for (T& x : k1) x += (rnd() - T(0.5)) * step;
        pairs.push_back({ "jitter", mesh, k1, T(0) });
    }
    {
        std::vector<T> k0(mesh), k1(mesh);
        for (size_t k = 0; k < mesh.size(); ++k) {
            k0[k] = mesh[k] + T(1e4);
            k1[k] = k0[k];
            for (int u = 1 + (int)(hash32((uint32_t)k) % 3); u > 0; --u) k1[k] = std::nextafter(k1[k], std::numeric_limits<T>::infinity());
        }
        pairs.push_back({ "ulps", k0, k1, T(1e4) });
    }
    {
        std::vector<T> k1(mesh);
        for (T& x : k1) x += (rnd() - T(0.5)) * step;
        std::vector<T> k0(mesh);
        k0[4] = std::numeric_limits<T>::quiet_NaN();
        if (prim_count > 1) k1[9 + 2] = std::numeric_limits<T>::infinity();
        pairs.push_back({ "non_finite", k0, k1, T(0) });
    }
    {
        std::vector<T> k1(mesh);
        for (size_t t = prim_count / 2; t < prim_count; ++t)
            for (int q = 0; q < 9; ++q) k1[9 * t + q] += (q % 3 == 0 ? step : T(0));
        pairs.push_back({ "partial", mesh, k1, T(0) });
    }

    std::vector<size_t> offsets(kPaths + 1, 0);
    for (size_t i = 0; i < kPaths; ++i) offsets[i + 1] = offsets[i] + path_length(i);
    const size_t seg_count = offsets[kPaths];
    unsigned long long cursor = 0;
    int failures = 0;

    for (const Pair& pair : pairs) {
        const T off = pair.offset;
        std::vector<T> verts0(pair.k0);                  // the static bottom: key 0 (finite entries only matter)
        for (T& x : verts0) if (!std::isfinite(x)) x = T(0);
        std::vector<T> rays(base_rays);
        for (size_t i = 0; i < ray_count; ++i)
            for (int a = 0; a < 3; ++a) rays[8 * i + a] += off;
        // static bottom: the golden topology refitted over key 0's triangles, with its triangles
        std::vector<bvhb200::DevNode<T>> snodes(node_count + 1), dnodes(node_count + 1);
        for (size_t i = 0; i < node_count; ++i) snodes[i + 1].index = dnodes[i + 1].index = bvh.nodes[i].index.value;
        std::vector<uint32_t> parent(node_count + 1);
        std::vector<int> flags(node_count + 1);
        const cu::MotionTriangles<T> still { { verts0.data(), verts0.data() }, prim_count }, moving { { pair.k0.data(), pair.k1.data() }, prim_count };
        auto refit = [&](std::vector<bvhb200::DevNode<T>>& nodes, const cu::MotionTriangles<T>& keys) {
            std::vector<BBox> boxes(prim_count);
            std::vector<VecC> centres(prim_count);
            cu::prepare_motion_triangles(keys, boxes.data(), centres.data());
            std::fill(parent.begin(), parent.end(), 0u);
            std::fill(flags.begin(), flags.end(), 0);
            for (size_t i = 1; i <= node_count; ++i) bvhb200::refit_link(nodes.data(), node_count + 1, i, parent.data(), flags.data());
            for (size_t i = node_count + 1; i-- > 1;)
                bvhb200::refit_from_leaf<T>(nodes.data(), i, parent.data(), flags.data(), ids32.data(),
                                            bvhb200::BoxSource<T> { reinterpret_cast<const T*>(boxes.data()) });
        };
        refit(snodes, still);
        refit(dnodes, moving);
        std::vector<bvhb200::DevTri<T>> stris(prim_count);
        for (size_t k = 0; k < prim_count; ++k) stris[k] = bvhb200::precompute_tri(&verts0[9 * ids[k]]);
        View sview, dview;
        sview.nodes = snodes.data(); sview.prim_ids = ids32.data(); sview.tris = stris.data();
        sview.node_count = node_count; sview.prim_count = prim_count; sview.depth = depth;
        dview = sview;
        dview.nodes = dnodes.data(); dview.tris = nullptr;
        std::vector<cu::MotionNode<T>> mnodes(node_count + 1);
        std::vector<uint32_t> ws(2 * (node_count + 1));
        cu::prepare_motion_nodes(dview, moving, mnodes.data(), ws.data(), ws.size() * 4);
        const cu::MotionNodes<T> mn { mnodes.data(), node_count };

        // a scene of every kind under moving placements; record 4's placement is singular at time 0
        std::vector<cu::DeformingInstance<T>> recs;
        std::vector<cu::MotionInstance<T>> motion;
        for (int k = 0; k < 9; ++k) {
            const T sx = off + T(k % 3 - 1) * size * T(1.2), sy = off + T(k / 3 - 1) * size * T(1.2);
            Key<T> a = place<T>(T(0.3) * T(k), T(k % 2 ? 0.5 : 1), sx - off, sy - off, T(0));
            Key<T> b = place<T>(T(0.3) * T(k) + T(0.2), T(k % 2 ? 0.5 : 1), sx - off + step, sy - off, step);
            for (int row = 0; row < 3; ++row) {                  // about the mesh's offset
                a.m[4 * row + 3] += off - (a.m[4 * row] + a.m[4 * row + 1] + a.m[4 * row + 2]) * off;
                b.m[4 * row + 3] += off - (b.m[4 * row] + b.m[4 * row + 1] + b.m[4 * row + 2]) * off;
            }
            if (k == 4) for (int q : { 0, 1, 2, 4, 5, 6, 8, 9, 10 }) a.m[q] = T(0);
            const int kind = k % 3;
            recs.push_back(kind == 0 ? cu::make_deforming_instance(sview, a.m, b.m)
                           : kind == 1 ? cu::make_deforming_instance(dview, a.m, b.m, moving)
                                       : cu::make_deforming_instance(dview, a.m, b.m, moving, mn));
        }
        auto top_of = [&](std::vector<cu::DeformingInstance<T>>& r, std::vector<bvhb200::DevNode<T>>& tn, std::vector<uint32_t>& tid,
                          std::vector<BBox>& boxes) {
            const size_t n = r.size();
            boxes.resize(n);
            std::vector<VecC> centres(n);
            cu::prepare_deforming_instances(cu::DeformingInstances<T> { r.data(), n, depth }, boxes.data(), centres.data());
            // a top tree of one leaf over all records
            tn.assign(2, bvhb200::DevNode<T> {});
            const T inf = std::numeric_limits<T>::infinity();
            T* b = tn[1].bounds;
            b[0] = b[2] = b[4] = inf; b[1] = b[3] = b[5] = -inf;
            for (const BBox& x : boxes) {
                b[0] = std::min(b[0], x.min.x); b[2] = std::min(b[2], x.min.y); b[4] = std::min(b[4], x.min.z);
                b[1] = std::max(b[1], x.max.x); b[3] = std::max(b[3], x.max.y); b[5] = std::max(b[5], x.max.z);
            }
            tn[1].index = bvhb200::make_index<typename View::Index>(0, (uint32_t)n);
            tid.resize(n);
            for (size_t k = 0; k < n; ++k) tid[k] = (uint32_t)k;
            View top;
            top.nodes = tn.data(); top.prim_ids = tid.data(); top.node_count = 1; top.prim_count = n; top.depth = 0;
            return top;
        };
        std::vector<bvhb200::DevNode<T>> tn;
        std::vector<uint32_t> tid;
        std::vector<BBox> boxes;
        // (a top leaf holds at most 15 records: 9 here)
        const View top = top_of(recs, tn, tid, boxes);
        const cu::DeformingInstances<T> inst { recs.data(), recs.size(), depth };

        // containment, at 65 uniform, adversarial and 1024 random full-mantissa times
        int box_bad = 0, plain = 0;
        std::vector<T> times;
        for (int s = 0; s <= 64; ++s) times.push_back(T(s) / T(64));
        for (T t : { T(0.5), std::nextafter(T(0.5), T(0)), std::nextafter(T(0.5), T(1)), std::nextafter(T(1), T(0)),
                     std::numeric_limits<T>::denorm_min(), std::numeric_limits<T>::min() }) times.push_back(t);
        for (int s = 0; s < 1024; ++s) times.push_back(T(rnd() * T(0.999)));
        for (size_t k = 0; k < recs.size(); ++k) {
            const cu::DeformingInstance<T>& r = recs[k];
            const BBox& b = boxes[k];
            const T blo[3] = { b.min.x, b.min.y, b.min.z }, bhi[3] = { b.max.x, b.max.y, b.max.z };
            for (T tau : times) {
                const cu::Instance<T> at = cu::instance_at(r, tau);
                for (size_t id = 0; id < prim_count; ++id) {
                    T v[9];
                    bool finite = true;
                    for (int q = 0; q < 9; ++q) finite = finite && std::isfinite(pair.k0[9 * id + q]) && std::isfinite(pair.k1[9 * id + q]);
                    if (!finite) continue;
                    if (r.vertices[0]) cu::triangle_at(moving, id, tau, v);
                    else std::memcpy(v, &verts0[9 * id], sizeof v);
                    for (int p = 0; p < 3; ++p) {
                        if (r.vertices[0])
                            for (int a = 0; a < 3; ++a) {
                                const T c0 = pair.k0[9 * id + 3 * p + a], c1 = pair.k1[9 * id + 3 * p + a];
                                plain += v[3 * p + a] < std::min(c0, c1) || v[3 * p + a] > std::max(c0, c1);
                            }
                        for (int a = 0; a < 3; ++a) {
                            const T* row = at.object_to_world + 4 * a;
                            const long double x = (long double)row[0] * v[3 * p] + (long double)row[1] * v[3 * p + 1] +
                                                  (long double)row[2] * v[3 * p + 2] + row[3];
                            box_bad += !((long double)blo[a] <= x && x <= (long double)bhi[a]);
                        }
                    }
                }
            }
        }
        std::printf("pair %s box misses %d plain misses %d\n", pair.name, box_bad, plain);
        failures += box_bad;

        // the object-space bottom boxes the world boxes rest on, checked directly (the world box's own widening would
        // hide an ulp): triangle_at of every finite triangle against (a) its leaf's motion-node keys, unioned, (b) the
        // root's two key boxes unioned, the bottom box B of prepare_deforming_instance, and (c) the same leaf boxes
        // recomputed from the keys without the widening, which the blend must leave for the widening to matter
        int leaf_bad = 0, root_bad = 0, unwidened = 0;
        {
            std::vector<size_t> leaf_of(prim_count, 0);
            for (size_t slot = 1; slot <= node_count; ++slot) {
                const auto index = dnodes[slot].index;
                if (bvhb200::index_count(index) == 0) continue;
                for (size_t q = bvhb200::index_first(index); q < bvhb200::index_first(index) + bvhb200::index_count(index); ++q)
                    leaf_of[ids32[q]] = slot;
            }
            auto key_union = [&](size_t slot, T lo_[3], T hi_[3]) {
                const cu::MotionNode<T>& m = mnodes[slot];
                for (int a = 0; a < 2; ++a) {
                    lo_[a] = std::min(m.xy[0][2 * a], m.xy[1][2 * a]);
                    hi_[a] = std::max(m.xy[0][2 * a + 1], m.xy[1][2 * a + 1]);
                }
                lo_[2] = std::min(m.z[0][0], m.z[1][0]);
                hi_[2] = std::max(m.z[0][1], m.z[1][1]);
            };
            const T inf = std::numeric_limits<T>::infinity();
            std::vector<T> plo(3 * (node_count + 1), inf), phi(3 * (node_count + 1), -inf);     // unwidened leaf unions
            auto finite_tri = [&](size_t id) {
                for (int q = 0; q < 9; ++q)
                    if (!std::isfinite(pair.k0[9 * id + q]) || !std::isfinite(pair.k1[9 * id + q])) return false;
                return true;
            };
            for (size_t id = 0; id < prim_count; ++id) {
                if (!finite_tri(id)) continue;
                for (int q = 0; q < 9; ++q) {
                    T* l = &plo[3 * leaf_of[id] + q % 3];
                    T* h = &phi[3 * leaf_of[id] + q % 3];
                    *l = std::min({ *l, pair.k0[9 * id + q], pair.k1[9 * id + q] });
                    *h = std::max({ *h, pair.k0[9 * id + q], pair.k1[9 * id + q] });
                }
            }
            T rlo[3], rhi[3];
            key_union(1, rlo, rhi);
            for (T tau : times)
                for (size_t id = 0; id < prim_count; ++id) {
                    if (!finite_tri(id)) continue;
                    T v[9], llo[3], lhi[3];
                    cu::triangle_at(moving, id, tau, v);
                    key_union(leaf_of[id], llo, lhi);
                    for (int q = 0; q < 9; ++q) {
                        const int a = q % 3;
                        leaf_bad += v[q] < llo[a] || v[q] > lhi[a];
                        root_bad += v[q] < rlo[a] || v[q] > rhi[a];
                        unwidened += v[q] < plo[3 * leaf_of[id] + a] || v[q] > phi[3 * leaf_of[id] + a];
                    }
                }
        }
        std::printf("pair %s leaf misses %d root misses %d unwidened misses %d\n", pair.name, leaf_bad, root_bad, unwidened);
        failures += leaf_bad + root_bad;

        for (int filter = 0; filter < 3; ++filter)
            for (int mode = 0; mode < 8; ++mode) {
                int bad_static = 0, bad_ident = 0, bad_equal = 0, hits = 0;
                by_mode(mode, [&](auto any, auto rob, auto lst) {
                    constexpr bool A = decltype(any)::value, Rb = decltype(rob)::value, L = decltype(lst)::value;
                    std::vector<Out> got(ray_count), want(ray_count);
                    auto fresh = [&] { std::memset(got.data(), 0, got.size() * sizeof(Out)); std::memset(want.data(), 0, want.size() * sizeof(Out)); };
                    // the whole scene, for the hit count
                    fresh();
                    top.template trace_instances<A, Rb, L>(ray_count, inst, Recorder<T> { rays.data(), filter, got.data(), 0, SIZE_MAX }, &cursor, sizeof cursor);
                    for (const Out& o : got) hits += o.inst != kNone;
                    // static bottoms only: the motion trace_instances
                    std::vector<cu::DeformingInstance<T>> st(recs);
                    std::vector<cu::MotionInstance<T>> mo(recs.size());
                    for (size_t k = 0; k < st.size(); ++k) {
                        st[k] = cu::make_deforming_instance(sview, recs[k].object_to_world[0], recs[k].object_to_world[1]);
                        mo[k] = cu::make_motion_instance(sview, recs[k].object_to_world[0], recs[k].object_to_world[1]);
                    }
                    std::vector<BBox> bx(st.size());
                    std::vector<VecC> cx(st.size());
                    cu::prepare_deforming_instances(cu::DeformingInstances<T> { st.data(), st.size(), depth }, bx.data(), cx.data());
                    cu::prepare_motion_instances(cu::MotionInstances<T> { mo.data(), mo.size(), depth }, bx.data(), cx.data());
                    fresh();
                    top.template trace_instances<A, Rb, L>(ray_count, cu::DeformingInstances<T> { st.data(), st.size(), depth },
                                                           Recorder<T> { rays.data(), filter, got.data(), 0, SIZE_MAX }, &cursor, sizeof cursor);
                    top.template trace_instances<A, Rb, L>(ray_count, cu::MotionInstances<T> { mo.data(), mo.size(), depth },
                                                           Recorder<T> { rays.data(), filter, want.data(), 0, SIZE_MAX }, &cursor, sizeof cursor);
                    bad_static += compare(got, want);
                    // one identity record: the motion (node) trace_triangles on the mesh
                    const T id12[12] = { 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0 };
                    for (int kind = 1; kind < 3; ++kind) {
                        std::vector<cu::DeformingInstance<T>> one { kind == 1 ? cu::make_deforming_instance(dview, id12, id12, moving)
                                                                              : cu::make_deforming_instance(dview, id12, id12, moving, mn) };
                        std::vector<bvhb200::DevNode<T>> otn;
                        std::vector<uint32_t> otid;
                        std::vector<BBox> ob;
                        const View otop = top_of(one, otn, otid, ob);
                        fresh();
                        otop.template trace_instances<A, Rb, L>(ray_count, cu::DeformingInstances<T> { one.data(), 1, depth },
                                                                Recorder<T> { rays.data(), filter, got.data(), 0, SIZE_MAX }, &cursor, sizeof cursor);
                        if (kind == 1) dview.template trace_triangles<A, Rb, L>(ray_count, moving, Recorder<T> { rays.data(), filter, want.data(), 0, SIZE_MAX },
                                                                                 &cursor, sizeof cursor);
                        else dview.template trace_triangles<A, Rb, L>(ray_count, moving, mn, Recorder<T> { rays.data(), filter, want.data(), 0, SIZE_MAX },
                                                                       &cursor, sizeof cursor);
                        bad_ident += compare(got, want);
                    }
                    // equal vertex keys: every kind is the static bottom on the same tree (the equal pair's trees are one)
                    if (std::string(pair.name) == "equal") {
                        std::vector<cu::DeformingInstance<T>> eq(recs);
                        for (size_t k = 0; k < eq.size(); ++k) {
                            eq[k] = cu::make_deforming_instance(sview, recs[k].object_to_world[0], recs[k].object_to_world[1]);
                            if (k % 3) { eq[k].vertices[0] = pair.k0.data(); eq[k].vertices[1] = pair.k1.data(); }
                            if (k % 3 == 2) eq[k].motion_nodes = mnodes.data();
                        }
                        std::vector<BBox> eb(eq.size());
                        std::vector<VecC> ec(eq.size());
                        cu::prepare_deforming_instances(cu::DeformingInstances<T> { eq.data(), eq.size(), depth }, eb.data(), ec.data());
                        fresh();
                        top.template trace_instances<A, Rb, L>(ray_count, cu::DeformingInstances<T> { eq.data(), eq.size(), depth },
                                                               Recorder<T> { rays.data(), filter, got.data(), 0, SIZE_MAX }, &cursor, sizeof cursor);
                        top.template trace_instances<A, Rb, L>(ray_count, cu::DeformingInstances<T> { st.data(), st.size(), depth },
                                                               Recorder<T> { rays.data(), filter, want.data(), 0, SIZE_MAX }, &cursor, sizeof cursor);
                        bad_equal += compare(got, want);
                        bad_equal += std::memcmp(eb.data(), bx.data(), eb.size() * sizeof(BBox)) != 0;
                    }
                });
                std::printf("rays %s filter %d mode %d static %d identity %d equal %d hits %d\n", pair.name, filter, mode, bad_static, bad_ident,
                            bad_equal, hits);
                failures += bad_static + bad_ident + bad_equal;
            }

        // paths: each segment against trace_instances of its world ray at the path's time
        for (int mode = 0; mode < 4; ++mode) {
            std::vector<Out> segs(seg_count + 1), want(seg_count + 1);
            std::memset(segs.data(), 0, segs.size() * sizeof(Out));
            std::memset(want.data(), 0, want.size() * sizeof(Out));
            std::vector<uint32_t> finishes(kPaths);
            int bad = 0;
            by_mode(mode << 1, [&](auto, auto rob, auto lst) {
                constexpr bool Rb = decltype(rob)::value, L = decltype(lst)::value;
                top.template trace_instance_paths<Rb, L>(kPaths, inst, PathRecorder<T> { rays.data(), ray_count, 0, offsets.data(), segs.data(), finishes.data() },
                                                         &cursor, sizeof cursor);
                for (size_t i = 0; i < kPaths; ++i)
                    for (size_t j = 0; j < path_length(i); ++j) {
                        const uint32_t h = segment_hash(i, j);
                        const Recorder<T> r { rays.data(), 0, want.data() + offsets[i] + j, h % ray_count, i };
                        if (h >> 31) top.template trace_instances<true, Rb, L>(1, inst, r, &cursor, sizeof cursor);
                        else top.template trace_instances<false, Rb, L>(1, inst, r, &cursor, sizeof cursor);
                    }
            });
            bad += compare(segs, want);
            for (uint32_t f : finishes) bad += f != 1;
            std::printf("paths %s mode %d segments %zu mismatches %d\n", pair.name, mode, seg_count, bad);
            failures += bad;
        }

        // two copies of the deforming mesh at one place: ties go to the lower instance
        if (std::string(pair.name) == "jitter") {
            const T id12[12] = { 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0 };
            std::vector<cu::DeformingInstance<T>> two { cu::make_deforming_instance(dview, id12, id12, moving, mn),
                                                        cu::make_deforming_instance(dview, id12, id12, moving, mn) };
            std::vector<bvhb200::DevNode<T>> otn;
            std::vector<uint32_t> otid;
            std::vector<BBox> ob;
            const View otop = top_of(two, otn, otid, ob);
            std::vector<Out> got(ray_count);
            otop.template trace_instances<false, true>(ray_count, cu::DeformingInstances<T> { two.data(), 2, depth },
                                                       Recorder<T> { rays.data(), 0, got.data(), 0, SIZE_MAX }, &cursor, sizeof cursor);
            int ties = 0, upper = 0;
            for (const Out& o : got) { ties += o.inst != kNone; upper += o.inst == 1; }
            std::printf("pair copies hits %d upper %d\n", ties, upper);
            failures += upper;
        }

        if (std::string(pair.name) == "jitter") {
            // errors: make_deforming_instance's counts and null pointers, the calls' record count, workspace and stack
            int threw = 0;
            const T id12[12] = { 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0 };
            auto expect = [&](auto&& f, const char* name, int kind) {
                try { f(); } catch (const std::length_error& e) {
                    threw += kind == 2 && std::string(e.what()).find(name) != std::string::npos;
                } catch (const std::invalid_argument& e) {
                    threw += kind == 1 && std::string(e.what()).find(name) != std::string::npos;
                }
            };
            const cu::MotionTriangles<T> fewer { { pair.k0.data(), pair.k1.data() }, prim_count - 1 }, null_keys { { nullptr, nullptr }, prim_count };
            const cu::MotionNodes<T> fewer_nodes { mnodes.data(), node_count + 1 }, null_nodes { nullptr, node_count };
            const char* mk = "make_deforming_instance";
            expect([&] { cu::make_deforming_instance(dview, id12, id12, fewer); }, mk, 1);
            expect([&] { cu::make_deforming_instance(dview, id12, id12, null_keys); }, mk, 1);
            expect([&] { cu::make_deforming_instance(dview, id12, id12, moving, fewer_nodes); }, mk, 1);
            expect([&] { cu::make_deforming_instance(dview, id12, id12, moving, null_nodes); }, mk, 1);
            expect([&] { cu::make_deforming_instance(dview, id12, id12); }, mk, 1);       // a static bottom without triangles
            std::vector<Out> out(ray_count);
            std::vector<uint32_t> finishes(kPaths);
            const Recorder<T> rec { rays.data(), 0, out.data(), 0, SIZE_MAX };
            const PathRecorder<T> paths { rays.data(), ray_count, 0, offsets.data(), out.data(), finishes.data() };
            cu::DeformingInstances<T> less = inst, deep = inst;
            less.count -= 1;
            deep.max_depth = 60000;
            const char* ti = "DeviceView::trace_instances (deforming):";
            const char* tp = "DeviceView::trace_instance_paths (deforming):";
            expect([&] { top.template trace_instances<false, false>(1, less, rec, &cursor, sizeof cursor); }, ti, 1);
            expect([&] { top.template trace_instances<false, false>(1, inst, rec, &cursor, sizeof cursor - 1); }, ti, 2);
            expect([&] { top.template trace_instances<false, false>(1, deep, rec, &cursor, sizeof cursor); }, ti, 2);
            expect([&] { top.template trace_instance_paths<false>(1, less, paths, &cursor, sizeof cursor); }, tp, 1);
            expect([&] { top.template trace_instance_paths<false>(1, inst, paths, &cursor, sizeof cursor - 1); }, tp, 2);
            expect([&] { top.template trace_instance_paths<false>(1, deep, paths, &cursor, sizeof cursor); }, tp, 2);
            top.template trace_instance_paths<false>(0, inst, paths, &cursor, sizeof cursor);
            const bool empty_ok = finishes[0] == 0;
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
