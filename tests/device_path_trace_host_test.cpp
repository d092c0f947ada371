// tests/device_path_trace_host_test.cpp — DeviceView::trace_paths (include/bvh/v2/cuda/intersect.cuh) compiled as plain
// host C++, against Bvh<Node>::intersect of the C++ surface (include/bvh/v2/b200_surface.h) with a leaf that loops
// PrecomputedTri::intersect, applies the same tie rule and the same filter.
//
//   device_path_trace_host_test <case file> f|d    input as tests/device_trace_host_test.cpp reads it (written by
//                                                   tests/test_device_path_trace_host.py).  A recording shader runs
//                                                   scripted paths: path i has length(i) segments (0 to 64; path 0 has
//                                                   none, path 1 has 64), segment j traces ray hash(i, j) of the case as a
//                                                   Closest or an Occlusion segment by another bit of the hash.  For both
//                                                   robust settings and both tie rules it compares per segment the
//                                                   accept-call count, a hash of the accept sequence (original id and the
//                                                   bits of t, u, v) and the record (id, bits of t, u, v) with
//                                                   Bvh::intersect<IsAnyHit = Occlusion, IsRobust>, checks that next
//                                                   receives the scripted ray unchanged, and that start and finish are
//                                                   called once per path, in index order, with finish after the path's
//                                                   last segment.
// The filter drops every original id with id % 3 == 1.
#include <bvh/v2/bvh.h>
#include <bvh/v2/cuda/intersect.cuh>
#include <bvh/v2/stack.h>
#include <bvh/v2/tri.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <stdexcept>
#include <vector>

namespace {

using bvh::v2::cuda::PathStep;

uint64_t mix(uint64_t h, uint64_t x) { return (h ^ x) * 1099511628211ull; }
constexpr uint64_t kSeed = 1469598103934665603ull;
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

bool keep(size_t id) { return id % 3 != 1; }

struct Seg { uint64_t id, t, u, v; uint32_t calls; uint64_t hash; bool ray_ok; };
struct PathOut { uint32_t starts, finishes, segments, finish_order; };

template <typename T> struct Recorder {
    using View = bvh::v2::cuda::DeviceView<T>;
    using Ray = typename View::Ray;
    using Hit = typename View::Hit;
    struct Payload { size_t seg; uint32_t calls; uint64_t hash; };
    const T* rays;
    size_t ray_count;
    const size_t* offsets;
    std::vector<Seg>* segs;
    std::vector<PathOut>* paths;
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
        (*paths)[i].starts += 1;
        order->push_back(i);
        p.seg = 0; p.calls = 0; p.hash = kSeed;
        return path_length(i) ? segment(i, 0, ray) : PathStep::End;
    }
    bool accept(Payload& p, size_t prim_id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(p.hash, prim_id), bits(t)), bits(u)), bits(v));
        return keep(prim_id);
    }
    PathStep next(size_t i, Payload& p, const Hit& hit, Ray& ray) const {
        Ray want;
        segment(i, p.seg, want);
        Seg& s = (*segs)[offsets[i] + p.seg];
        s.ray_ok = std::memcmp(&want, &ray, sizeof ray) == 0;
        s.id = hit.prim_id; s.t = bits(hit.t); s.u = bits(hit.u); s.v = bits(hit.v);
        s.calls = p.calls; s.hash = p.hash;
        ++p.seg; p.calls = 0; p.hash = kSeed;
        return p.seg < path_length(i) ? segment(i, p.seg, ray) : PathStep::End;
    }
    void finish(size_t i, const Payload& p) const {
        (*paths)[i].finishes += 1;
        (*paths)[i].segments = (uint32_t)p.seg;
        (*paths)[i].finish_order = (*finished)++;
    }
};

// All ones in the record's id width
template <typename T> constexpr uint64_t kMissId = sizeof(T) == 4 ? 0xFFFFFFFFull : ~0ull;

template <typename T, bool Robust, bool Last>
void trace(const bvh::v2::cuda::DeviceView<T>& view, size_t n, const Recorder<T>& shader, unsigned long long& cursor) {
    view.template trace_paths<Robust, Last>(n, shader, &cursor, sizeof cursor);
}

template <typename T>
int run(std::ifstream& in) {
    using Node = bvh::v2::Node<T, 3>;
    using Bvh = bvh::v2::Bvh<Node>;
    using Vec3 = bvh::v2::Vec<T, 3>;
    using View = bvh::v2::cuda::DeviceView<T>;
    uint64_t node_count, prim_count, ray_count;
    in.read((char*)&node_count, 8); in.read((char*)&prim_count, 8); in.read((char*)&ray_count, 8);
    Bvh bvh;
    bvh.nodes.resize(node_count);
    in.read((char*)bvh.nodes.data(), node_count * sizeof(Node));
    std::vector<uint64_t> ids(prim_count);
    in.read((char*)ids.data(), prim_count * 8);
    bvh.prim_ids.assign(ids.begin(), ids.end());
    std::vector<T> verts(9 * prim_count), rays(8 * ray_count);
    in.read((char*)verts.data(), verts.size() * sizeof(T));
    in.read((char*)rays.data(), rays.size() * sizeof(T));
    if (!in) { std::puts("short input"); return 2; }

    // the device layout, as bvhNN_get_device_view reports it
    std::vector<bvhb200::DevNode<T>> dev_nodes(node_count + 1);
    std::memset(dev_nodes.data(), 0, dev_nodes.size() * sizeof(dev_nodes[0]));
    size_t depth = 0;
    {   // longest chain of inner nodes below the root
        std::vector<std::pair<size_t, size_t>> todo { { 0, 0 } };
        while (!todo.empty()) {
            auto [i, d] = todo.back(); todo.pop_back();
            if (bvh.nodes[i].is_leaf()) continue;
            depth = d > depth ? d : depth;
            todo.push_back({ bvh.nodes[i].index.first_id(), d + 1 });
            todo.push_back({ bvh.nodes[i].index.first_id() + 1, d + 1 });
        }
    }
    for (size_t i = 0; i < node_count; ++i) {
        for (int k = 0; k < 6; ++k) dev_nodes[i + 1].bounds[k] = bvh.nodes[i].bounds[k];
        dev_nodes[i + 1].index = bvh.nodes[i].index.value;
    }
    std::vector<uint32_t> ids32(ids.begin(), ids.end());
    std::vector<bvhb200::DevTri<T>> dev_tris(prim_count);
    std::vector<bvh::v2::PrecomputedTri<T>> tris(prim_count);
    for (size_t k = 0; k < prim_count; ++k) {
        const T* v = &verts[9 * ids[k]];
        dev_tris[k] = bvhb200::precompute_tri(v);
        tris[k] = bvh::v2::PrecomputedTri<T>(Vec3(v[0], v[1], v[2]), Vec3(v[3], v[4], v[5]), Vec3(v[6], v[7], v[8]));
    }
    View view;
    view.nodes = dev_nodes.data(); view.prim_ids = ids32.data(); view.tris = dev_tris.data();
    view.node_count = node_count; view.prim_count = prim_count; view.depth = depth;

    std::vector<size_t> offsets(kPaths + 1, 0);
    for (size_t i = 0; i < kPaths; ++i) offsets[i + 1] = offsets[i] + path_length(i);
    const size_t seg_count = offsets[kPaths];

    unsigned long long cursor = 0;
    int failures = 0;
    for (int mode = 0; mode < 4; ++mode) {       // bit 0 robust, bit 1 last visited
        const bool robust = mode & 1, last = mode & 2;
        std::vector<Seg> segs(seg_count);
        std::vector<PathOut> paths(kPaths);
        std::memset(segs.data(), 0, segs.size() * sizeof(segs[0]));
        std::memset(paths.data(), 0, paths.size() * sizeof(paths[0]));
        std::vector<size_t> order;
        uint32_t finished = 0;
        const Recorder<T> shader { rays.data(), ray_count, offsets.data(), &segs, &paths, &order, &finished };
        switch (mode) {
        case 0: trace<T, false, false>(view, kPaths, shader, cursor); break;
        case 1: trace<T, true, false>(view, kPaths, shader, cursor); break;
        case 2: trace<T, false, true>(view, kPaths, shader, cursor); break;
        case 3: trace<T, true, true>(view, kPaths, shader, cursor); break;
        }
        int bad = 0, hits = 0, occlusion = 0, nan = 0, path_bad = 0;
        uint64_t calls = 0;
        for (size_t i = 0; i < kPaths; ++i) {
            const PathOut& po = paths[i];
            if (po.starts != 1 || po.finishes != 1 || po.segments != path_length(i) || po.finish_order != i || order[i] != i) {
                if (path_bad < 3) std::printf("  path %zu: starts %u finishes %u segments %u/%zu\n", i, po.starts, po.finishes,
                                              po.segments, path_length(i));
                ++path_bad;
            }
            for (size_t j = 0; j < path_length(i); ++j) {
                const uint32_t h = segment_hash(i, j);
                const bool any = h >> 31;
                const T* r = &rays[8 * (h % ray_count)];
                bvh::v2::Ray<T, 3> ray(Vec3(r[0], r[1], r[2]), Vec3(r[3], r[4], r[5]), r[6], r[7]);
                bvh::v2::GrowingStack<typename Node::Index> stack;
                size_t best = SIZE_MAX;
                T bu = T(0), bv = T(0);
                uint32_t want_calls = 0;
                uint64_t want_hash = kSeed;
                auto leaf_fn = [&](size_t b, size_t e) {
                    for (size_t k = b; k < e; ++k) {
                        const auto hit = tris[k].intersect(ray);
                        if (!hit) continue;
                        const auto [t, u, v] = *hit;
                        const size_t id = bvh.prim_ids[k];
                        // the canonical rule takes an exact tie only from a lower original id
                        if (!last && best != SIZE_MAX && !(t < ray.tmax) && !(id < bvh.prim_ids[best])) continue;
                        ++want_calls;
                        want_hash = mix(mix(mix(mix(want_hash, id), bits(t)), bits(u)), bits(v));
                        if (!keep(id)) continue;
                        ray.tmax = t; best = k; bu = u; bv = v;
                    }
                    return best != SIZE_MAX;
                };
                const auto root = bvh.get_root().index;
                switch ((any ? 1 : 0) | (robust ? 2 : 0)) {
                case 0: bvh.template intersect<false, false>(ray, root, stack, leaf_fn); break;
                case 1: bvh.template intersect<true, false>(ray, root, stack, leaf_fn); break;
                case 2: bvh.template intersect<false, true>(ray, root, stack, leaf_fn); break;
                case 3: bvh.template intersect<true, true>(ray, root, stack, leaf_fn); break;
                }
                const uint64_t want_id = best == SIZE_MAX ? kMissId<T> : (uint64_t)bvh.prim_ids[best];
                const Seg& g = segs[offsets[i] + j];
                calls += g.calls;
                hits += g.id != kMissId<T>;
                occlusion += any;
                nan += r[6] != r[6] || r[7] != r[7];
                // a miss reports the input tmax, which is ray.tmax unchanged
                if (g.id != want_id || g.t != bits(ray.tmax) || g.u != bits(bu) || g.v != bits(bv) || g.calls != want_calls ||
                    g.hash != want_hash || !g.ray_ok) {
                    if (bad < 3) std::printf("  path %zu segment %zu: calls %u/%u id %llu/%llu ray %s\n", i, j, g.calls, want_calls,
                                             (unsigned long long)g.id, (unsigned long long)want_id, g.ray_ok ? "ok" : "CHANGED");
                    ++bad;
                }
            }
        }
        std::printf("mode %d segments %zu occlusion %d nan %d mismatches %d path mismatches %d hits %d accept calls %llu\n", mode,
                    seg_count, occlusion, nan, bad, path_bad, hits, (unsigned long long)calls);
        failures += bad + path_bad;
    }

    {   // n = 0 calls nothing; a small or missing workspace, or a tree too deep for the shared-memory stack, throws
        // std::length_error; a view without triangles throws std::invalid_argument
        std::vector<Seg> segs(seg_count);
        std::vector<PathOut> paths(kPaths);
        std::vector<size_t> order;
        uint32_t finished = 0;
        const Recorder<T> shader { rays.data(), ray_count, offsets.data(), &segs, &paths, &order, &finished };
        view.template trace_paths<false>(0, shader, &cursor, sizeof cursor);
        const bool empty_ok = order.empty() && finished == 0;
        bool threw = false, threw_null = false, threw_deep = false, threw_boxes = false;
        try { view.template trace_paths<false>(1, shader, &cursor, sizeof cursor - 1); } catch (const std::length_error&) { threw = true; }
        try { view.template trace_paths<false>(1, shader, nullptr, sizeof cursor); } catch (const std::length_error&) { threw_null = true; }
        View deep = view;
        deep.depth = 400;
        try { deep.template trace_paths<false>(1, shader, &cursor, sizeof cursor); } catch (const std::length_error&) { threw_deep = true; }
        View boxes = view;
        boxes.tris = nullptr;
        try { boxes.template trace_paths<false>(1, shader, &cursor, sizeof cursor); } catch (const std::invalid_argument&) { threw_boxes = true; }
        std::printf("empty batch %s, small workspace %s, null workspace %s, deep tree %s, no triangles %s\n", empty_ok ? "ok" : "CALLED",
                    threw ? "throws" : "DID NOT THROW", threw_null ? "throws" : "DID NOT THROW", threw_deep ? "throws" : "DID NOT THROW",
                    threw_boxes ? "throws" : "DID NOT THROW");
        if (!empty_ok || !threw || !threw_null || !threw_deep || !threw_boxes || !order.empty()) ++failures;
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
