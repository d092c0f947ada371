// tests/device_triangle_trace_host_test.cpp — DeviceView::trace_triangles (include/bvh/v2/cuda/intersect.cuh) compiled as
// plain host C++, against Bvh<Node>::intersect of the C++ surface (include/bvh/v2/b200_surface.h) with a leaf that loops
// PrecomputedTri::intersect, applies the same tie rule and the same filter.
//
//   device_triangle_trace_host_test <case file> f|d    input as tests/device_trace_host_test.cpp reads it (written by
//                                                       tests/test_device_triangle_trace_host.py).  For the four
//                                                       IsAnyHit x IsRobust combinations, both tie rules and the filters
//                                                       below it compares per ray the accept-call count, a hash of the
//                                                       accept sequence (original id and the bits of t, u, v) and the final
//                                                       record (id, bits of t, u, v), and checks that start and finish are
//                                                       called once per ray, in index order.  The accept-all records must
//                                                       also equal the host emulation's traverse_ray (traverse_core.cuh).
// Filters: 0 accept all, 1 reject all, 2 reject odd ids, 3 an alpha cut-out on (u, v), 4 reject the ray's origin triangle
// (here: the triangle the closest-hit, lowest-id, accept-all pass found for that ray).
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

uint64_t mix(uint64_t h, uint64_t x) { return (h ^ x) * 1099511628211ull; }
constexpr uint64_t kSeed = 1469598103934665603ull;
constexpr uint32_t kNone = 0xFFFFFFFFu;

template <typename T> uint64_t bits(T x) {
    if constexpr (sizeof(T) == 4) { uint32_t b; std::memcpy(&b, &x, 4); return b; }
    else { uint64_t b; std::memcpy(&b, &x, 8); return b; }
}

enum Filter : int { kAll = 0, kNoneAccepted, kEvenIds, kAlpha, kNotOrigin, kFilters };

// The filters, on the original id and the candidate's barycentrics.
template <typename T> bool keep(int filter, size_t id, T u, T v, uint32_t origin) {
    switch (filter) {
    case kAll: return true;
    case kNoneAccepted: return false;
    case kEvenIds: return (id & 1) == 0;
    case kAlpha: return u < T(0.5) || v < T(0.25);     // a cut-out: the corner u >= 0.5, v >= 0.25 is transparent
    case kNotOrigin: return id != origin;
    }
    return true;
}

template <typename T> struct Out { uint64_t id; uint64_t t, u, v; uint32_t calls, starts, finishes; uint64_t hash; };

template <typename T> struct RayPodOf;
template <> struct RayPodOf<float> { using Type = bvh_ray3f; };
template <> struct RayPodOf<double> { using Type = bvh_ray3d; };

// A recording shader: the accept calls go into the payload, finish writes the record.
template <typename T> struct RecordShader {
    using View = bvh::v2::cuda::DeviceView<T>;
    using Ray = typename View::Ray;
    struct Payload { size_t i; uint32_t calls; uint64_t hash; };
    const T* rays;
    int filter;
    const uint32_t* origins;
    Out<T>* out;
    size_t* order;                      // the index sequence of start calls
    size_t* started;

    Ray start(size_t i, Payload& p) const {
        const T* r = rays + 8 * i;
        Ray ray;
        ray.org.x = r[0]; ray.org.y = r[1]; ray.org.z = r[2];
        ray.dir.x = r[3]; ray.dir.y = r[4]; ray.dir.z = r[5];
        ray.tmin = r[6]; ray.tmax = r[7];
        p.i = i; p.calls = 0; p.hash = kSeed;
        out[i].starts += 1;
        order[(*started)++] = i;
        return ray;
    }
    bool accept(Payload& p, size_t prim_id, T t, T u, T v) const {
        ++p.calls;
        p.hash = mix(mix(mix(mix(p.hash, prim_id), bits(t)), bits(u)), bits(v));
        return keep<T>(filter, prim_id, u, v, origins[p.i]);
    }
    void finish(size_t i, const Payload& p, const typename View::Hit& hit) const {
        out[i].id = hit.prim_id; out[i].t = bits(hit.t); out[i].u = bits(hit.u); out[i].v = bits(hit.v);
        out[i].calls = p.calls;
        out[i].hash = p.hash;
        out[i].finishes += 1;
    }
};

// All ones in the record's id width
template <typename T> constexpr uint64_t kMissId = sizeof(T) == 4 ? 0xFFFFFFFFull : ~0ull;

template <typename T, bool Any, bool Robust, bool Last>
void trace(const bvh::v2::cuda::DeviceView<T>& view, size_t n, const RecordShader<T>& shader, unsigned long long& cursor) {
    view.template trace_triangles<Any, Robust, Last>(n, shader, &cursor, sizeof cursor);
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

    unsigned long long cursor = 0;
    int failures = 0;
    std::vector<uint32_t> origins(ray_count, kNone);
    for (int filter = 0; filter < kFilters; ++filter) {
        for (int mode = 0; mode < 8; ++mode) {       // bit 0 any-hit, bit 1 robust, bit 2 last visited
            const bool any = mode & 1, robust = mode & 2, last = mode & 4;
            std::vector<Out<T>> got(ray_count);
            std::memset(got.data(), 0, got.size() * sizeof(got[0]));
            std::vector<size_t> order(ray_count + 1);
            size_t started = 0;
            const RecordShader<T> shader { rays.data(), filter, origins.data(), got.data(), order.data(), &started };
            switch (mode) {
            case 0: trace<T, false, false, false>(view, ray_count, shader, cursor); break;
            case 1: trace<T, true, false, false>(view, ray_count, shader, cursor); break;
            case 2: trace<T, false, true, false>(view, ray_count, shader, cursor); break;
            case 3: trace<T, true, true, false>(view, ray_count, shader, cursor); break;
            case 4: trace<T, false, false, true>(view, ray_count, shader, cursor); break;
            case 5: trace<T, true, false, true>(view, ray_count, shader, cursor); break;
            case 6: trace<T, false, true, true>(view, ray_count, shader, cursor); break;
            case 7: trace<T, true, true, true>(view, ray_count, shader, cursor); break;
            }
            int bad = 0, hits = 0, emul_bad = 0;
            uint64_t calls = 0;
            for (size_t i = 0; i < ray_count; ++i) {
                const T* r = &rays[8 * i];
                bvh::v2::Ray<T, 3> ray(Vec3(r[0], r[1], r[2]), Vec3(r[3], r[4], r[5]), r[6], r[7]);
                bvh::v2::GrowingStack<typename Node::Index> stack;
                size_t best = SIZE_MAX;
                T bu = T(0), bv = T(0);
                uint32_t want_calls = 0;
                uint64_t want_hash = kSeed;
                auto leaf_fn = [&](size_t b, size_t e) {
                    for (size_t k = b; k < e; ++k) {
                        const auto h = tris[k].intersect(ray);
                        if (!h) continue;
                        const auto [t, u, v] = *h;
                        const size_t id = bvh.prim_ids[k];
                        // the canonical rule takes an exact tie only from a lower original id
                        if (!last && best != SIZE_MAX && !(t < ray.tmax) && !(id < bvh.prim_ids[best])) continue;
                        ++want_calls;
                        want_hash = mix(mix(mix(mix(want_hash, id), bits(t)), bits(u)), bits(v));
                        if (!keep<T>(filter, id, u, v, origins[i])) continue;
                        ray.tmax = t; best = k; bu = u; bv = v;
                    }
                    return best != SIZE_MAX;
                };
                const auto root = bvh.get_root().index;
                switch (mode & 3) {
                case 0: bvh.template intersect<false, false>(ray, root, stack, leaf_fn); break;
                case 1: bvh.template intersect<true, false>(ray, root, stack, leaf_fn); break;
                case 2: bvh.template intersect<false, true>(ray, root, stack, leaf_fn); break;
                case 3: bvh.template intersect<true, true>(ray, root, stack, leaf_fn); break;
                }
                const uint64_t want_id = best == SIZE_MAX ? kMissId<T> : (uint64_t)bvh.prim_ids[best];
                const Out<T>& g = got[i];
                calls += g.calls;
                hits += g.id != kMissId<T>;
                // a miss reports the input tmax, which is ray.tmax unchanged
                if (g.id != want_id || g.t != bits(ray.tmax) || g.u != bits(bu) || g.v != bits(bv) || g.calls != want_calls ||
                    g.hash != want_hash || g.starts != 1 || g.finishes != 1 || order[i] != i) {
                    if (bad < 3) std::printf("  ray %zu: calls %u/%u id %llu/%llu starts %u finishes %u\n", i, g.calls, want_calls,
                                             (unsigned long long)g.id, (unsigned long long)want_id, g.starts, g.finishes);
                    ++bad;
                }
                if (filter == kAll) {
                    // the host emulation of the library's kernels on the same arrays
                    bvhb200::RayCtx<T> rc;
                    for (int a = 0; a < 3; ++a) { rc.org[a] = r[a]; rc.dir[a] = r[3 + a]; }
                    rc.tmin = r[6]; rc.tmax = r[7];
                    const T tmax_in = rc.tmax;
                    bvhb200::HitState<T> hs { bvhb200::kInvalidId, rc.tmax, T(0), T(0) };
                    bvh::v2::cuda::detail::VectorStack<typename View::Index> es;
                    if (robust) bvhb200::ray_prologue<T, true>(rc); else bvhb200::ray_prologue<T, false>(rc);
                    switch (mode & 3) {
                    case 0: bvhb200::traverse_ray<T, false, false>(dev_nodes.data(), dev_tris.data(), ids32.data(), !last, view.root_index(), rc, hs, es, nullptr); break;
                    case 1: bvhb200::traverse_ray<T, true, false>(dev_nodes.data(), dev_tris.data(), ids32.data(), !last, view.root_index(), rc, hs, es, nullptr); break;
                    case 2: bvhb200::traverse_ray<T, false, true>(dev_nodes.data(), dev_tris.data(), ids32.data(), !last, view.root_index(), rc, hs, es, nullptr); break;
                    case 3: bvhb200::traverse_ray<T, true, true>(dev_nodes.data(), dev_tris.data(), ids32.data(), !last, view.root_index(), rc, hs, es, nullptr); break;
                    }
                    const bvhb200::DevHit<T> rec = bvhb200::make_record(hs, tmax_in, ids32.data());
                    if ((uint64_t)rec.prim_id != g.id || bits(rec.t) != g.t || bits(rec.u) != g.u || bits(rec.v) != g.v) ++emul_bad;
                    if (mode == 0) origins[i] = (uint32_t)g.id;
                }
            }
            std::printf("filter %d mode %d mismatches %d emulation mismatches %d hits %d accept calls %llu\n", filter, mode, bad,
                        emul_bad, hits, (unsigned long long)calls);
            failures += bad + emul_bad;
        }
    }

    {   // n = 0 calls nothing; a small or missing workspace throws std::length_error; a view without triangles throws
        // std::invalid_argument
        std::vector<Out<T>> got(1);
        std::memset(got.data(), 0, sizeof(got[0]));
        size_t order[1], started = 0;
        const RecordShader<T> shader { rays.data(), 0, origins.data(), got.data(), order, &started };
        view.template trace_triangles<false, false>(0, shader, &cursor, sizeof cursor);
        const bool empty_ok = started == 0 && got[0].finishes == 0;
        bool threw = false, threw_null = false, threw_boxes = false;
        try { view.template trace_triangles<false, false>(1, shader, &cursor, sizeof cursor - 1); } catch (const std::length_error&) { threw = true; }
        try { view.template trace_triangles<false, false>(1, shader, nullptr, sizeof cursor); } catch (const std::length_error&) { threw_null = true; }
        View boxes = view;
        boxes.tris = nullptr;
        try { boxes.template trace_triangles<false, false>(1, shader, &cursor, sizeof cursor); } catch (const std::invalid_argument&) { threw_boxes = true; }
        std::printf("empty batch %s, small workspace %s, null workspace %s, no triangles %s\n", empty_ok ? "ok" : "CALLED",
                    threw ? "throws" : "DID NOT THROW", threw_null ? "throws" : "DID NOT THROW", threw_boxes ? "throws" : "DID NOT THROW");
        if (!empty_ok || !threw || !threw_null || !threw_boxes || started != 0) ++failures;
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
