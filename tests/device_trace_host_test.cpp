// tests/device_trace_host_test.cpp — DeviceView::trace (include/bvh/v2/cuda/intersect.cuh) compiled as plain host C++,
// against Bvh<Node>::intersect of the C++ surface (include/bvh/v2/b200_surface.h).
//
//   device_trace_host_test <case file> f|d     input as tests/device_api_host_test.cpp reads it (written by
//                                               tests/test_device_trace_host.py).  For the four flag combinations and
//                                               the leaves below it compares per ray the leaf-call count, a hash of the
//                                               (begin, end) sequence, the hit id and the final tmax, and checks that
//                                               start and finish are called once per ray, in index order.
//   device_trace_host_test plan                 prints persistent_run_rays and persistent_grid (trace_plan.h) over a
//                                               table of batch sizes and SM counts, one "n sms chunk per_sm run grid" line
//                                               per entry.
// Leaves: 0 the triangle test (shrinks tmax), 1 record only, 2 the triangle test that sets tmax to NaN on its second call.
#include <bvh/v2/bvh.h>
#include <bvh/v2/cuda/intersect.cuh>
#include <bvh/v2/stack.h>
#include <bvh/v2/tri.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <limits>
#include <stdexcept>
#include <vector>

namespace {

uint64_t mix(uint64_t h, uint64_t x) { return (h ^ x) * 1099511628211ull; }
constexpr uint64_t kSeed = 1469598103934665603ull;

template <typename T> struct Out { uint32_t id, calls, starts, finishes; uint64_t hash; T tmax; };

template <typename T> struct RayPodOf;
template <> struct RayPodOf<float> { using Type = bvh_ray3f; };
template <> struct RayPodOf<double> { using Type = bvh_ray3d; };

// A recording tracer: the leaf's calls go into the payload, finish writes the ray's record.
template <typename T> struct RecordTracer {
    using View = bvh::v2::cuda::DeviceView<T>;
    using Ray = typename View::Ray;
    struct Payload { size_t best; uint32_t calls; uint64_t hash; };
    View view;
    const T* rays;
    int leaf_kind;
    Out<T>* out;
    size_t* order;                      // the index sequence of start calls
    size_t* started;

    Ray start(size_t i, Payload& p) const {
        const T* r = rays + 8 * i;
        Ray ray;
        ray.org.x = r[0]; ray.org.y = r[1]; ray.org.z = r[2];
        ray.dir.x = r[3]; ray.dir.y = r[4]; ray.dir.z = r[5];
        ray.tmin = r[6]; ray.tmax = r[7];
        p.best = SIZE_MAX; p.calls = 0; p.hash = kSeed;
        out[i].starts += 1;
        order[(*started)++] = i;
        return ray;
    }
    bool leaf(Payload& p, Ray& ray, size_t begin, size_t end) const {
        ++p.calls;
        p.hash = mix(mix(p.hash, begin), end);
        if (leaf_kind != 1)
            for (size_t k = begin; k < end; ++k) {
                T t, u, v;
                if (view.intersect_tri(k, ray, t, u, v)) { ray.tmax = t; p.best = k; }
            }
        if (leaf_kind == 2 && p.calls == 2) ray.tmax = std::numeric_limits<T>::quiet_NaN();
        return p.best != SIZE_MAX;
    }
    void finish(size_t i, const Payload& p, const Ray& ray) const {
        out[i].id = p.best == SIZE_MAX ? 0xFFFFFFFFu : (uint32_t)view.prim_id(p.best);
        out[i].calls = p.calls;
        out[i].hash = p.hash;
        out[i].tmax = ray.tmax;
        out[i].finishes += 1;
    }
};

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
    for (int mode = 0; mode < 4; ++mode) {           // 0 closest fast, 1 any fast, 2 closest robust, 3 any robust
        for (int leaf = 0; leaf < 3; ++leaf) {
            std::vector<Out<T>> got(ray_count);
            std::memset(got.data(), 0, got.size() * sizeof(got[0]));
            std::vector<size_t> order(ray_count + 1);
            size_t started = 0;
            const RecordTracer<T> tracer { view, rays.data(), leaf, got.data(), order.data(), &started };
            if (mode == 0) view.template trace<false, false>(ray_count, tracer, &cursor, sizeof cursor);
            if (mode == 1) view.template trace<true, false>(ray_count, tracer, &cursor, sizeof cursor);
            if (mode == 2) view.template trace<false, true>(ray_count, tracer, &cursor, sizeof cursor);
            if (mode == 3) view.template trace<true, true>(ray_count, tracer, &cursor, sizeof cursor);
            int bad = 0, hits = 0;
            uint64_t calls = 0;
            for (size_t i = 0; i < ray_count; ++i) {
                const T* r = &rays[8 * i];
                Out<T> want { 0xFFFFFFFFu, 0, 1, 1, kSeed, T(0) };
                bvh::v2::Ray<T, 3> ray(Vec3(r[0], r[1], r[2]), Vec3(r[3], r[4], r[5]), r[6], r[7]);
                bvh::v2::GrowingStack<typename Node::Index> stack;
                size_t best = SIZE_MAX;
                auto leaf_fn = [&](size_t b, size_t e) {
                    ++want.calls; want.hash = mix(mix(want.hash, b), e);
                    if (leaf != 1)
                        for (size_t k = b; k < e; ++k)
                            if (auto hit = tris[k].intersect(ray)) { ray.tmax = std::get<0>(*hit); best = k; }
                    if (leaf == 2 && want.calls == 2) ray.tmax = std::numeric_limits<T>::quiet_NaN();
                    return best != SIZE_MAX;
                };
                const auto root = bvh.get_root().index;
                if (mode == 0) bvh.template intersect<false, false>(ray, root, stack, leaf_fn);
                if (mode == 1) bvh.template intersect<true, false>(ray, root, stack, leaf_fn);
                if (mode == 2) bvh.template intersect<false, true>(ray, root, stack, leaf_fn);
                if (mode == 3) bvh.template intersect<true, true>(ray, root, stack, leaf_fn);
                want.id = best == SIZE_MAX ? 0xFFFFFFFFu : (uint32_t)bvh.prim_ids[best];
                want.tmax = ray.tmax;
                const Out<T>& g = got[i];
                calls += g.calls;
                hits += g.id != 0xFFFFFFFFu;
                if (g.id != want.id || g.calls != want.calls || g.hash != want.hash || g.starts != 1 || g.finishes != 1 ||
                    order[i] != i || std::memcmp(&g.tmax, &want.tmax, sizeof(T)) != 0) {
                    if (bad < 3) std::printf("  ray %zu: calls %u/%u id %u/%u starts %u finishes %u\n", i, g.calls, want.calls,
                                             g.id, want.id, g.starts, g.finishes);
                    ++bad;
                }
            }
            std::printf("mode %d leaf %d mismatches %d hits %d leaf calls %llu\n", mode, leaf, bad, hits, (unsigned long long)calls);
            failures += bad;
        }
    }

    {   // n = 0 calls nothing; a workspace that is too small throws std::length_error
        std::vector<Out<T>> got(1);
        std::memset(got.data(), 0, sizeof(got[0]));
        size_t order[1], started = 0;
        const RecordTracer<T> tracer { view, rays.data(), 0, got.data(), order, &started };
        view.template trace<false, false>(0, tracer, &cursor, sizeof cursor);
        const bool empty_ok = started == 0 && got[0].finishes == 0;
        bool threw = false, threw_null = false;
        try { view.template trace<false, false>(1, tracer, &cursor, sizeof cursor - 1); } catch (const std::length_error&) { threw = true; }
        try { view.template trace<false, false>(1, tracer, nullptr, sizeof cursor); } catch (const std::length_error&) { threw_null = true; }
        std::printf("empty batch %s, small workspace %s, null workspace %s\n", empty_ok ? "ok" : "CALLED", threw ? "throws" : "DID NOT THROW",
                    threw_null ? "throws" : "DID NOT THROW");
        if (!empty_ok || !threw || !threw_null || started != 0) ++failures;
    }
    return failures;
}

int plan() {
    const unsigned long long ns[] = { 1, 31, 32, 33, 1000, 4096, 33791, 33792, 33793, 100000, 1000000, 10004569, 1ull << 32 };
    const int sms[] = { 1, 16, 114, 132, 148 };
    const uint32_t chunks[] = { 32, 64, 100, 256 };
    const int per_sms[] = { 0, 1, 4, 9 };
    for (unsigned long long n : ns)
        for (int sm : sms)
            for (uint32_t chunk : chunks)
                for (int per_sm : per_sms)
                    std::printf("%llu %d %u %d %u %llu\n", n, sm, chunk, per_sm, bvhb200::persistent_run_rays(chunk, n, sm),
                                bvhb200::persistent_grid(sm, per_sm, n, 32, bvhb200::kTraceBlock / 32));
    return 0;
}

} // namespace

int main(int argc, char** argv) {
    if (argc == 2 && std::strcmp(argv[1], "plan") == 0) return plan();
    if (argc < 3) return 2;
    std::ifstream in(argv[1], std::ios::binary);
    if (!in) return 2;
    const int failures = argv[2][0] == 'd' ? run<double>(in) : run<float>(in);
    std::printf("failures %d\n", failures);
    return failures ? 1 : 0;
}
