// tests/device_api_host_test.cpp — the device traversal API (include/bvh/v2/cuda/intersect.cuh) compiled as plain host
// C++ and run on host copies of a tree, against Bvh<Node>::intersect of the C++ surface (include/bvh/v2/b200_surface.h).
//
// Input (written by tests/test_device_api_host.py): node_count, prim_count, ray_count (u64), the reference-layout nodes,
// the u64 primitive ids, the triangles' vertices in original order and the rays.  For the fast, robust and any-hit
// traversals, started at the root and at reference node 1, and with a triangle leaf (which shrinks tmax) and a leaf that
// only records (tmax never shrinks), it compares per ray the leaf-call count, a hash of the (begin, end) sequence, the
// inner-hook count, the hit id and the final tmax, and prints the mismatches.  It writes the triangle leaf's ids and t
// from the root for modes 0 (closest, fast), 1 (any, fast), 2 (closest, robust) to the output file.
#include <bvh/v2/bvh.h>
#include <bvh/v2/cuda/intersect.cuh>
#include <bvh/v2/stack.h>
#include <bvh/v2/tri.h>

#include <cstdio>
#include <fstream>
#include <vector>

namespace {

uint64_t mix(uint64_t h, uint64_t x) { return (h ^ x) * 1099511628211ull; }

struct Result { uint32_t id, leaves, inner; uint64_t hash; };

template <typename T> struct RayPodOf;
template <> struct RayPodOf<float> { using Type = bvh_ray3f; };
template <> struct RayPodOf<double> { using Type = bvh_ray3d; };

template <typename T>
int run(std::ifstream& in, const char* out_path) {
    using Node = bvh::v2::Node<T, 3>;
    using Bvh = bvh::v2::Bvh<Node>;
    using Vec3 = bvh::v2::Vec<T, 3>;
    using View = bvh::v2::cuda::DeviceView<T>;
    using RayPod = typename RayPodOf<T>::Type;
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

    // the device layout, as bvhNN_get_device_view reports it: node i at slot i + 1, u32 ids, BVH-order PrecomputedTri
    std::vector<bvhb200::DevNode<T>> dev_nodes(node_count + 1);
    std::memset(dev_nodes.data(), 0, dev_nodes.size() * sizeof(dev_nodes[0]));
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
    view.node_count = node_count; view.prim_count = prim_count;

    std::vector<uint32_t> out_ids(3 * ray_count);
    std::vector<T> out_t(3 * ray_count);
    int failures = 0;
    for (int mode = 0; mode < 4; ++mode) {           // 0 closest fast, 1 any fast, 2 closest robust, 3 any robust
        for (int leaf = 0; leaf < 2; ++leaf) {      // 0 triangles, 1 record only
            for (int from = 0; from < (node_count > 1 ? 2 : 1); ++from) {
                int bad = 0, hits = 0;
                uint64_t calls = 0;
                for (size_t i = 0; i < ray_count; ++i) {
                    const T* r = &rays[8 * i];
                    Result want { 0xFFFFFFFFu, 0, 0, 1469598103934665603ull }, got = want;
                    T want_tmax, got_tmax;
                    {   // the C++ surface on the host
                        bvh::v2::Ray<T, 3> ray(Vec3(r[0], r[1], r[2]), Vec3(r[3], r[4], r[5]), r[6], r[7]);
                        bvh::v2::SmallStack<typename Node::Index, 256> stack;
                        size_t best = SIZE_MAX;
                        auto leaf_fn = [&](size_t b, size_t e) {
                            ++want.leaves; want.hash = mix(mix(want.hash, b), e);
                            if (leaf == 0)
                                for (size_t k = b; k < e; ++k)
                                    if (auto hit = tris[k].intersect(ray)) { ray.tmax = std::get<0>(*hit); best = k; }
                            return best != SIZE_MAX;
                        };
                        auto inner_fn = [&](const Node&, const Node&) { ++want.inner; };
                        const auto start = bvh.nodes[from].index;
                        if (mode == 0) bvh.template intersect<false, false>(ray, start, stack, leaf_fn, inner_fn);
                        if (mode == 1) bvh.template intersect<true, false>(ray, start, stack, leaf_fn, inner_fn);
                        if (mode == 2) bvh.template intersect<false, true>(ray, start, stack, leaf_fn, inner_fn);
                        if (mode == 3) bvh.template intersect<true, true>(ray, start, stack, leaf_fn, inner_fn);
                        want.id = best == SIZE_MAX ? 0xFFFFFFFFu : (uint32_t)bvh.prim_ids[best];
                        want_tmax = ray.tmax;
                    }
                    {   // the device API's traversal, compiled for the host
                        RayPod ray;
                        ray.org.x = r[0]; ray.org.y = r[1]; ray.org.z = r[2];
                        ray.dir.x = r[3]; ray.dir.y = r[4]; ray.dir.z = r[5];
                        ray.tmin = r[6]; ray.tmax = r[7];
                        typename View::template SmallStack<256> stack;
                        size_t best = SIZE_MAX;
                        auto leaf_fn = [&](size_t b, size_t e) {
                            ++got.leaves; got.hash = mix(mix(got.hash, b), e);
                            if (leaf == 0)
                                for (size_t k = b; k < e; ++k) {
                                    T t, u, v;
                                    if (view.intersect_tri(k, ray, t, u, v)) { ray.tmax = t; best = k; }
                                }
                            return best != SIZE_MAX;
                        };
                        auto inner_fn = [&](size_t) { ++got.inner; };
                        const auto start = view.node(from).index;
                        if (mode == 0) view.template intersect<false, false>(ray, start, stack, leaf_fn, inner_fn);
                        if (mode == 1) view.template intersect<true, false>(ray, start, stack, leaf_fn, inner_fn);
                        if (mode == 2) view.template intersect<false, true>(ray, start, stack, leaf_fn, inner_fn);
                        if (mode == 3) view.template intersect<true, true>(ray, start, stack, leaf_fn, inner_fn);
                        got.id = best == SIZE_MAX ? 0xFFFFFFFFu : (uint32_t)view.prim_id(best);
                        got_tmax = ray.tmax;
                    }
                    calls += got.leaves;
                    hits += got.id != 0xFFFFFFFFu;
                    if (got.id != want.id || got.leaves != want.leaves || got.hash != want.hash || got.inner != want.inner ||
                        std::memcmp(&got_tmax, &want_tmax, sizeof(T)) != 0) {
                        if (bad < 3) std::printf("  ray %zu: leaves %u/%u inner %u/%u id %u/%u\n", i, got.leaves, want.leaves,
                                                 got.inner, want.inner, got.id, want.id);
                        ++bad;
                    }
                    if (leaf == 0 && from == 0 && mode < 3) { out_ids[mode * ray_count + i] = got.id; out_t[mode * ray_count + i] = got_tmax; }
                }
                std::printf("mode %d leaf %d start %d mismatches %d hits %d leaf calls %llu\n", mode, leaf, from, bad, hits,
                            (unsigned long long)calls);
                failures += bad;
            }
        }
    }
    std::ofstream out(out_path, std::ios::binary);
    out.write((const char*)out_ids.data(), out_ids.size() * 4);
    out.write((const char*)out_t.data(), out_t.size() * sizeof(T));
    return failures;
}

} // namespace

int main(int argc, char** argv) {
    if (argc < 4) return 2;
    std::ifstream in(argv[1], std::ios::binary);
    if (!in) return 2;
    const int failures = argv[2][0] == 'd' ? run<double>(in, argv[3]) : run<float>(in, argv[3]);
    std::printf("failures %d\n", failures);
    return failures ? 1 : 0;
}
