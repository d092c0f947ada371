// tests/device_query_host_test.cpp — DeviceView::traverse_top_down (include/bvh/v2/cuda/intersect.cuh) compiled as plain
// host C++ and run on host copies of a tree, against Bvh<Node>::traverse_top_down of the C++ surface
// (include/bvh/v2/b200_surface.h) with the same node and leaf functions.
//
// Input (written by tests/test_device_query_host.py): node_count, prim_count, query_count (u64), the reference-layout
// nodes, the u64 primitive ids, the primitives' boxes (min3, max3) in original order and the query boxes (min3, max3;
// the point queries use min3).  For every query, query kind and start node (0: the root, 1: reference node 1, 2: the
// first leaf), it compares the leaf-call count, a hash of the (begin, end) sequence, the node-function count and the
// query's result, and prints one line per kind and start:
//   kind K start S mismatches M leaf_calls L node_calls N result R
// where R sums the results over the queries.  Kinds:
//   0 overlap      every primitive whose box overlaps the query box (result: count and a hash of the id set)
//   1 contains     IsAnyHit: the first primitive whose box contains the point; the node test is containment
//   2 nearest      the primitive box nearest to the point: descends nearer child first (should_swap) and the leaf
//                  shrinks the search radius the node test reads (result: id and squared distance)
//   3 reject-all   the node test hits nothing
//   4 accept-all   the node test hits both children, in order: every leaf below the start, in the reference's order
//   5 accept-all, swapped, IsAnyHit: right child first; the third leaf call returns true and ends the traversal
#include <bvh/v2/bvh.h>
#include <bvh/v2/stack.h>

#include "device_queries.h"

#include <cstdio>
#include <cstring>
#include <fstream>
#include <tuple>
#include <vector>

namespace {

struct Record { uint64_t leaves = 0, nodes = 0, hash = dq::kHashSeed, r0 = 0, r1 = 0; };

// The query `kind` through traverse(start, stack, leaf_fn, node_fn) of either implementation.  `slot_id(k)` is the
// original id of BVH-order primitive k.
template <typename T, typename Traverse, typename SlotId>
Record run_kind(int kind, const T* q, const std::vector<T>& boxes, SlotId slot_id, Traverse traverse) {
    Record rec;
    const T* p = q;                                      // the point queries use min3
    T best = T(1) / T(0);
    uint64_t best_id = ~0ull;
    auto leaf_fn = [&](size_t begin, size_t end) {
        ++rec.leaves;
        rec.hash = dq::mix(dq::mix(rec.hash, begin), end);
        for (size_t k = begin; k < end; ++k) {
            const uint64_t id = slot_id(k);
            const T* b = &boxes[6 * id];
            if (kind == 0 && dq::overlaps<T>(dq::AsNode<T>{ b }, q)) { ++rec.r0; rec.r1 += dq::id_hash(id); }
            if (kind == 1 && dq::contains<T>(dq::AsNode<T>{ b }, p)) { rec.r0 = id; return true; }
            if (kind == 2) {
                const T d = dq::box_dist2<T>(dq::AsNode<T>{ b }, p);
                if (d < best) { best = d; best_id = id; }
            }
        }
        return kind == 5 && rec.leaves == 3;
    };
    auto node_fn = [&](const auto& l, const auto& r) {
        ++rec.nodes;
        switch (kind) {
        case 0: return std::make_tuple(dq::overlaps<T>(l.bounds, q), dq::overlaps<T>(r.bounds, q), false);
        case 1: return std::make_tuple(dq::contains<T>(l.bounds, p), dq::contains<T>(r.bounds, p), false);
        case 2: {
            const T dl = dq::box_dist2<T>(l.bounds, p), dr = dq::box_dist2<T>(r.bounds, p);
            return std::make_tuple(dl < best, dr < best, dl > dr);
        }
        case 3: return std::make_tuple(false, false, false);
        case 4: return std::make_tuple(true, true, false);
        default: return std::make_tuple(true, true, true);
        }
    };
    traverse(leaf_fn, node_fn);
    if (kind == 2) { rec.r0 = best_id; std::memcpy(&rec.r1, &best, sizeof(T)); }
    return rec;
}

template <typename T>
int run(std::ifstream& in) {
    using Node = bvh::v2::Node<T, 3>;
    using Bvh = bvh::v2::Bvh<Node>;
    using View = bvh::v2::cuda::DeviceView<T>;
    uint64_t node_count, prim_count, query_count;
    in.read((char*)&node_count, 8); in.read((char*)&prim_count, 8); in.read((char*)&query_count, 8);
    Bvh bvh;
    bvh.nodes.resize(node_count);
    in.read((char*)bvh.nodes.data(), node_count * sizeof(Node));
    std::vector<uint64_t> ids(prim_count);
    in.read((char*)ids.data(), prim_count * 8);
    bvh.prim_ids.assign(ids.begin(), ids.end());
    std::vector<T> boxes(6 * prim_count), queries(6 * query_count);
    in.read((char*)boxes.data(), boxes.size() * sizeof(T));
    in.read((char*)queries.data(), queries.size() * sizeof(T));
    if (!in) { std::puts("short input"); return 2; }

    // the device layout, as bvhNN_get_device_view reports it: node i at slot i + 1, u32 ids
    std::vector<bvhb200::DevNode<T>> dev_nodes(node_count + 1);
    std::memset(dev_nodes.data(), 0, dev_nodes.size() * sizeof(dev_nodes[0]));
    for (size_t i = 0; i < node_count; ++i) {
        for (int k = 0; k < 6; ++k) dev_nodes[i + 1].bounds[k] = bvh.nodes[i].bounds[k];
        dev_nodes[i + 1].index = bvh.nodes[i].index.value;
    }
    std::vector<uint32_t> ids32(ids.begin(), ids.end());
    View view;
    view.nodes = dev_nodes.data(); view.prim_ids = ids32.data();
    view.node_count = node_count; view.prim_count = prim_count;

    size_t first_leaf = 0;
    while (first_leaf < node_count && !bvh.nodes[first_leaf].is_leaf()) ++first_leaf;
    const size_t starts[3] = { 0, node_count > 1 ? size_t(1) : size_t(0), first_leaf };

    int failures = 0;
    for (int kind = 0; kind < 6; ++kind) {
        for (int s = 0; s < 3; ++s) {
            const size_t start = starts[s];
            int bad = 0;
            uint64_t leaves = 0, nodes = 0, result = 0;
            for (size_t i = 0; i < query_count; ++i) {
                const T* q = &queries[6 * i];
                auto reference = [&](auto& leaf_fn, auto& node_fn) {
                    bvh::v2::SmallStack<typename Node::Index, 256> stack;
                    if (kind == 1 || kind == 5) bvh.template traverse_top_down<true>(bvh.nodes[start].index, stack, leaf_fn, node_fn);
                    else                        bvh.template traverse_top_down<false>(bvh.nodes[start].index, stack, leaf_fn, node_fn);
                };
                auto device = [&](auto& leaf_fn, auto& node_fn) {
                    typename View::template SmallStack<256> stack;
                    auto pick = [&](const typename View::Node& l, const typename View::Node& r) {
                        const auto [a, b, c] = node_fn(l, r);
                        return dq::Pick { a, b, c };
                    };
                    // odd kinds through an aggregate, even ones with the tuple itself
                    if (kind == 1 || kind == 5) view.template traverse_top_down<true>(view.node(start).index, stack, leaf_fn, pick);
                    else if (kind == 3)         view.template traverse_top_down<false>(view.node(start).index, stack, leaf_fn, pick);
                    else                        view.template traverse_top_down<false>(view.node(start).index, stack, leaf_fn, node_fn);
                };
                const Record want = run_kind<T>(kind, q, boxes, [&](size_t k) { return (uint64_t)bvh.prim_ids[k]; }, reference);
                const Record got = run_kind<T>(kind, q, boxes, [&](size_t k) { return (uint64_t)view.prim_id(k); }, device);
                leaves += got.leaves; nodes += got.nodes; result += got.r0 + got.r1;
                if (got.leaves != want.leaves || got.nodes != want.nodes || got.hash != want.hash || got.r0 != want.r0 ||
                    got.r1 != want.r1) {
                    if (bad < 3) std::printf("  query %zu: leaves %llu/%llu nodes %llu/%llu result %llu/%llu\n", i,
                                             (unsigned long long)got.leaves, (unsigned long long)want.leaves,
                                             (unsigned long long)got.nodes, (unsigned long long)want.nodes,
                                             (unsigned long long)got.r0, (unsigned long long)want.r0);
                    ++bad;
                }
            }
            std::printf("kind %d start %d mismatches %d leaf_calls %llu node_calls %llu result %llu\n", kind, s, bad,
                        (unsigned long long)leaves, (unsigned long long)nodes, (unsigned long long)result);
            failures += bad;
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
