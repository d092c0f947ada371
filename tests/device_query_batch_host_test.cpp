// tests/device_query_batch_host_test.cpp — DeviceView::query (include/bvh/v2/cuda/intersect.cuh) compiled as plain host
// C++ and run on host copies of a tree, against Bvh<Node>::traverse_top_down of the C++ surface
// (include/bvh/v2/b200_surface.h) with the same node and leaf functions.
//
//   device_query_batch_host_test <case file> f|d   input as tests/device_query_host_test.cpp reads it (written by
//                                                   tests/test_device_query_batch_host.py).  For every node test below,
//                                                   in its two-argument and its three-argument form, it records per
//                                                   query the whole call sequence — each node call with the two
//                                                   children's packed indices and, in the three-argument form, the left
//                                                   child's reference index; each leaf call with its range — and compares
//                                                   it with the reference's.  It also checks that start and finish run once
//                                                   per query, start in index order, and prints one line per test and form:
//                                                     kind K form F mismatches M events E starts_ok S finishes_ok F
//                                                   then "empty batch ok, small workspace throws, null workspace throws".
//   device_query_batch_host_test plan               prints plan_query() (trace_plan.h): "refill_min R inner_budget B".
// Node tests: 0 overlap, 1 containment with IsAnyHit (a leaf that finds one ends the query), 2 nearest box (nearer child
// first; the leaf shrinks the radius the node test reads), 3 reject-all, 4 accept-all.
#include <bvh/v2/bvh.h>
#include <bvh/v2/stack.h>

#include "device_queries.h"

#include <array>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <stdexcept>
#include <tuple>
#include <vector>

namespace {

using Event = std::array<uint64_t, 4>;   // node: {0, left.index, right.index, left_index or ~0}; leaf: {1, begin, end, 0}
constexpr uint64_t kNoIndex = ~0ull;

enum Kind : int { kOverlap = 0, kContains = 1, kNearest = 2, kRejectAll = 3, kAcceptAll = 4, kKinds = 5 };

// The node test and the leaf of one query, on either side.  `best` is the nearest search's squared radius.
template <typename T> struct Logic {
    int kind;
    const T* q;
    const std::vector<T>* boxes;
    template <typename B> dq::Pick pick(const B& l, const B& r, T best) const {
        switch (kind) {
        case kOverlap: return dq::Pick { dq::overlaps<T>(l, q), dq::overlaps<T>(r, q), false };
        case kContains: return dq::Pick { dq::contains<T>(l, q), dq::contains<T>(r, q), false };
        case kNearest: {
            const T dl = dq::box_dist2<T>(l, q), dr = dq::box_dist2<T>(r, q);
            return dq::Pick { dl < best, dr < best, dl > dr };
        }
        case kRejectAll: return dq::Pick { false, false, false };
        default: return dq::Pick { true, true, false };
        }
    }
    // the primitive with original id `id`; true when a containment query found it
    bool visit(uint64_t id, T& best) const {
        const dq::AsNode<T> b { boxes->data() + 6 * id };
        if (kind == kContains) return dq::contains<T>(b, q);
        if (kind == kNearest) { const T d = dq::box_dist2<T>(b, q); if (d < best) best = d; }
        return false;
    }
};

struct Counters { std::vector<int> starts, finishes; std::vector<size_t> order; };

// A recording querier; kThreeArg selects the node function's form.
template <typename T, bool kThreeArg> struct Recorder;
template <typename T> struct RecorderBase {
    using Node = typename bvh::v2::cuda::DeviceView<T>::Node;
    struct Payload { size_t i; T best; };
    int kind;
    const std::vector<T>* queries;
    const std::vector<T>* boxes;
    const uint32_t* prim_ids;
    std::vector<std::vector<Event>>* log;
    Counters* counters;
    Logic<T> logic(size_t i) const { return Logic<T> { kind, queries->data() + 6 * i, boxes }; }
    void start(size_t i, Payload& p) const {
        p.i = i;
        p.best = T(1) / T(0);
        counters->starts[i] += 1;
        counters->order.push_back(i);
    }
    dq::Pick node_call(Payload& p, const Node& l, const Node& r, uint64_t left) const {
        (*log)[p.i].push_back(Event { 0, (uint64_t)l.index, (uint64_t)r.index, left });
        return logic(p.i).pick(l.bounds, r.bounds, p.best);
    }
    bool leaf(Payload& p, size_t begin, size_t end) const {
        (*log)[p.i].push_back(Event { 1, begin, end, 0 });
        bool found = false;
        for (size_t k = begin; k < end; ++k) found |= logic(p.i).visit(prim_ids[k], p.best);
        return found;
    }
    void finish(size_t i, const Payload& p) const {
        if (p.i != i) throw std::logic_error("finish with another query's payload");
        counters->finishes[i] += 1;
    }
};
template <typename T> struct Recorder<T, false> : RecorderBase<T> {
    using typename RecorderBase<T>::Payload;
    using typename RecorderBase<T>::Node;
    dq::Pick node(Payload& p, const Node& l, const Node& r) const { return this->node_call(p, l, r, kNoIndex); }
};
template <typename T> struct Recorder<T, true> : RecorderBase<T> {
    using typename RecorderBase<T>::Payload;
    using typename RecorderBase<T>::Node;
    dq::Pick node(Payload& p, const Node& l, const Node& r, size_t left) const { return this->node_call(p, l, r, left); }
};

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
    size_t depth = 0;
    std::vector<size_t> level(node_count, 0);
    for (size_t i = 0; i < node_count; ++i) {
        for (int k = 0; k < 6; ++k) dev_nodes[i + 1].bounds[k] = bvh.nodes[i].bounds[k];
        dev_nodes[i + 1].index = bvh.nodes[i].index.value;
        if (!bvh.nodes[i].is_leaf()) {
            const size_t c = bvh.nodes[i].index.first_id();
            level[c] = level[c + 1] = level[i] + 1;
            depth = std::max(depth, level[i] + 1);
        }
    }
    std::vector<uint32_t> ids32(ids.begin(), ids.end());
    View view;
    view.nodes = dev_nodes.data(); view.prim_ids = ids32.data();
    view.node_count = node_count; view.prim_count = prim_count; view.depth = depth;
    unsigned long long workspace = 0;

    int failures = 0;
    for (int kind = 0; kind < kKinds; ++kind) {
        for (int form = 0; form < 2; ++form) {
            // the reference: Bvh::traverse_top_down per query, with the same logic
            std::vector<std::vector<Event>> want(query_count), got(query_count);
            for (size_t i = 0; i < query_count; ++i) {
                const Logic<T> logic { kind, &queries[6 * i], &boxes };
                T best = T(1) / T(0);
                auto leaf_fn = [&](size_t begin, size_t end) {
                    want[i].push_back(Event { 1, begin, end, 0 });
                    bool found = false;
                    for (size_t k = begin; k < end; ++k) found |= logic.visit(bvh.prim_ids[k], best);
                    return found;
                };
                auto node_fn = [&](const Node& l, const Node& r) {
                    want[i].push_back(Event { 0, (uint64_t)l.index.value, (uint64_t)r.index.value,
                                              form ? (uint64_t)(&l - bvh.nodes.data()) : kNoIndex });
                    const dq::Pick d = logic.pick(l.bounds, r.bounds, best);
                    return std::make_tuple(d.hit_left, d.hit_right, d.should_swap);
                };
                bvh::v2::GrowingStack<typename Node::Index> stack;
                if (kind == kContains) bvh.template traverse_top_down<true>(bvh.get_root().index, stack, leaf_fn, node_fn);
                else                   bvh.template traverse_top_down<false>(bvh.get_root().index, stack, leaf_fn, node_fn);
            }
            Counters counters { std::vector<int>(query_count), std::vector<int>(query_count), {} };
            auto batch = [&](const auto& querier) {
                if (kind == kContains) view.template query<true>(query_count, querier, &workspace, sizeof(workspace));
                else                   view.template query<false>(query_count, querier, &workspace, sizeof(workspace));
            };
            if (form) batch(Recorder<T, true> { { kind, &queries, &boxes, ids32.data(), &got, &counters } });
            else      batch(Recorder<T, false> { { kind, &queries, &boxes, ids32.data(), &got, &counters } });
            int bad = 0;
            size_t events = 0;
            for (size_t i = 0; i < query_count; ++i) {
                events += got[i].size();
                if (got[i] != want[i]) {
                    if (bad < 3) std::printf("  kind %d form %d query %zu: %zu events, reference %zu\n", kind, form, i, got[i].size(), want[i].size());
                    ++bad;
                }
            }
            bool starts_ok = counters.order.size() == query_count, finishes_ok = true;
            for (size_t i = 0; i < query_count; ++i) {
                starts_ok = starts_ok && counters.starts[i] == 1 && counters.order[i] == i;
                finishes_ok = finishes_ok && counters.finishes[i] == 1;
            }
            std::printf("kind %d form %d mismatches %d events %zu starts_ok %d finishes_ok %d\n", kind, form, bad, events,
                        (int)starts_ok, (int)finishes_ok);
            failures += bad + !starts_ok + !finishes_ok;
        }
    }

    // n == 0 makes no call; a workspace that is too small, or none, throws before any call
    std::vector<std::vector<Event>> log(query_count);
    Counters counters { std::vector<int>(query_count), std::vector<int>(query_count), {} };
    const Recorder<T, false> rec { { kOverlap, &queries, &boxes, ids32.data(), &log, &counters } };
    view.template query<false>(0, rec, &workspace, sizeof(workspace));
    bool small_throws = false, null_throws = false;
    try { view.template query<false>(query_count, rec, &workspace, sizeof(workspace) - 1); } catch (const std::length_error&) { small_throws = true; }
    try { view.template query<false>(query_count, rec, nullptr, sizeof(workspace)); } catch (const std::length_error&) { null_throws = true; }
    if (counters.order.empty() && small_throws && null_throws && view.query_workspace_bytes() == sizeof(workspace))
        std::puts("empty batch ok, small workspace throws, null workspace throws");
    else
        ++failures;
    return failures;
}

} // namespace

int main(int argc, char** argv) {
    if (argc == 2 && std::strcmp(argv[1], "plan") == 0) {
        const bvhb200::QueryPlan plan = bvhb200::plan_query();
        std::printf("refill_min %u inner_budget %u\n", plan.refill_min, plan.inner_budget);
        return 0;
    }
    if (argc < 3) return 2;
    std::ifstream in(argv[1], std::ios::binary);
    if (!in) return 2;
    const int failures = argv[2][0] == 'd' ? run<double>(in) : run<float>(in);
    std::printf("failures %d\n", failures);
    return failures ? 1 : 0;
}
