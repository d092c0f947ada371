// tests/device_bottom_up_host_test.cpp — DeviceView::traverse_bottom_up and the three-argument node test of
// DeviceView::traverse_top_down (include/bvh/v2/cuda/intersect.cuh) compiled as plain host C++, against
// Bvh<Node>::traverse_bottom_up, Bvh<Node>::refit and Bvh<Node>::traverse_top_down of the C++ surface
// (include/bvh/v2/b200_surface.h).  Driven by tests/test_device_bottom_up_host.py and tests/test_device_bottom_up_gpu.py.
//
//   device_bottom_up_host_test check <case.bin> f|d
// case.bin: u64 node_count, prim_count, query_count; the reference-layout nodes; u64 prim_ids; the primitives' boxes
// (min3, max3) in original order; the query boxes (min3, max3).  Prints one line per check, each with its mismatch count:
//   sequence calls C leaves L inners I mismatches M      the (leaf or inner, index) call sequence of both passes
//   counts mismatches M                                  subtree primitive counts (bu::CountBox)
//   boxes mismatches M                                   box unions (bu::CountBox) against Bvh::refit, bit for bit
//   audit mismatches M                                   one call per node of the right kind, children first (bu::Audit)
//   node_index kind K start S mismatches M node_calls N leaf_calls L
//                                                        the three-argument node test (kind 0: box overlap, 1: accept
//                                                        all; start 0: the root, 1: node 1, 2: the first leaf): its
//                                                        left_index sequence against `&left - nodes.data()` on the C++
//                                                        surface, and its leaf calls and result against the two-argument
//                                                        form's
//   workspace mismatches M                               a workspace one byte too small, and none, throw length_error
//
//   device_bottom_up_host_test physics <case.bin> f|d <out.bin>
// case.bin: u64 node_count, prim_count, point_count; the reference-layout nodes; u64 prim_ids; T pos[prim_count][3];
// T mass[prim_count]; T points[point_count][3]; T theta2, eps2.  Runs bu::MassCentre through the host pass and
// bu::Potential through the three-argument traverse_top_down; out.bin: T node_mass[node_count],
// T node_centre[node_count][3], T phi[point_count], u32 approximated[point_count].
#include <bvh/v2/bvh.h>
#include <bvh/v2/stack.h>

#include "device_bottom_up.h"

#include <cstdio>
#include <cstring>
#include <fstream>
#include <limits>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

namespace {

template <typename T> struct Tree {
    using Node = bvh::v2::Node<T, 3>;
    bvh::v2::Bvh<Node> bvh;
    std::vector<bvhb200::DevNode<T>> dev_nodes;
    std::vector<uint32_t> ids32;
    bvh::v2::cuda::DeviceView<T> view;

    // the reference-layout nodes and u64 ids, and the device layout as bvhNN_get_device_view reports it
    bool read(std::ifstream& in, size_t node_count, size_t prim_count) {
        bvh.nodes.resize(node_count);
        in.read((char*)bvh.nodes.data(), node_count * sizeof(Node));
        std::vector<uint64_t> ids(prim_count);
        in.read((char*)ids.data(), prim_count * 8);
        bvh.prim_ids.assign(ids.begin(), ids.end());
        dev_nodes.resize(node_count + 1);
        std::memset(dev_nodes.data(), 0, dev_nodes.size() * sizeof(dev_nodes[0]));
        for (size_t i = 0; i < node_count; ++i) {
            for (int k = 0; k < 6; ++k) dev_nodes[i + 1].bounds[k] = bvh.nodes[i].bounds[k];
            dev_nodes[i + 1].index = bvh.nodes[i].index.value;
        }
        ids32.assign(ids.begin(), ids.end());
        view.nodes = dev_nodes.data(); view.prim_ids = ids32.data();
        view.node_count = node_count; view.prim_count = prim_count;
        return (bool)in;
    }
    std::vector<unsigned char> workspace() const { return std::vector<unsigned char>(view.bottom_up_workspace_bytes()); }
};

template <typename T> std::vector<T> read_array(std::ifstream& in, size_t n) {
    std::vector<T> v(n);
    in.read((char*)v.data(), n * sizeof(T));
    return v;
}

// (leaf or inner, index) as one value
uint64_t call(bool leaf, size_t i) { return 2 * (uint64_t)i + (leaf ? 1 : 0); }

template <typename T> int check(std::ifstream& in) {
    uint64_t head[3];
    in.read((char*)head, sizeof head);
    Tree<T> t;
    if (!t.read(in, head[0], head[1])) { std::puts("short input"); return 2; }
    const size_t n = head[0], prims = head[1], query_count = head[2];
    const std::vector<T> boxes = read_array<T>(in, 6 * prims), queries = read_array<T>(in, 6 * query_count);
    if (!in) { std::puts("short input"); return 2; }
    auto& bvh = t.bvh;
    const auto& view = t.view;
    using Node = typename Tree<T>::Node;
    int failures = 0;

    // the call sequence
    std::vector<uint64_t> want, got;
    bvh.traverse_bottom_up([&](Node& node) { want.push_back(call(true, &node - bvh.nodes.data())); },
                           [&](Node& node) { want.push_back(call(false, &node - bvh.nodes.data())); });
    {
        auto ws = t.workspace();
        view.traverse_bottom_up(ws.data(), ws.size(), [&](size_t i, size_t, size_t) { got.push_back(call(true, i)); },
                                [&](size_t i, size_t) { got.push_back(call(false, i)); });
    }
    size_t bad = want.size() != got.size() ? 1 : 0, leaves = 0;
    for (size_t k = 0; k < want.size() && k < got.size(); ++k) bad += want[k] != got[k];
    for (uint64_t c : got) leaves += c & 1;
    std::printf("sequence calls %zu leaves %zu inners %zu mismatches %zu\n", got.size(), leaves, got.size() - leaves, bad);
    failures += (int)bad;

    // subtree counts and box unions, twice through the same workspace
    std::vector<uint32_t> counts(n, ~0u), want_counts(n, 0);
    std::vector<T> node_boxes(6 * n, std::numeric_limits<T>::quiet_NaN());
    {
        auto ws = t.workspace();
        const bu::CountBox<T> pass { t.ids32.data(), boxes.data(), counts.data(), node_boxes.data() };
        view.traverse_bottom_up(ws.data(), ws.size(), pass, pass);
        std::vector<uint32_t> first = counts;
        view.traverse_bottom_up(ws.data(), ws.size(), pass, pass);
        bad = first != counts;
    }
    bvh.traverse_bottom_up([&](Node& node) { want_counts[&node - bvh.nodes.data()] = (uint32_t)node.index.prim_count(); },
                           [&](Node& node) {
                               const size_t f = node.index.first_id();
                               want_counts[&node - bvh.nodes.data()] = want_counts[f] + want_counts[f + 1];
                           });
    for (size_t i = 0; i < n; ++i) bad += counts[i] != want_counts[i];
    std::printf("counts mismatches %zu\n", bad);
    failures += (int)bad;
    bvh.refit([&](Node& node) {
        auto b = bvh::v2::BBox<T, 3>::make_empty();
        for (size_t k = node.index.first_id(); k < node.index.first_id() + node.index.prim_count(); ++k) {
            const T* p = &boxes[6 * bvh.prim_ids[k]];
            b.extend(bvh::v2::BBox<T, 3>(bvh::v2::Vec<T, 3>(p[0], p[1], p[2]), bvh::v2::Vec<T, 3>(p[3], p[4], p[5])));
        }
        node.set_bbox(b);
    });
    bad = 0;
    for (size_t i = 0; i < n; ++i) bad += std::memcmp(&node_boxes[6 * i], bvh.nodes[i].bounds.data(), 6 * sizeof(T)) != 0;
    std::printf("boxes mismatches %zu\n", bad);
    failures += (int)bad;

    // the rules
    {
        std::vector<uint32_t> leaf_calls(n), inner_calls(n), marks(n), errors(1);
        auto ws = t.workspace();
        const bu::Audit audit { leaf_calls.data(), inner_calls.data(), marks.data(), errors.data() };
        view.traverse_bottom_up(ws.data(), ws.size(), audit, audit);
        bad = errors[0];
        for (size_t i = 0; i < n; ++i) {
            const bool leaf = bvh.nodes[i].is_leaf();
            bad += leaf_calls[i] != (leaf ? 1u : 0u) || inner_calls[i] != (leaf ? 0u : 1u);
        }
        std::printf("audit mismatches %zu\n", bad);
        failures += (int)bad;
    }

    // the three-argument node test
    size_t first_leaf = 0;
    while (first_leaf < n && !bvh.nodes[first_leaf].is_leaf()) ++first_leaf;
    const size_t starts[3] = { 0, n > 1 ? size_t(1) : size_t(0), first_leaf };
    for (int kind = 0; kind < 2; ++kind) {
        for (int s = 0; s < 3; ++s) {
            bad = 0;
            size_t node_calls = 0, leaf_calls = 0;
            for (size_t qi = 0; qi < query_count; ++qi) {
                const T* q = &queries[6 * qi];
                auto test = [&](const auto& l, const auto& r) {
                    return kind == 0 ? dq::Pick { dq::overlaps<T>(l.bounds, q), dq::overlaps<T>(r.bounds, q), false }
                                     : dq::Pick { true, true, false };
                };
                std::vector<uint64_t> want_index, got_index, want_leaves, got_leaves, two_leaves;
                bvh::v2::SmallStack<typename Node::Index, 256> ref_stack;
                bvh.template traverse_top_down<false>(bvh.nodes[starts[s]].index, ref_stack,
                    [&](size_t b, size_t e) { want_leaves.push_back(dq::mix(b, e)); return false; },
                    [&](const Node& l, const Node& r) {
                        want_index.push_back(&l - bvh.nodes.data());
                        const dq::Pick p = test(l, r);
                        return std::make_tuple(p.hit_left, p.hit_right, p.should_swap);
                    });
                typename bvh::v2::cuda::DeviceView<T>::template SmallStack<256> stack;
                using VNode = typename bvh::v2::cuda::DeviceView<T>::Node;
                view.template traverse_top_down<false>(view.node(starts[s]).index, stack,
                    [&](size_t b, size_t e) { got_leaves.push_back(dq::mix(b, e)); return false; },
                    [&](const VNode& l, const VNode& r, size_t left) { got_index.push_back(left); return test(l, r); });
                view.template traverse_top_down<false>(view.node(starts[s]).index, stack,
                    [&](size_t b, size_t e) { two_leaves.push_back(dq::mix(b, e)); return false; },
                    [&](const VNode& l, const VNode& r) { return test(l, r); });
                bad += want_index != got_index || want_leaves != got_leaves || two_leaves != got_leaves;
                node_calls += got_index.size();
                leaf_calls += got_leaves.size();
            }
            std::printf("node_index kind %d start %d mismatches %zu node_calls %zu leaf_calls %zu\n", kind, s, bad, node_calls,
                        leaf_calls);
            failures += (int)bad;
        }
    }

    // the workspace check
    bad = 0;
    {
        auto ws = t.workspace();
        auto nothing = [](size_t, size_t) {};
        auto leaf_nothing = [](size_t, size_t, size_t) {};
        try { view.traverse_bottom_up(ws.data(), ws.size() - 1, leaf_nothing, nothing); ++bad; }
        catch (const std::length_error& e) { bad += std::string(e.what()).find("too small") == std::string::npos; }
        try { view.traverse_bottom_up(nullptr, ws.size(), leaf_nothing, nothing); ++bad; }
        catch (const std::length_error&) {}
    }
    std::printf("workspace mismatches %zu\n", bad);
    failures += (int)bad;
    return failures;
}

template <typename T> int physics(std::ifstream& in, const char* out_path) {
    uint64_t head[3];
    in.read((char*)head, sizeof head);
    Tree<T> t;
    if (!t.read(in, head[0], head[1])) { std::puts("short input"); return 2; }
    const size_t n = head[0], prims = head[1], m = head[2];
    const std::vector<T> pos = read_array<T>(in, 3 * prims), mass = read_array<T>(in, prims), points = read_array<T>(in, 3 * m),
                         params = read_array<T>(in, 2);
    if (!in) { std::puts("short input"); return 2; }
    std::vector<T> node_mass(n), node_centre(3 * n), phi(m);
    std::vector<uint32_t> approximated(m);
    auto ws = t.workspace();
    const bu::MassCentre<T> mc { t.ids32.data(), pos.data(), mass.data(), node_mass.data(), node_centre.data() };
    t.view.traverse_bottom_up(ws.data(), ws.size(), mc, mc);
    using VNode = typename bvh::v2::cuda::DeviceView<T>::Node;
    for (size_t i = 0; i < m; ++i) {
        bu::Potential<T> pot { t.ids32.data(), pos.data(), mass.data(), node_mass.data(), node_centre.data(), &points[3 * i],
                               params[0], params[1] };
        typename bvh::v2::cuda::DeviceView<T>::template SmallStack<256> stack;
        t.view.template traverse_top_down<false>(t.view.root_index(), stack,
            [&](size_t b, size_t e) { return pot.leaf(b, e); },
            [&](const VNode& l, const VNode& r, size_t left) { return pot.node(l.bounds, r.bounds, left); });
        phi[i] = pot.sum;
        approximated[i] = pot.approximated;
    }
    std::ofstream out(out_path, std::ios::binary);
    out.write((const char*)node_mass.data(), n * sizeof(T));
    out.write((const char*)node_centre.data(), 3 * n * sizeof(T));
    out.write((const char*)phi.data(), m * sizeof(T));
    out.write((const char*)approximated.data(), m * sizeof(uint32_t));
    return out ? 0 : 1;
}

} // namespace

int main(int argc, char** argv) {
    if (argc < 4) return 2;
    const std::string mode = argv[1];
    std::ifstream in(argv[2], std::ios::binary);
    if (!in) return 2;
    const bool dbl = argv[3][0] == 'd';
    if (mode == "physics" && argc == 5) return dbl ? physics<double>(in, argv[4]) : physics<float>(in, argv[4]);
    if (mode != "check") return 2;
    const int failures = dbl ? check<double>(in) : check<float>(in);
    std::printf("failures %d\n", failures);
    return failures ? 1 : 0;
}
