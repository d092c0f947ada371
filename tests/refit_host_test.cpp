// The refit pass of bvh_b200/csrc/refit_core.cuh compiled by g++ as host code (tests/test_refit_boxes_host.py).
//
//   refit_host_test <case.bin> f|d <out.bin>
// case.bin: u64 node_count, prim_count, order_count; u64 index[node_count] (reference layout); u64 prim_ids[prim_count];
//           T boxes[prim_count][6] (min xyz, max xyz, original order); u64 order[order_count] (reference node indices, the
//           order in which the per-slot step runs: the GPU's arrival order is arbitrary).
// out.bin:  T bounds[node_count][6] (minx, maxx, miny, maxy, minz, maxz).  Every record starts as NaN, so a node the pass
//           never writes shows up in the comparison.
#include <cstdio>
#include <fstream>
#include <limits>
#include <vector>

#include "refit_core.cuh"

using namespace bvhb200;

template <typename T> int run(std::ifstream& in, const char* out_path) {
    using U = typename Real<T>::UInt;
    uint64_t head[3];
    in.read(reinterpret_cast<char*>(head), sizeof head);
    const size_t node_count = head[0], prim_count = head[1], order_count = head[2];
    std::vector<uint64_t> index(node_count), ids64(prim_count), order(order_count);
    std::vector<T> boxes(6 * prim_count);
    in.read(reinterpret_cast<char*>(index.data()), node_count * 8);
    in.read(reinterpret_cast<char*>(ids64.data()), prim_count * 8);
    in.read(reinterpret_cast<char*>(boxes.data()), boxes.size() * sizeof(T));
    in.read(reinterpret_cast<char*>(order.data()), order_count * 8);
    if (!in) { std::fprintf(stderr, "short case file\n"); return 1; }

    const size_t slots = node_count + 1;
    std::vector<DevNode<T>> nodes(slots);
    for (size_t i = 0; i < slots; ++i) {
        for (T& b : nodes[i].bounds) b = std::numeric_limits<T>::quiet_NaN();
        nodes[i].index = i ? (U)index[i - 1] : 0;
        nodes[i].pad = 0;
    }
    std::vector<uint32_t> prim_ids(prim_count), parent(slots, 0);
    for (size_t k = 0; k < prim_count; ++k) prim_ids[k] = (uint32_t)ids64[k];
    std::vector<int> flags(slots, -1);
    for (size_t i = 1; i < slots; ++i) refit_link(nodes.data(), slots, i, parent.data(), flags.data());
    const BoxSource<T> source{ boxes.data() };
    for (uint64_t r : order) refit_from_leaf(nodes.data(), (size_t)r + 1, parent.data(), flags.data(), prim_ids.data(), source);

    std::ofstream out(out_path, std::ios::binary);
    for (size_t i = 1; i < slots; ++i) out.write(reinterpret_cast<const char*>(nodes[i].bounds), 6 * sizeof(T));
    return out ? 0 : 1;
}

int main(int argc, char** argv) {
    if (argc != 4) { std::fprintf(stderr, "usage: %s case.bin f|d out.bin\n", argv[0]); return 2; }
    std::ifstream in(argv[1], std::ios::binary);
    return argv[2][0] == 'd' ? run<double>(in, argv[3]) : run<float>(in, argv[3]);
}
