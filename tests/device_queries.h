// tests/device_queries.h — node and primitive tests shared by the traverse_top_down tests (tests/device_query_host_test.cpp,
// tests/device_query_kernels.cu).  A box `b` is anything indexable in the node layout (minx, maxx, miny, maxy, minz,
// maxz): the bounds of the C++ surface's Node<T, 3> on the host and of DeviceView<T>::Node anywhere.  A query box `q`
// is min3, max3 (struct bvh_bboxNN); a point `p` is x, y, z.
#pragma once

#include <bvh/v2/cuda/intersect.cuh>

#include <cstdint>

namespace dq {

// what a node function returns here: an aggregate of three bools (the other tests return tuples)
struct Pick { bool hit_left, hit_right, should_swap; };

template <typename T, typename B> BVH_HD bool overlaps(const B& b, const T* q) {
    return b[0] <= q[3] && q[0] <= b[1] && b[2] <= q[4] && q[1] <= b[3] && b[4] <= q[5] && q[2] <= b[5];
}

template <typename T, typename B> BVH_HD bool contains(const B& b, const T* p) {
    return b[0] <= p[0] && p[0] <= b[1] && b[2] <= p[1] && p[1] <= b[3] && b[4] <= p[2] && p[2] <= b[5];
}

// squared distance from p to the box b (0 inside), summed x, y, z
template <typename T, typename B> BVH_HD T box_dist2(const B& b, const T* p) {
    T d = T(0);
    for (int a = 0; a < 3; ++a) {
        const T below = b[2 * a] - p[a], above = p[a] - b[2 * a + 1];
        const T e = below > above ? below : above;
        const T c = e > T(0) ? e : T(0);
        d = d + c * c;
    }
    return d;
}

// squared distance between two points, summed x, y, z
template <typename T> BVH_HD T point_dist2(const T* a, const T* p) {
    T d = T(0);
    for (int k = 0; k < 3; ++k) { const T e = a[k] - p[k]; d = d + e * e; }
    return d;
}

// a primitive box min3, max3 in the node layout
template <typename T> struct AsNode {
    const T* q;
    BVH_HD T operator[](int k) const { return q[(k & 1) * 3 + (k >> 1)]; }
};

// 64-bit hash of a leaf-call sequence, and a per-id hash whose sum over a set does not depend on the order
BVH_HD uint64_t mix(uint64_t h, uint64_t x) { return (h ^ x) * 1099511628211ull; }
constexpr uint64_t kHashSeed = 1469598103934665603ull;
BVH_HD uint64_t id_hash(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

} // namespace dq
