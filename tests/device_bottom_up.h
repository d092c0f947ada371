// tests/device_bottom_up.h — leaf and inner functions of the DeviceView::traverse_bottom_up tests, and the Barnes-Hut
// query that reads their results, shared by the host harness (tests/device_bottom_up_host_test.cpp, g++) and the test
// kernels (tests/device_bottom_up_kernels.cu, nvcc --fmad=false), so that both sides run the same arithmetic.
//
// Each pass object serves as both functions: operator()(node, begin, end) is the leaf function and operator()(node,
// left) the inner one.  Node data is indexed by reference node index; node boxes are in the node layout (minx, maxx,
// miny, maxy, minz, maxz); primitive boxes are min3, max3 in the original order.
#pragma once

#include "device_queries.h"

#include <cmath>
#include <cstdint>

namespace bu {

template <typename T> BVH_HD void bump(T* p) {
#if defined(__CUDA_ARCH__)
    atomicAdd(p, T(1));
#else
    ++*p;
#endif
}

// Subtree primitive counts and box unions: a leaf folds its primitives' boxes into the empty box in BVH order, an inner
// node unions its children's (left first), the refit's order.
template <typename T> struct CountBox {
    const uint32_t* prim_ids;
    const T* boxes;
    uint32_t* counts;
    T* node_boxes;
    BVH_HD void operator()(size_t node, size_t begin, size_t end) const {
        using R = bvhb200::Real<T>;
        T b[6];
        for (int a = 0; a < 3; ++a) { b[2 * a] = R::max(); b[2 * a + 1] = R::neg(R::max()); }
        for (size_t k = begin; k < end; ++k) {
            const T* p = boxes + 6 * (size_t)prim_ids[k];
            for (int a = 0; a < 3; ++a) {
                b[2 * a] = bvhb200::robust_min(b[2 * a], p[a]);
                b[2 * a + 1] = bvhb200::robust_max(b[2 * a + 1], p[3 + a]);
            }
        }
        counts[node] = (uint32_t)(end - begin);
        for (int k = 0; k < 6; ++k) node_boxes[6 * node + k] = b[k];
    }
    BVH_HD void operator()(size_t node, size_t left) const {
        counts[node] = counts[left] + counts[left + 1];
        const T* l = node_boxes + 6 * left;
        const T* r = node_boxes + 6 * (left + 1);
        for (int k = 0; k < 6; ++k) node_boxes[6 * node + k] = k & 1 ? bvhb200::robust_max(l[k], r[k]) : bvhb200::robust_min(l[k], r[k]);
    }
};

// The rules themselves: calls per node and kind, and an error for every inner call made before both children's marks
// were set.  The arrays start zeroed.
struct Audit {
    uint32_t* leaf_calls;
    uint32_t* inner_calls;
    uint32_t* marks;
    uint32_t* errors;
    BVH_HD void operator()(size_t node, size_t, size_t) const {
        bump(leaf_calls + node);
        marks[node] = 1;
    }
    BVH_HD void operator()(size_t node, size_t left) const {
        bump(inner_calls + node);
        if (!marks[left] || !marks[left + 1]) bump(errors);
        marks[node] = 1;
    }
};

// Subtree mass and centre of mass.  pos: x, y, z per particle, mass per particle, both in the original order.
template <typename T> struct MassCentre {
    const uint32_t* prim_ids;
    const T* pos;
    const T* mass;
    T* node_mass;
    T* node_centre;
    BVH_HD void operator()(size_t node, size_t begin, size_t end) const {
        T m = T(0), c[3] = { T(0), T(0), T(0) };
        for (size_t k = begin; k < end; ++k) {
            const size_t id = prim_ids[k];
            m = m + mass[id];
            for (int a = 0; a < 3; ++a) c[a] = c[a] + mass[id] * pos[3 * id + a];
        }
        node_mass[node] = m;
        for (int a = 0; a < 3; ++a) node_centre[3 * node + a] = c[a] / m;
    }
    BVH_HD void operator()(size_t node, size_t left) const {
        const T ml = node_mass[left], mr = node_mass[left + 1], m = ml + mr;
        node_mass[node] = m;
        for (int a = 0; a < 3; ++a)
            node_centre[3 * node + a] = (ml * node_centre[3 * left + a] + mr * node_centre[3 * (left + 1) + a]) / m;
    }
};

// The softened potential -sum m / sqrt(d^2 + eps2) at one point, Barnes-Hut style: a child whose largest box extent s
// satisfies s^2 < theta2 * d^2 (d: distance to its centre of mass) counts as its mass at its centre and is not
// descended; theta2 = 0 opens every node (the exact sum, in the tree's order).
template <typename T> struct Potential {
    const uint32_t* prim_ids;
    const T* pos;
    const T* mass;
    const T* node_mass;
    const T* node_centre;
    const T* p;
    T theta2, eps2;
    T sum = T(0);
    uint32_t approximated = 0;
    BVH_HD T dist2(const T* c) const {
        T d = T(0);
        for (int a = 0; a < 3; ++a) { const T e = c[a] - p[a]; d = d + e * e; }
        return d;
    }
    BVH_HD bool leaf(size_t begin, size_t end) {
        using std::sqrt;
        for (size_t k = begin; k < end; ++k) {
            const size_t id = prim_ids[k];
            sum = sum - mass[id] / sqrt(dist2(pos + 3 * id) + eps2);
        }
        return false;
    }
    template <typename B> BVH_HD bool open(const B& b, size_t node) {
        using std::sqrt;
        const T x = b[1] - b[0], y = b[3] - b[2], z = b[5] - b[4];
        const T s = x > y ? (x > z ? x : z) : (y > z ? y : z);
        const T d2 = dist2(node_centre + 3 * node);
        if (s * s < theta2 * d2) {
            sum = sum - node_mass[node] / sqrt(d2 + eps2);
            ++approximated;
            return false;
        }
        return true;
    }
    template <typename B> BVH_HD dq::Pick node(const B& l, const B& r, size_t left) {
        const bool open_left = open(l, left);
        const bool open_right = open(r, left + 1);
        return dq::Pick { open_left, open_right, false };
    }
};

} // namespace bu
