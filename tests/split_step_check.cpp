// tests/split_step_check.cpp — one closest-hit inner step of the traversal (traverse_core.cuh inner_step, which for
// float tests the x/y half of each child first and loads the z half only when that does not already reject it; double
// loads whole nodes) against the decision taken from
// the full node_test of both children, for given sibling pairs and rays.  Compiled with g++ by
// tests/test_split_node_fetch.py.
#include <cstdint>
#include <cstring>

#include "traverse_core.cuh"

using namespace bvhb200;

namespace {

template <typename U> struct Stack {
    U data[4];
    uint32_t sp = 0;
    void push(U v) { data[sp++] = v; }
    bool try_pop(U& out) { if (sp == 0) return false; out = data[--sp]; return true; }
};

// pairs: per case 3 device slots (slot 0 padding, slots 1, 2 the children), rays: 8 scalars per case.  face_mode per
// case: 0 keeps tmin / tmax, 1 sets tmax to the left child's far plane on axis (case % 3), 2 sets tmin to its near
// plane, computed with node_test's arithmetic after the prologue.  out per case: step top, pushed entry (or ~0),
// full-test top, full-test pushed entry.
template <typename T, bool kRobust>
void check(const DevNode<T>* nodes, const T* rays, const uint8_t* face_mode, size_t m, uint64_t* out) {
    using U = typename Real<T>::UInt;
    const U sentinel = (U)0x0ABCDEF0;                          // what the pop returns: a stacked entry below the step
    for (size_t i = 0; i < m; ++i) {
        const DevNode<T>* pair = nodes + 3 * i;
        RayCtx<T> r;
        for (int k = 0; k < 3; ++k) { r.org[k] = rays[8 * i + k]; r.dir[k] = rays[8 * i + 3 + k]; }
        r.tmin = rays[8 * i + 6]; r.tmax = rays[8 * i + 7];
        ray_prologue<T, kRobust>(r);
        if (face_mode[i]) {
            const int axis = (int)(i % 3);
            RayCtx<T> one = r;                                 // the plane distances of that axis alone
            one.tmin = -Real<T>::max(); one.tmax = Real<T>::max();
            T tn = one.tmin, tf = one.tmax;
            if (axis == 0)      node_test_axes<T, kRobust, 0, 1>(pair[1].bounds, one, tn, tf);
            else if (axis == 1) node_test_axes<T, kRobust, 1, 2>(pair[1].bounds, one, tn, tf);
            else                node_test_axes<T, kRobust, 2, 3>(pair[1].bounds, one, tn, tf);
            if (face_mode[i] == 1) r.tmax = tf; else r.tmin = tn;
        }
        if (ray_interval_is_nan(r)) { out[4 * i] = out[4 * i + 1] = out[4 * i + 2] = out[4 * i + 3] = 0; continue; }
        Stack<U> st;
        st.push(sentinel);
        U top = 0;                                             // index_first(0) = 0: children at slots 1, 2 of `pair`
        inner_step<T, false, kRobust>(pair, r, top, st);
        U pushed = ~(U)0, v;
        if (st.sp == 2 && st.try_pop(v)) pushed = v;
        out[4 * i] = (uint64_t)top; out[4 * i + 1] = (uint64_t)pushed;
        // the decision from the full test (reference bvh.h:167-181)
        T l0, l1, r0, r1;
        node_test<T, kRobust>(pair[1].bounds, r, l0, l1);
        node_test<T, kRobust>(pair[2].bounds, r, r0, r1);
        const bool hl = l0 <= l1, hr = r0 <= r1;
        U want_top, want_push = ~(U)0;
        if (hl && hr) {
            const bool rf = l0 > r0;
            want_top = rf ? pair[2].index : pair[1].index;
            want_push = rf ? pair[1].index : pair[2].index;
        } else if (hl) want_top = pair[1].index;
        else if (hr) want_top = pair[2].index;
        else want_top = sentinel;
        out[4 * i + 2] = (uint64_t)want_top; out[4 * i + 3] = (uint64_t)want_push;
    }
}

} // namespace

extern "C" {
void split_step_check_3f(const void* nodes, const float* rays, const uint8_t* face, size_t m, int robust, uint64_t* out) {
    if (robust) check<float, true>((const DevNode<float>*)nodes, rays, face, m, out);
    else        check<float, false>((const DevNode<float>*)nodes, rays, face, m, out);
}
void split_step_check_3d(const void* nodes, const double* rays, const uint8_t* face, size_t m, int robust, uint64_t* out) {
    if (robust) check<double, true>((const DevNode<double>*)nodes, rays, face, m, out);
    else        check<double, false>((const DevNode<double>*)nodes, rays, face, m, out);
}
}
