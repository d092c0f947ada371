// tests/device_bottom_up_kernels.cu — test entry points for DeviceView::traverse_bottom_up and the three-argument node
// test of DeviceView::traverse_top_down (include/bvh/v2/cuda/intersect.cuh).
//
// Compiled for sm_90a with the library's NVCC_FLAGS (--fmad=false among them) into
// tests/_build/libdevice_bottom_up_kernels.so (bvh_b200/build_ext.py build_device_bottom_up_tests) and driven by
// tests/test_device_bottom_up_gpu.py and scripts/bottom_up_bench.py.  Every entry point takes device pointers, launches
// on the handle's stream without waiting for it, and returns 0, or -1 with a message in bu_last_error().
//   bu_workspace_bytes*  DeviceView::bottom_up_workspace_bytes of the handle's tree
//   bu_count_box*        the pass with bu::CountBox: subtree primitive counts and box unions
//   bu_audit*            the pass with bu::Audit: calls per node and kind, inner calls made before a child's
//   bu_mass*             the pass with bu::MassCentre: subtree mass and centre of mass
//   bu_potential*        bu::Potential per point through traverse_top_down with the three-argument node test
// The functions are those of tests/device_bottom_up.h, which the host harness runs through the header's host pass.
#include <cuda_runtime.h>

#include "device_bottom_up.h"

#include <stdexcept>
#include <string>

namespace {

using bvh::v2::cuda::DeviceView;

thread_local std::string g_error;

constexpr unsigned kBlock = 128;
constexpr unsigned kSmallStack = 128;

template <typename T> struct Api;
template <> struct Api<float> {
    using Handle = bvh3f; using View = bvh_device_view3f;
    static int view(Handle* h, View* v) { return bvh3f_get_device_view(h, v); }
};
template <> struct Api<double> {
    using Handle = bvh3d; using View = bvh_device_view3d;
    static int view(Handle* h, View* v) { return bvh3d_get_device_view(h, v); }
};

template <typename T> int get_view(typename Api<T>::Handle* h, DeviceView<T>& view) {
    typename Api<T>::View c {};
    if (!h || Api<T>::view(h, &c)) { g_error = h ? bvh_last_error() : "null handle"; return -1; }
    try { view = DeviceView<T>::from(c, kSmallStack); } catch (const std::exception& e) { g_error = e.what(); return -1; }
    return 0;
}

// One pass with `fn` as both the leaf and the inner function.
template <typename T, typename Fn> int pass(typename Api<T>::Handle* h, void* workspace, size_t bytes, const Fn& fn) {
    DeviceView<T> view;
    if (get_view(h, view)) return -1;
    try {
        view.traverse_bottom_up(workspace, bytes, fn, fn);
    } catch (const std::exception& e) {
        g_error = e.what();
        return -1;
    }
    return 0;
}

template <typename T> int workspace_bytes(typename Api<T>::Handle* h, size_t* bytes) {
    DeviceView<T> view;
    if (get_view(h, view)) return -1;
    *bytes = view.bottom_up_workspace_bytes();
    return 0;
}

template <typename T>
int count_box(typename Api<T>::Handle* h, void* workspace, size_t bytes, const T* boxes, uint32_t* counts, T* node_boxes) {
    DeviceView<T> view;
    if (get_view(h, view)) return -1;
    return pass<T>(h, workspace, bytes, bu::CountBox<T> { view.prim_ids, boxes, counts, node_boxes });
}

template <typename T>
int audit(typename Api<T>::Handle* h, void* workspace, size_t bytes, uint32_t* leaf_calls, uint32_t* inner_calls, uint32_t* marks,
          uint32_t* errors) {
    return pass<T>(h, workspace, bytes, bu::Audit { leaf_calls, inner_calls, marks, errors });
}

template <typename T>
int mass(typename Api<T>::Handle* h, void* workspace, size_t bytes, const T* pos, const T* m, T* node_mass, T* node_centre) {
    DeviceView<T> view;
    if (get_view(h, view)) return -1;
    return pass<T>(h, workspace, bytes, bu::MassCentre<T> { view.prim_ids, pos, m, node_mass, node_centre });
}

template <typename T>
__global__ void __launch_bounds__(kBlock)
potential_kernel(DeviceView<T> view, const T* pos, const T* m, const T* node_mass, const T* node_centre, const T* points,
                 size_t count, T theta2, T eps2, T* phi, uint32_t* approximated) {
    using Node = typename DeviceView<T>::Node;
    const size_t i = (size_t)blockIdx.x * kBlock + threadIdx.x;
    if (i >= count) return;
    const T p[3] = { points[3 * i], points[3 * i + 1], points[3 * i + 2] };
    bu::Potential<T> pot { view.prim_ids, pos, m, node_mass, node_centre, p, theta2, eps2 };
    typename DeviceView<T>::template SmallStack<kSmallStack> stack;
    view.template traverse_top_down<false>(view.root_index(), stack,
        [&](size_t begin, size_t end) { return pot.leaf(begin, end); },
        [&](const Node& l, const Node& r, size_t left) { return pot.node(l.bounds, r.bounds, left); });
    phi[i] = pot.sum;
    if (approximated) approximated[i] = pot.approximated;
}

template <typename T>
int potential(typename Api<T>::Handle* h, const T* pos, const T* m, const T* node_mass, const T* node_centre, const T* points,
              size_t count, T theta2, T eps2, T* phi, uint32_t* approximated) {
    if (!pos || !m || !node_mass || !node_centre || !points || !phi) { g_error = "null argument"; return -1; }
    DeviceView<T> view;
    if (get_view(h, view)) return -1;
    if (count == 0) return 0;
    cudaError_t e = cudaSetDevice(view.device);
    if (e == cudaSuccess) {
        potential_kernel<T><<<(unsigned)((count + kBlock - 1) / kBlock), kBlock, 0, static_cast<cudaStream_t>(view.stream)>>>(
            view, pos, m, node_mass, node_centre, points, count, theta2, eps2, phi, approximated);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { g_error = std::string("potential_kernel: ") + cudaGetErrorString(e); return -1; }
    return 0;
}

} // namespace

#define BU_EXPORT extern "C" __attribute__((visibility("default")))
#define BU_ENTRY(T, S)                                                                                                 \
    BU_EXPORT int bu_workspace_bytes##S(bvh##S* h, size_t* bytes) { return workspace_bytes<T>(h, bytes); }            \
    BU_EXPORT int bu_count_box##S(bvh##S* h, void* ws, size_t bytes, const T* boxes, uint32_t* counts, T* node_boxes) { \
        return count_box<T>(h, ws, bytes, boxes, counts, node_boxes); }                                                \
    BU_EXPORT int bu_audit##S(bvh##S* h, void* ws, size_t bytes, uint32_t* leaf_calls, uint32_t* inner_calls,          \
                              uint32_t* marks, uint32_t* errors) {                                                     \
        return audit<T>(h, ws, bytes, leaf_calls, inner_calls, marks, errors); }                                       \
    BU_EXPORT int bu_mass##S(bvh##S* h, void* ws, size_t bytes, const T* pos, const T* m, T* node_mass, T* node_centre) { \
        return mass<T>(h, ws, bytes, pos, m, node_mass, node_centre); }                                                \
    BU_EXPORT int bu_potential##S(bvh##S* h, const T* pos, const T* m, const T* node_mass, const T* node_centre,        \
                                  const T* points, size_t count, T theta2, T eps2, T* phi, uint32_t* approximated) {    \
        return potential<T>(h, pos, m, node_mass, node_centre, points, count, theta2, eps2, phi, approximated); }

BU_ENTRY(float, 3f)
BU_ENTRY(double, 3d)

BU_EXPORT const char* bu_last_error() { return g_error.c_str(); }
