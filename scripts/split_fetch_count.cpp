// scripts/split_fetch_count.cpp — counts, for every child box test of a traversal, which half of the 32-byte node
// (float; 64-byte for double) already rejects the box.  Built and called by scripts/split_fetch_count.py.
//
// The replay is the library's own stack machine (traverse_top_down + inner_step from traverse_core.cuh, compiled by g++
// as in the host emulation); the counting sits in its per-step hook, which sees the two children of the node about to
// be expanded, the ray's current interval and whether the ray has a hit yet.
#include <cstdint>
#include <vector>

#include "traverse_core.cuh"

using namespace bvhb200;

namespace {

template <typename U> struct CountStack {
    U data[256];
    uint32_t sp = 0;
    void push(U v) { data[sp++] = v; }
    bool try_pop(U& out) { if (sp == 0) return false; out = data[--sp]; return true; }
};

// out[((has_hit * 2 + xy_rejects) * 2 + z_rejects) * 2 + hit]: child box tests, by whether the ray had a hit before the
// step, whether the x/y half alone rejects the box, whether the z half alone does, and whether the full test hits it.
template <typename T, bool kAny>
void count(const DevNode<T>* nodes, const DevTri<T>* tris, const uint32_t* prim_ids, const T* rays, size_t m,
           uint64_t* out, uint64_t* steps_out) {
    using U = typename Real<T>::UInt;
    const U root = nodes[1].index;
    std::vector<uint64_t> total(16, 0);
    uint64_t steps = 0;
    #pragma omp parallel
    {
        uint64_t c[16] = {};
        uint64_t s = 0;
        #pragma omp for schedule(dynamic, 4096)
        for (long long i = 0; i < (long long)m; ++i) {
            RayCtx<T> r;
            const T* ray = rays + 8 * i;
            for (int k = 0; k < 3; ++k) { r.org[k] = ray[k]; r.dir[k] = ray[3 + k]; }
            r.tmin = ray[6]; r.tmax = ray[7];
            if (ray_interval_is_nan(r)) continue;
            ray_prologue<T, false>(r);
            HitState<T> hit { kInvalidId, r.tmax, (T)0, (T)0 };
            CountStack<U> stack;
            traverse_top_down<T, kAny, false>(
                nodes, r, root, stack,
                [&](U begin, U end) {
                    leaf_range<T>(tris, prim_ids, true, (uint32_t)begin, (uint32_t)(end - begin), r, hit, nullptr);
                    return hit.slot != kInvalidId;
                },
                [&](U first) {
                    ++s;
                    const unsigned has_hit = hit.slot != kInvalidId;
                    for (int side = 0; side < 2; ++side) {
                        const T* b = nodes[first + 1 + side].bounds;
                        T x0 = r.tmin, x1 = r.tmax, z0 = r.tmin, z1 = r.tmax, t0, t1;
                        node_test_axes<T, false, 0, 2>(b, r, x0, x1);
                        node_test_axes<T, false, 2, 3>(b, r, z0, z1);
                        node_test<T, false>(b, r, t0, t1);
                        ++c[((has_hit * 2 + !(x0 <= x1)) * 2 + !(z0 <= z1)) * 2 + (t0 <= t1)];
                    }
                });
        }
        #pragma omp critical
        {
            for (int k = 0; k < 16; ++k) total[k] += c[k];
            steps += s;
        }
    }
    for (int k = 0; k < 16; ++k) out[k] = total[k];
    *steps_out = steps;
}

} // namespace

extern "C" {
void count_split_fetch_3f(const void* nodes, const void* tris, const uint32_t* prim_ids, const float* rays, size_t m, int any,
                          uint64_t* out, uint64_t* steps) {
    if (any) count<float, true>((const DevNode<float>*)nodes, (const DevTri<float>*)tris, prim_ids, rays, m, out, steps);
    else     count<float, false>((const DevNode<float>*)nodes, (const DevTri<float>*)tris, prim_ids, rays, m, out, steps);
}
void count_split_fetch_3d(const void* nodes, const void* tris, const uint32_t* prim_ids, const double* rays, size_t m, int any,
                          uint64_t* out, uint64_t* steps) {
    if (any) count<double, true>((const DevNode<double>*)nodes, (const DevTri<double>*)tris, prim_ids, rays, m, out, steps);
    else     count<double, false>((const DevNode<double>*)nodes, (const DevTri<double>*)tris, prim_ids, rays, m, out, steps);
}
}
