// bvh_b200/csrc/core.cuh — per-ray and per-node arithmetic shared by every kernel.
//
// Everything here is written one IEEE-754 operation per call (round-to-nearest intrinsics on the
// device, plain operators compiled with -ffp-contract=off in the host-side emulation used by the
// CPU tests) and in the exact operation order of the reference, so that hit distances and
// barycentrics are bit-identical to the reference built with -ffp-contract=off:
//   ray prologue      reference bvh.h:161-165, ray.h:29-48, utils.h:46-63
//   ray/box slab test reference node.h:59-88,105-117 (octant-selected planes, NaN-swallowing order)
//   ray/triangle test reference tri.h:35-37,55-74 with dot = ((0+a0*b0)+a1*b1)+a2*b2 (vec.h:98-99)
//   bbox / centre     reference tri.h:24-25, bbox.h:23-38
// The header is also compiled by g++ (tests/host_emul.cpp) to check the logic without a GPU.
#pragma once

#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define BVH_HD __host__ __device__ __forceinline__
#else
#define BVH_HD inline
#endif

namespace bvhb200 {

constexpr uint32_t kInvalidId = 0xFFFFFFFFu;

// ---------------------------------------------------------------------------------------------
// Exactly-rounded scalar operations (never contracted into FMAs by the compiler).
// ---------------------------------------------------------------------------------------------
template <typename T> struct Real;

template <> struct Real<float> {
    using UInt = uint32_t;
    static constexpr int index_bits = 32;
    static BVH_HD float max() { return FLT_MAX; }
    static BVH_HD float eps() { return FLT_EPSILON; }
#if defined(__CUDA_ARCH__)
    static BVH_HD float add(float a, float b) { return __fadd_rn(a, b); }
    static BVH_HD float sub(float a, float b) { return __fsub_rn(a, b); }
    static BVH_HD float mul(float a, float b) { return __fmul_rn(a, b); }
    static BVH_HD float div(float a, float b) { return __fdiv_rn(a, b); }
    static BVH_HD float fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
    static BVH_HD uint32_t bits(float a) { return __float_as_uint(a); }
    static BVH_HD float from_bits(uint32_t u) { return __uint_as_float(u); }
#else
    static BVH_HD float add(float a, float b) { return a + b; }
    static BVH_HD float sub(float a, float b) { return a - b; }
    static BVH_HD float mul(float a, float b) { return a * b; }
    static BVH_HD float div(float a, float b) { return a / b; }
    static BVH_HD float fma(float a, float b, float c) { return __builtin_fmaf(a, b, c); }
    static BVH_HD uint32_t bits(float a) { uint32_t u; std::memcpy(&u, &a, 4); return u; }
    static BVH_HD float from_bits(uint32_t u) { float a; std::memcpy(&a, &u, 4); return a; }
#endif
    static BVH_HD bool is_finite(float a) { return (bits(a) & 0x7F800000u) != 0x7F800000u; }
    static BVH_HD bool sign(float a) { return (bits(a) >> 31) != 0; }
    static BVH_HD float neg(float a) { return from_bits(bits(a) ^ 0x80000000u); }
    static BVH_HD float abs(float a) { return from_bits(bits(a) & 0x7FFFFFFFu); }
};

template <> struct Real<double> {
    using UInt = uint64_t;
    static constexpr int index_bits = 64;
    static BVH_HD double max() { return DBL_MAX; }
    static BVH_HD double eps() { return DBL_EPSILON; }
#if defined(__CUDA_ARCH__)
    static BVH_HD double add(double a, double b) { return __dadd_rn(a, b); }
    static BVH_HD double sub(double a, double b) { return __dsub_rn(a, b); }
    static BVH_HD double mul(double a, double b) { return __dmul_rn(a, b); }
    static BVH_HD double div(double a, double b) { return __ddiv_rn(a, b); }
    static BVH_HD double fma(double a, double b, double c) { return __fma_rn(a, b, c); }
    static BVH_HD uint64_t bits(double a) { return (uint64_t)__double_as_longlong(a); }
    static BVH_HD double from_bits(uint64_t u) { return __longlong_as_double((long long)u); }
#else
    static BVH_HD double add(double a, double b) { return a + b; }
    static BVH_HD double sub(double a, double b) { return a - b; }
    static BVH_HD double mul(double a, double b) { return a * b; }
    static BVH_HD double div(double a, double b) { return a / b; }
    static BVH_HD double fma(double a, double b, double c) { return __builtin_fma(a, b, c); }
    static BVH_HD uint64_t bits(double a) { uint64_t u; std::memcpy(&u, &a, 8); return u; }
    static BVH_HD double from_bits(uint64_t u) { double a; std::memcpy(&a, &u, 8); return a; }
#endif
    static BVH_HD bool is_finite(double a) { return (bits(a) & 0x7FF0000000000000ull) != 0x7FF0000000000000ull; }
    static BVH_HD bool sign(double a) { return (bits(a) >> 63) != 0; }
    static BVH_HD double neg(double a) { return from_bits(bits(a) ^ 0x8000000000000000ull); }
    static BVH_HD double abs(double a) { return from_bits(bits(a) & 0x7FFFFFFFFFFFFFFFull); }
};

// reference utils.h:40-43 — the SECOND argument comes back when the first is a NaN
template <typename T> BVH_HD T robust_min(T a, T b) { return a < b ? a : b; }
template <typename T> BVH_HD T robust_max(T a, T b) { return a > b ? a : b; }

// ---------------------------------------------------------------------------------------------
// Device-side data layout (DESIGN.md "Data layout in HBM")
// ---------------------------------------------------------------------------------------------
// One node = the reference's Node<T,3> (bounds [minx,maxx,miny,maxy,minz,maxz] + packed index,
// node.h:31-37) padded to a power of two: 32 B for float, 64 B for double.  The device array is the
// reference's node array shifted by ONE slot (device slot = reference index + 1), which makes every
// sibling pair (reference indices 2k+1, 2k+2; bvh.h:34-51) one naturally aligned 64 B / 128 B line.
template <typename T> struct DevNode;
template <> struct alignas(32) DevNode<float>  { float  bounds[6]; uint32_t index; uint32_t pad; };
template <> struct alignas(64) DevNode<double> { double bounds[6]; uint64_t index; uint64_t pad; };
static_assert(sizeof(DevNode<float>) == 32 && sizeof(DevNode<double>) == 64, "packed node size");

// reference tri.h:30-37 (PrecomputedTri): p0, e1 = p0-p1, e2 = p2-p0, n = cross(e1, e2)
// PrecomputedTri (tri.h:30-37), packed: 48 / 96 bytes, three / six 128-bit loads per test.  The padded form (BVH_TRI_PAD:
// 64 / 128 bytes, four / eight 128-bit loads) costs 16 MB more footprint per million triangles; not measured on the H100.
#ifndef BVH_TRI_PAD
#define BVH_TRI_PAD 0              // 1: 64 / 128-byte records
#endif
#if BVH_TRI_PAD
template <typename T> struct alignas(16 * sizeof(T)) DevTri { T p0[3], e1[3], e2[3], n[3], pad[4]; };
static_assert(sizeof(DevTri<float>) == 64 && sizeof(DevTri<double>) == 128, "padded triangle size");
#else
template <typename T> struct alignas(16) DevTri { T p0[3], e1[3], e2[3], n[3]; };
static_assert(sizeof(DevTri<float>) == 48 && sizeof(DevTri<double>) == 96, "packed triangle size");
#endif

// bvh_ray3f / bvh_ray3d (reference c_api/bvh.h:70-73)
template <typename T> struct alignas(16) DevRay { T org[3], dir[3], tmin, tmax; };
static_assert(sizeof(DevRay<float>) == 32 && sizeof(DevRay<double>) == 64, "ray size");

// bvh_hit3f / bvh_hit3d (include/bvh_b200.h)
template <typename T> struct DevHit;
template <> struct alignas(16) DevHit<float>  { uint32_t prim_id; float t, u, v; };
template <> struct alignas(16) DevHit<double> { uint64_t prim_id; double t, u, v; };
static_assert(sizeof(DevHit<float>) == 16 && sizeof(DevHit<double>) == 32, "hit size");

// reference index.h:51-53,75-78: value = first_id << 4 | prim_count; leaf iff prim_count != 0
constexpr int kPrimCountBits = 4;
constexpr uint32_t kMaxLeafPrims = 15;
template <typename U> BVH_HD U index_first(U v) { return v >> kPrimCountBits; }
template <typename U> BVH_HD uint32_t index_count(U v) { return (uint32_t)(v & (U)kMaxLeafPrims); }
template <typename U> BVH_HD U make_index(U first, uint32_t count) { return (U)((first << kPrimCountBits) | (U)count); }

// ---------------------------------------------------------------------------------------------
// Geometry helpers
// ---------------------------------------------------------------------------------------------
template <typename T> BVH_HD T dot3(const T a[3], const T b[3]) {
    using R = Real<T>;
    T acc = R::add((T)0, R::mul(a[0], b[0]));      // 0 + x keeps the reference's -0 -> +0 behaviour
    acc = R::add(acc, R::mul(a[1], b[1]));
    acc = R::add(acc, R::mul(a[2], b[2]));
    return acc;
}

template <typename T> BVH_HD void cross3(const T a[3], const T b[3], T out[3]) {
    using R = Real<T>;
    T x = R::sub(R::mul(a[1], b[2]), R::mul(a[2], b[1]));
    T y = R::sub(R::mul(a[2], b[0]), R::mul(a[0], b[2]));
    T z = R::sub(R::mul(a[0], b[1]), R::mul(a[1], b[0]));
    out[0] = x; out[1] = y; out[2] = z;
}

// reference tri.h:35-37
template <typename T> BVH_HD DevTri<T> precompute_tri(const T v[9]) {
    using R = Real<T>;
    DevTri<T> t;
#if BVH_TRI_PAD
    for (int k = 0; k < 4; ++k) t.pad[k] = (T)0;
#endif
    for (int k = 0; k < 3; ++k) {
        t.p0[k] = v[k];
        t.e1[k] = R::sub(v[k], v[3 + k]);
        t.e2[k] = R::sub(v[6 + k], v[k]);
    }
    cross3(t.e1, t.e2, t.n);
    return t;
}

// reference tri.h:24-25: bbox = BBox(p0).extend(p1).extend(p2); centre = (p0+p1+p2) * T(1./3.)
template <typename T> BVH_HD void tri_bounds_center(const T v[9], T bmin[3], T bmax[3], T center[3]) {
    using R = Real<T>;
    const T third = (T)(1. / 3.);
    for (int k = 0; k < 3; ++k) {
        bmin[k] = robust_min(robust_min(v[k], v[3 + k]), v[6 + k]);
        bmax[k] = robust_max(robust_max(v[k], v[3 + k]), v[6 + k]);
        center[k] = R::mul(R::add(R::add(v[k], v[3 + k]), v[6 + k]), third);
    }
}

// reference bbox.h:32-38
template <typename T> BVH_HD T half_area(const T bmin[3], const T bmax[3]) {
    using R = Real<T>;
    T d0 = R::sub(bmax[0], bmin[0]), d1 = R::sub(bmax[1], bmin[1]), d2 = R::sub(bmax[2], bmin[2]);
    return R::add(R::mul(R::add(d0, d1), d2), R::mul(d0, d1));
}

// reference utils.h:58-63
template <typename T> BVH_HD T safe_inverse(T x) {
    using R = Real<T>;
    if (R::abs(x) <= R::eps()) return R::sign(x) ? R::neg(R::max()) : R::max();
    return R::div((T)1, x);
}

// reference utils.h:46-55
template <typename T> BVH_HD T add_ulp_magnitude(T t, unsigned ulp) {
    using R = Real<T>;
    if (!R::is_finite(t)) return t;
    return R::from_bits(R::bits(t) + (typename R::UInt)ulp);
}

// ---------------------------------------------------------------------------------------------
// Per-ray state
// ---------------------------------------------------------------------------------------------
template <typename T> struct RayCtx {
    T org[3], dir[3], tmin, tmax;
    T inv_dir[3];
    T aux[3];          // fast: inv_org = -inv_dir*org; robust: inv_dir_pad
    uint32_t oct;      // bit i = signbit(dir[i])
};

// reference bvh.h:161-165
template <typename T, bool kRobust, int kDim = 3> BVH_HD void ray_prologue(RayCtx<T>& r) {
    using R = Real<T>;
    r.oct = 0;
    for (int i = 0; i < kDim; ++i) {
        // ray.h:29-34: get_inv_dir<SafeInverse = !IsRobust>
        r.inv_dir[i] = kRobust ? R::div((T)1, r.dir[i]) : safe_inverse(r.dir[i]);
        if (kRobust) r.aux[i] = add_ulp_magnitude(r.inv_dir[i], 2);           // ray.h:46-48
        else         r.aux[i] = R::mul(R::neg(r.inv_dir[i]), r.org[i]);       // bvh.h:163
        r.oct |= (R::sign(r.dir[i]) ? 1u : 0u) << i;                          // ray.h:36-43
    }
}

// Accumulation step of make_intersection_result (node.h:105-117): t0 = robust_max(tn, t0),
// t1 = robust_min(tf, t1), i.e. `tn > t0 ? tn : t0` — the accumulator comes back when tn is a NaN.
// On the device this is one FMNMX: fmaxf/fminf also return the non-NaN operand, the accumulator
// itself is never a NaN (rays whose tmin/tmax is a NaN are retired as misses before traversal, which
// is what the reference's comparisons do with them), and the only other difference — which zero comes
// back when the operands are +0 and -0 — cannot change `t0 <= t1` or `t0L > t0R`, the only uses.
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ float acc_max(float tn, float t0) { return fmaxf(tn, t0); }
__device__ __forceinline__ float acc_min(float tf, float t1) { return fminf(tf, t1); }
__device__ __forceinline__ double acc_max(double tn, double t0) { return fmax(tn, t0); }
__device__ __forceinline__ double acc_min(double tf, double t1) { return fmin(tf, t1); }
#else
template <typename T> inline T acc_max(T tn, T t0) { return robust_max(tn, t0); }
template <typename T> inline T acc_min(T tf, T t1) { return robust_min(tf, t1); }
#endif

// A ray with a NaN interval can never report a hit in the reference (every comparison against
// tmin/tmax fails: node.h:110-115, tri.h:69); callers retire it as a miss without traversing.
template <typename T> BVH_HD bool ray_interval_is_nan(const RayCtx<T>& r) { return r.tmin != r.tmin || r.tmax != r.tmax; }

// The slab test of node_test over the axes [kFirst, kLast) only, continuing the interval t0, t1 of the axes tested
// before them (r.tmin, r.tmax before any).  The accumulation only raises t0 and lowers t1, so an interval that is
// already empty stays empty whatever the remaining axes give: the box is missed.
template <typename T, bool kRobust, int kFirst, int kLast> BVH_HD void node_test_axes(const T* b, const RayCtx<T>& r, T& t0, T& t1) {
    using R = Real<T>;
    for (int i = kFirst; i < kLast; ++i) {
        const bool neg = (r.oct >> i) & 1u;
        const T bnear = neg ? b[2 * i + 1] : b[2 * i];       // get_min_bounds(octant), :59-61
        const T bfar  = neg ? b[2 * i] : b[2 * i + 1];       // get_max_bounds(octant), :63-65
        T tn, tf;
        if (kRobust) {
            tn = R::mul(R::sub(bnear, r.org[i]), r.inv_dir[i]);
            tf = R::mul(R::sub(bfar,  r.org[i]), r.aux[i]);
        } else {
            tn = R::fma(bnear, r.inv_dir[i], r.aux[i]);      // fast_mul_add is std::fma (utils.h:75-76)
            tf = R::fma(bfar,  r.inv_dir[i], r.aux[i]);
        }
        t0 = acc_max(tn, t0);
        t1 = acc_min(tf, t1);
    }
}

// reference node.h:68-88 + make_intersection_result (:105-117).  b = [minx,maxx,miny,maxy,minz,maxz]
// (kDim = 2: [minx,maxx,miny,maxy], the reference's Node<T, 2>)
template <typename T, bool kRobust, int kDim = 3> BVH_HD void node_test(const T* b, const RayCtx<T>& r, T& t0, T& t1) {
    t0 = r.tmin; t1 = r.tmax;
    node_test_axes<T, kRobust, 0, kDim>(b, r, t0, t1);
}

// Closest-hit bookkeeping while a ray is in flight.  `slot` is the BVH-order primitive index
// (position in prim_ids / in the permuted triangle array); the original id is looked up on demand.
template <typename T> struct HitState {
    uint32_t slot;
    T t, u, v;
};

// tri_test's default filter: every candidate hit counts.
struct AcceptAll {
    template <typename T> BVH_HD bool operator()(uint32_t, T, T, T) const { return true; }
};

// reference tri.h:55-74 with the caller's leaf convention (benchmark.cpp:281-292).  Returns true
// when the triangle was accepted as the new closest hit (and tmax was shrunk).
//   kLowestId = false: reference example semantics, `t <= tmax` so the LAST visited of equal-t hits wins
//   kLowestId = true : canonical tree-independent rule, accept iff t < best || (t == best && id < best id)
//                      with ids being ORIGINAL primitive ids (prim_ids[slot]); a miss has id UINT_MAX
// accept(slot, t, u, v) is the caller's filter (DeviceView::trace_triangles): called for a triangle that passes the test,
// the interval and the tie rule, before anything is updated; false drops the hit.
template <typename T, typename Accept = AcceptAll>
BVH_HD bool tri_test(const DevTri<T>& tri, uint32_t slot, const uint32_t* __restrict__ prim_ids,
                     bool kLowestId, RayCtx<T>& r, HitState<T>& hit, Accept&& accept = {}) {
    using R = Real<T>;
    const T tolerance = R::neg(R::eps());
    T c[3] = { R::sub(tri.p0[0], r.org[0]), R::sub(tri.p0[1], r.org[1]), R::sub(tri.p0[2], r.org[2]) };
    T rr[3];
    cross3(r.dir, c, rr);
    const T inv_det = R::div((T)1, dot3(tri.n, r.dir));
    const T u = R::mul(dot3(rr, tri.e2), inv_det);
    const T v = R::mul(dot3(rr, tri.e1), inv_det);
    const T w = R::sub(R::sub((T)1, u), v);
    if (u >= tolerance && v >= tolerance && w >= tolerance) {
        const T t = R::mul(dot3(tri.n, c), inv_det);
        if (t >= r.tmin && t <= r.tmax) {
            if (kLowestId) {
                if (!(t < hit.t) && hit.slot != kInvalidId) {     // exact tie with the current best
                    if (!(prim_ids[slot] < prim_ids[hit.slot])) return false;
                }
            }
            if (!accept(slot, t, u, v)) return false;
            r.tmax = t;
            hit.slot = slot; hit.t = t; hit.u = u; hit.v = v;
            return true;
        }
    }
    return false;
}

} // namespace bvhb200
