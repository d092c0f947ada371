// include/bvh/v2/b200_surface.h — the reference library's C++ API surface on top of the CUDA engine.
//
// The reference is header-only C++20 templates (reference src/bvh/v2/*.h).  Its users write
//     bvh::v2::DefaultBuilder<Node>::build(thread_pool, bboxes, centers, config)   (default_builder.h:33-62)
//     bvh.intersect<IsAnyHit, IsRobust>(ray, bvh.get_root().index, stack, leaf_fn)  (bvh.h:159-182)
// against the POD-ish types Vec / BBox / Ray / Node / Index / Tri / PrecomputedTri / SmallStack.  This
// header re-declares that surface (same namespace, names, members and semantics; everything written from
// scratch) so such code compiles unchanged — the reference's own test/simple_example.cpp, serialize.cpp
// and benchmark.cpp are compiled unmodified against it by oracle/Makefile (target cxx_examples) — with
// one difference in substance: DefaultBuilder::build constructs the tree ON THE GPU through the C ABI of
// libbvh_c.so (bvh3f_build / bvh3d_build) and copies the reference-layout nodes back into Bvh<Node>.
// Per-ray Bvh::intersect keeps its template form: the leaf function is a caller-supplied host callable,
// which a device kernel cannot invoke, so it runs on the host exactly as in the reference.  Whole ray
// batches go through bvh::v2::cuda::Accel (bvhNN_build_triangles / bvhNN_intersect_rays), declared at the
// end of this file.
//
// The same-named reference headers (<bvh/v2/vec.h>, <bvh/v2/bvh.h>, ...) are thin includes of this one.
#ifndef BVH_V2_B200_SURFACE_H
#define BVH_V2_B200_SURFACE_H

#include <algorithm>
#include <array>
#include <atomic>
#include <cassert>
#include <climits>
#include <cmath>
#include <condition_variable>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <functional>
#include <istream>
#include <limits>
#include <mutex>
#include <numeric>
#include <optional>
#include <ostream>
#include <queue>
#include <span>
#include <stack>
#include <stdexcept>
#include <string>
#include <thread>
#include <tuple>
#include <type_traits>
#include <utility>
#include <vector>

#include <bvh_b200.h>
#include <bvh_b200_device.h>

#if defined(__GNUC__) || defined(__clang__)
#define BVH_ALWAYS_INLINE __attribute__((always_inline)) inline
#elif defined(_MSC_VER)
#define BVH_ALWAYS_INLINE __forceinline
#else
#define BVH_ALWAYS_INLINE inline
#endif
#define BVH_CLANG_ENABLE_FP_CONTRACT

namespace bvh::v2 {

// ------------------------------------------------------------------------------------------------
// utils (reference utils.h)
// ------------------------------------------------------------------------------------------------
template <size_t Bits> struct UnsignedInt;
template <> struct UnsignedInt<8>  { using Type = uint8_t; };
template <> struct UnsignedInt<16> { using Type = uint16_t; };
template <> struct UnsignedInt<32> { using Type = uint32_t; };
template <> struct UnsignedInt<64> { using Type = uint64_t; };
template <size_t Bits> using UnsignedIntType = typename UnsignedInt<Bits>::Type;

struct IgnoreArgs { template <typename... A> void operator()(A&&...) const {} };

template <typename U, std::enable_if_t<std::is_unsigned_v<U>, bool> = true>
constexpr U make_bitmask(size_t bits) {
    return bits >= size_t(std::numeric_limits<U>::digits) ? U(~U(0)) : U((U(1) << bits) - 1);
}

// the second argument comes back when the first is a NaN
template <typename T, std::enable_if_t<std::is_floating_point_v<T>, bool> = true>
BVH_ALWAYS_INLINE T robust_min(T a, T b) { return a < b ? a : b; }
template <typename T, std::enable_if_t<std::is_floating_point_v<T>, bool> = true>
BVH_ALWAYS_INLINE T robust_max(T a, T b) { return a > b ? a : b; }

template <typename T, std::enable_if_t<std::is_floating_point_v<T>, bool> = true>
BVH_ALWAYS_INLINE T add_ulp_magnitude(T x, unsigned ulps) {
    if (!std::isfinite(x)) return x;
    UnsignedIntType<sizeof(T) * CHAR_BIT> bits;
    std::memcpy(&bits, &x, sizeof bits);
    bits += ulps;
    std::memcpy(&x, &bits, sizeof bits);
    return x;
}

template <typename T, std::enable_if_t<std::is_floating_point_v<T>, bool> = true>
BVH_ALWAYS_INLINE T safe_inverse(T x) {
    if (std::fabs(x) <= std::numeric_limits<T>::epsilon()) return std::copysign(std::numeric_limits<T>::max(), x);
    return T(1) / x;
}

template <typename T, std::enable_if_t<std::is_floating_point_v<T>, bool> = true>
BVH_ALWAYS_INLINE T fast_mul_add(T a, T b, T c) {
#ifdef FP_FAST_FMAF
    return std::fma(a, b, c);
#else
    return a * b + c;
#endif
}

template <size_t Begin, size_t End, typename F>
BVH_ALWAYS_INLINE void static_for(F&& f) {
    if constexpr (Begin < End) { f(Begin); static_for<Begin + 1, End>(std::forward<F>(f)); }
}

template <typename U, std::enable_if_t<std::is_unsigned_v<U>, bool> = true>
constexpr U round_up_log2(U i, U p = 0) { return (U(1) << p) >= i ? p : round_up_log2(i, U(p + 1)); }

// spreads the low third of the bits of x so that two zero bits separate consecutive ones
template <typename U, std::enable_if_t<std::is_unsigned_v<U>, bool> = true>
BVH_ALWAYS_INLINE U split_bits(U x) {
    constexpr size_t width = sizeof(U) * CHAR_BIT;
    U mask = U(~U(0)) >> (width / 2);
    x &= mask;
    for (size_t n = width / 2; n > 1; n >>= 1) {
        mask = (mask | (mask << n)) & ~(mask << (n / 2));
        x = (x | (x << n)) & mask;
    }
    return x;
}
template <typename U, std::enable_if_t<std::is_unsigned_v<U>, bool> = true>
BVH_ALWAYS_INLINE U morton_encode(U x, U y, U z) { return split_bits(x) | (split_bits(y) << 1) | (split_bits(z) << 2); }

template <typename T> BVH_ALWAYS_INLINE T atomic_max(std::atomic<T>& a, const T& v) {
    T seen = a;
    while (seen < v && !a.compare_exchange_weak(seen, v)) {}
    return seen;
}

// ------------------------------------------------------------------------------------------------
// Vec (reference vec.h)
// ------------------------------------------------------------------------------------------------
template <typename T, size_t N>
struct Vec {
    T values[N];

    Vec() = default;
    template <typename... Rest>
    BVH_ALWAYS_INLINE Vec(T x, T y, Rest&&... rest) : values { x, y, static_cast<T>(std::forward<Rest>(rest))... } {}
    BVH_ALWAYS_INLINE explicit Vec(T x) { for (auto& v : values) v = x; }

    BVH_ALWAYS_INLINE T& operator[](size_t i) { return values[i]; }
    BVH_ALWAYS_INLINE T operator[](size_t i) const { return values[i]; }

    template <typename F> BVH_ALWAYS_INLINE static Vec generate(F&& f) {
        Vec v;
        static_for<0, N>([&](size_t i) { v[i] = f(i); });
        return v;
    }
    template <typename Cmp> BVH_ALWAYS_INLINE size_t get_best_axis(Cmp&& better) const {
        size_t axis = 0;
        static_for<1, N>([&](size_t i) { if (better(values[i], values[axis])) axis = i; });
        return axis;
    }
    BVH_ALWAYS_INLINE size_t get_largest_axis() const { return get_best_axis(std::greater<T>()); }
    BVH_ALWAYS_INLINE size_t get_smallest_axis() const { return get_best_axis(std::less<T>()); }
};

#define BVH_B200_VEC_OP(op)                                                                              \
    template <typename T, size_t N> BVH_ALWAYS_INLINE Vec<T, N> operator op(const Vec<T, N>& a, const Vec<T, N>& b) { \
        return Vec<T, N>::generate([&](size_t i) { return a[i] op b[i]; }); }
BVH_B200_VEC_OP(+) BVH_B200_VEC_OP(-) BVH_B200_VEC_OP(*) BVH_B200_VEC_OP(/)
#undef BVH_B200_VEC_OP
template <typename T, size_t N> BVH_ALWAYS_INLINE Vec<T, N> operator-(const Vec<T, N>& a) { return Vec<T, N>::generate([&](size_t i) { return -a[i]; }); }
template <typename T, size_t N> BVH_ALWAYS_INLINE Vec<T, N> operator*(const Vec<T, N>& a, T s) { return Vec<T, N>::generate([&](size_t i) { return a[i] * s; }); }
template <typename T, size_t N> BVH_ALWAYS_INLINE Vec<T, N> operator*(T s, const Vec<T, N>& a) { return a * s; }
template <typename T, size_t N> BVH_ALWAYS_INLINE Vec<T, N> operator/(T s, const Vec<T, N>& a) { return Vec<T, N>::generate([&](size_t i) { return s / a[i]; }); }
template <typename T, size_t N> BVH_ALWAYS_INLINE Vec<T, N> robust_min(const Vec<T, N>& a, const Vec<T, N>& b) { return Vec<T, N>::generate([&](size_t i) { return robust_min(a[i], b[i]); }); }
template <typename T, size_t N> BVH_ALWAYS_INLINE Vec<T, N> robust_max(const Vec<T, N>& a, const Vec<T, N>& b) { return Vec<T, N>::generate([&](size_t i) { return robust_max(a[i], b[i]); }); }
template <typename T, size_t N> BVH_ALWAYS_INLINE Vec<T, N> fast_mul_add(const Vec<T, N>& a, const Vec<T, N>& b, const Vec<T, N>& c) { return Vec<T, N>::generate([&](size_t i) { return fast_mul_add(a[i], b[i], c[i]); }); }
template <typename T, size_t N> BVH_ALWAYS_INLINE Vec<T, N> safe_inverse(const Vec<T, N>& a) { return Vec<T, N>::generate([&](size_t i) { return safe_inverse(a[i]); }); }
// left fold starting from T(0), like std::transform_reduce on N elements
template <typename T, size_t N> BVH_ALWAYS_INLINE T dot(const Vec<T, N>& a, const Vec<T, N>& b) {
    T acc = T(0);
    static_for<0, N>([&](size_t i) { acc = acc + a[i] * b[i]; });
    return acc;
}
template <typename T> BVH_ALWAYS_INLINE Vec<T, 3> cross(const Vec<T, 3>& a, const Vec<T, 3>& b) {
    return Vec<T, 3>(a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]);
}
template <typename T, size_t N> BVH_ALWAYS_INLINE T length(const Vec<T, N>& v) { return std::sqrt(dot(v, v)); }
template <typename T, size_t N> [[nodiscard]] BVH_ALWAYS_INLINE Vec<T, N> normalize(const Vec<T, N>& v) { return v * (T(1) / length(v)); }

// ------------------------------------------------------------------------------------------------
// BBox (reference bbox.h)
// ------------------------------------------------------------------------------------------------
template <typename T, size_t N>
struct BBox {
    Vec<T, N> min, max;

    BBox() = default;
    BVH_ALWAYS_INLINE BBox(const Vec<T, N>& lo, const Vec<T, N>& hi) : min(lo), max(hi) {}
    BVH_ALWAYS_INLINE explicit BBox(const Vec<T, N>& p) : min(p), max(p) {}

    BVH_ALWAYS_INLINE BBox& extend(const BBox& o) { min = robust_min(min, o.min); max = robust_max(max, o.max); return *this; }
    BVH_ALWAYS_INLINE BBox& extend(const Vec<T, N>& p) { return extend(BBox(p)); }
    BVH_ALWAYS_INLINE Vec<T, N> get_diagonal() const { return max - min; }
    BVH_ALWAYS_INLINE Vec<T, N> get_center() const { return (max + min) * T(0.5); }
    BVH_ALWAYS_INLINE T get_half_area() const {
        static_assert(N == 2 || N == 3);
        const auto d = get_diagonal();
        if constexpr (N == 3) return (d[0] + d[1]) * d[2] + d[0] * d[1];
        else return d[0] + d[1];
    }
    BVH_ALWAYS_INLINE static constexpr BBox make_empty() {
        return BBox(Vec<T, N>(+std::numeric_limits<T>::max()), Vec<T, N>(-std::numeric_limits<T>::max()));
    }
};

// ------------------------------------------------------------------------------------------------
// Ray (reference ray.h)
// ------------------------------------------------------------------------------------------------
struct Octant {
    uint32_t value = 0;
    static constexpr size_t max_dim = sizeof(uint32_t) * CHAR_BIT;
    uint32_t operator[](size_t i) const { return (value >> i) & 1u; }
};

template <typename T, size_t N>
struct Ray {
    Vec<T, N> org, dir;
    T tmin, tmax;

    Ray() = default;
    BVH_ALWAYS_INLINE Ray(const Vec<T, N>& o, const Vec<T, N>& d, T t0 = 0, T t1 = std::numeric_limits<T>::max())
        : org(o), dir(d), tmin(t0), tmax(t1) {}

    template <bool SafeInverse = false> BVH_ALWAYS_INLINE Vec<T, N> get_inv_dir() const {
        return Vec<T, N>::generate([&](size_t i) { return SafeInverse ? safe_inverse(dir[i]) : T(1) / dir[i]; });
    }
    BVH_ALWAYS_INLINE Octant get_octant() const {
        static_assert(N <= Octant::max_dim);
        Octant o;
        static_for<0, N>([&](size_t i) { o.value |= uint32_t(std::signbit(dir[i])) << i; });
        return o;
    }
    BVH_ALWAYS_INLINE static Vec<T, N> pad_inv_dir(const Vec<T, N>& inv) {
        return Vec<T, N>::generate([&](size_t i) { return add_ulp_magnitude(inv[i], 2); });
    }
};

// ------------------------------------------------------------------------------------------------
// streams (reference stream.h)
// ------------------------------------------------------------------------------------------------
class InputStream {
public:
    template <typename X> X read(X&& fallback = {}) {
        X x;
        if (read_raw(&x, sizeof(X)) != sizeof(X)) x = std::move(fallback);
        return x;
    }
protected:
    virtual size_t read_raw(void*, size_t) = 0;
};
class OutputStream {
public:
    template <typename X> bool write(const X& x) { return write_raw(&x, sizeof(X)); }
protected:
    virtual bool write_raw(const void*, size_t) = 0;
};
class StdInputStream : public InputStream {
public:
    StdInputStream(std::istream& s) : stream_(s) {}
    using InputStream::read;
protected:
    std::istream& stream_;
    size_t read_raw(void* p, size_t n) override { stream_.read(static_cast<char*>(p), std::streamsize(n)); return size_t(stream_.gcount()); }
};
class StdOutputStream : public OutputStream {
public:
    StdOutputStream(std::ostream& s) : stream_(s) {}
    using OutputStream::write;
protected:
    std::ostream& stream_;
    bool write_raw(const void* p, size_t n) override { stream_.write(static_cast<const char*>(p), std::streamsize(n)); return stream_.good(); }
};

// ------------------------------------------------------------------------------------------------
// Index, Node (reference index.h, node.h)
// ------------------------------------------------------------------------------------------------
template <size_t Bits, size_t PrimCountBits>
struct Index {
    using Type = UnsignedIntType<Bits>;
    static constexpr size_t bits = Bits;
    static constexpr size_t prim_count_bits = PrimCountBits;
    static constexpr Type max_prim_count = make_bitmask<Type>(PrimCountBits);
    static constexpr Type max_first_id = make_bitmask<Type>(Bits - PrimCountBits);
    static_assert(PrimCountBits < Bits);

    Type value;

    Index() = default;
    explicit Index(Type v) : value(v) {}
    bool operator==(const Index&) const = default;
    bool operator!=(const Index&) const = default;

    BVH_ALWAYS_INLINE Type first_id() const { return value >> PrimCountBits; }
    BVH_ALWAYS_INLINE Type prim_count() const { return value & max_prim_count; }
    BVH_ALWAYS_INLINE bool is_leaf() const { return prim_count() != 0; }
    BVH_ALWAYS_INLINE bool is_inner() const { return prim_count() == 0; }
    BVH_ALWAYS_INLINE void set_first_id(size_t id) { *this = pack(id, size_t(prim_count())); }
    BVH_ALWAYS_INLINE void set_prim_count(size_t n) { *this = pack(size_t(first_id()), n); }
    static BVH_ALWAYS_INLINE Index make_leaf(size_t first_prim, size_t count) { assert(count != 0); return pack(first_prim, count); }
    static BVH_ALWAYS_INLINE Index make_inner(size_t first_child) { return pack(first_child, 0); }

private:
    static BVH_ALWAYS_INLINE Index pack(size_t first, size_t count) {
        assert(first <= size_t(max_first_id) && count <= size_t(max_prim_count));
        return Index(Type((Type(first) << PrimCountBits) | (Type(count) & max_prim_count)));
    }
};

template <typename T, size_t Dim, size_t IndexBits = sizeof(T) * CHAR_BIT, size_t PrimCountBits = 4>
struct Node {
    using Scalar = T;
    using Index = bvh::v2::Index<IndexBits, PrimCountBits>;
    static constexpr size_t dimension = Dim;
    static constexpr size_t prim_count_bits = PrimCountBits;
    static constexpr size_t index_bits = IndexBits;

    std::array<T, Dim * 2> bounds;      // [min_x, max_x, min_y, max_y, ...]
    Index index;

    Node() = default;
    bool operator==(const Node&) const = default;
    bool operator!=(const Node&) const = default;

    BVH_ALWAYS_INLINE bool is_leaf() const { return index.is_leaf(); }
    BVH_ALWAYS_INLINE BBox<T, Dim> get_bbox() const {
        return BBox<T, Dim>(Vec<T, Dim>::generate([&](size_t i) { return bounds[2 * i]; }),
                            Vec<T, Dim>::generate([&](size_t i) { return bounds[2 * i + 1]; }));
    }
    BVH_ALWAYS_INLINE void set_bbox(const BBox<T, Dim>& b) {
        static_for<0, Dim>([&](size_t i) { bounds[2 * i] = b.min[i]; bounds[2 * i + 1] = b.max[i]; });
    }
    BVH_ALWAYS_INLINE Vec<T, Dim> get_min_bounds(const Octant& o) const {
        return Vec<T, Dim>::generate([&](size_t i) { return bounds[2 * uint32_t(i) + o[i]]; });
    }
    BVH_ALWAYS_INLINE Vec<T, Dim> get_max_bounds(const Octant& o) const {
        return Vec<T, Dim>::generate([&](size_t i) { return bounds[2 * uint32_t(i) + 1 - o[i]]; });
    }
    [[nodiscard]] BVH_ALWAYS_INLINE std::pair<T, T> intersect_robust(const Ray<T, Dim>& ray, const Vec<T, Dim>& inv_dir,
                                                                    const Vec<T, Dim>& inv_dir_pad, const Octant& o) const {
        return clip(ray, (get_min_bounds(o) - ray.org) * inv_dir, (get_max_bounds(o) - ray.org) * inv_dir_pad);
    }
    [[nodiscard]] BVH_ALWAYS_INLINE std::pair<T, T> intersect_fast(const Ray<T, Dim>& ray, const Vec<T, Dim>& inv_dir,
                                                                  const Vec<T, Dim>& inv_org, const Octant& o) const {
        return clip(ray, fast_mul_add(get_min_bounds(o), inv_dir, inv_org), fast_mul_add(get_max_bounds(o), inv_dir, inv_org));
    }
    BVH_ALWAYS_INLINE void serialize(OutputStream& s) const { for (const T& b : bounds) s.write(b); s.write(index.value); }
    [[nodiscard]] static BVH_ALWAYS_INLINE Node deserialize(InputStream& s) {
        Node n;
        for (T& b : n.bounds) b = s.read<T>();
        n.index = Index(s.read<typename Index::Type>());
        return n;
    }

private:
    static BVH_ALWAYS_INLINE std::pair<T, T> clip(const Ray<T, Dim>& ray, const Vec<T, Dim>& tn, const Vec<T, Dim>& tf) {
        T t0 = ray.tmin, t1 = ray.tmax;
        static_for<0, Dim>([&](size_t i) { t0 = robust_max(tn[i], t0); t1 = robust_min(tf[i], t1); });
        return { t0, t1 };
    }
};

// ------------------------------------------------------------------------------------------------
// stacks (reference stack.h)
// ------------------------------------------------------------------------------------------------
template <typename T, unsigned Capacity>
struct SmallStack {
    static constexpr unsigned capacity = Capacity;
    T elems[Capacity];
    unsigned size = 0;
    bool is_empty() const { return size == 0; }
    bool is_full() const { return size >= Capacity; }
    void push(const T& t) { assert(!is_full()); elems[size++] = t; }
    T pop() { assert(!is_empty()); return elems[--size]; }
};
template <typename T>
struct GrowingStack {
    std::vector<T> elems;
    bool is_empty() const { return elems.empty(); }
    void push(const T& t) { elems.push_back(t); }
    T pop() { assert(!is_empty()); T t = std::move(elems.back()); elems.pop_back(); return t; }
};

// ------------------------------------------------------------------------------------------------
// primitives (reference tri.h, sphere.h)
// ------------------------------------------------------------------------------------------------
template <typename T, size_t N>
struct Tri {
    Vec<T, N> p0, p1, p2;
    Tri() = default;
    BVH_ALWAYS_INLINE Tri(const Vec<T, N>& a, const Vec<T, N>& b, const Vec<T, N>& c) : p0(a), p1(b), p2(c) {}
    BVH_ALWAYS_INLINE BBox<T, N> get_bbox() const { return BBox<T, N>(p0).extend(p1).extend(p2); }
    BVH_ALWAYS_INLINE Vec<T, N> get_center() const { return (p0 + p1 + p2) * static_cast<T>(1. / 3.); }
};

template <typename T>
struct PrecomputedTri {
    Vec<T, 3> p0, e1, e2, n;
    PrecomputedTri() = default;
    BVH_ALWAYS_INLINE PrecomputedTri(const Vec<T, 3>& a, const Vec<T, 3>& b, const Vec<T, 3>& c)
        : p0(a), e1(a - b), e2(c - a), n(cross(e1, e2)) {}
    BVH_ALWAYS_INLINE PrecomputedTri(const Tri<T, 3>& t) : PrecomputedTri(t.p0, t.p1, t.p2) {}
    BVH_ALWAYS_INLINE Tri<T, 3> convert_to_tri() const { return Tri<T, 3>(p0, p0 - e1, e2 + p0); }
    BVH_ALWAYS_INLINE BBox<T, 3> get_bbox() const { return convert_to_tri().get_bbox(); }
    BVH_ALWAYS_INLINE Vec<T, 3> get_center() const { return convert_to_tri().get_center(); }

    // Moeller-Trumbore on the precomputed edges; (t, u, v) on a hit inside [tmin, tmax]
    [[nodiscard]] BVH_ALWAYS_INLINE std::optional<std::tuple<T, T, T>> intersect(
        const Ray<T, 3>& ray, T tolerance = -std::numeric_limits<T>::epsilon()) const {
        const auto c = p0 - ray.org;
        const auto r = cross(ray.dir, c);
        const T inv_det = T(1) / dot(n, ray.dir);
        const T u = dot(r, e2) * inv_det, v = dot(r, e1) * inv_det, w = T(1) - u - v;
        if (u >= tolerance && v >= tolerance && w >= tolerance) {      // false when anything is a NaN
            const T t = dot(n, c) * inv_det;
            if (t >= ray.tmin && t <= ray.tmax) return std::make_optional(std::make_tuple(t, u, v));
        }
        return std::nullopt;
    }
};

template <typename T, size_t N>
struct Sphere {
    Vec<T, N> center;
    T radius;
    Sphere() = default;
    BVH_ALWAYS_INLINE Sphere(const Vec<T, N>& c, T r) : center(c), radius(r) {}
    BVH_ALWAYS_INLINE Vec<T, N> get_center() const { return center; }
    BVH_ALWAYS_INLINE BBox<T, N> get_bbox() const { return BBox<T, N>(center - Vec<T, N>(radius), center + Vec<T, N>(radius)); }
    template <bool AssumeNormalized = false>
    [[nodiscard]] BVH_ALWAYS_INLINE std::optional<std::pair<T, T>> intersect(const Ray<T, N>& ray) const {
        const auto oc = ray.org - center;
        const T a = AssumeNormalized ? T(1) : dot(ray.dir, ray.dir);
        const T b = T(2) * dot(ray.dir, oc);
        const T c = dot(oc, oc) - radius * radius;
        const T delta = b * b - T(4) * a * c;
        if (delta >= 0) {
            const T inv = -T(0.5) / a, root = std::sqrt(delta);
            const T t0 = robust_max((b + root) * inv, ray.tmin), t1 = robust_min((b - root) * inv, ray.tmax);
            if (t0 <= t1) return std::make_optional(std::make_pair(t0, t1));
        }
        return std::nullopt;
    }
};

// ------------------------------------------------------------------------------------------------
// ThreadPool, executors (reference thread_pool.h, executor.h).  Kept for callers' own data preparation;
// the GPU builder itself does not use host threads.
// ------------------------------------------------------------------------------------------------
class ThreadPool {
public:
    using Task = std::function<void(size_t)>;
    ThreadPool(size_t thread_count = 0) {
        if (thread_count == 0) thread_count = std::max(1u, std::thread::hardware_concurrency());
        for (size_t id = 0; id < thread_count; ++id) workers_.emplace_back([this, id] { loop(id); });
    }
    ~ThreadPool() {
        wait();
        { std::lock_guard<std::mutex> lock(mutex_); quit_ = true; }
        wake_.notify_all();
        for (auto& w : workers_) w.join();
    }
    void push(Task&& task) {
        { std::lock_guard<std::mutex> lock(mutex_); queue_.push(std::move(task)); }
        wake_.notify_one();
    }
    void wait() {
        std::unique_lock<std::mutex> lock(mutex_);
        idle_.wait(lock, [this] { return running_ == 0 && queue_.empty(); });
    }
    size_t get_thread_count() const { return workers_.size(); }

private:
    void loop(size_t id) {
        for (;;) {
            Task task;
            {
                std::unique_lock<std::mutex> lock(mutex_);
                wake_.wait(lock, [this] { return quit_ || !queue_.empty(); });
                if (queue_.empty()) return;          // quit requested and nothing left
                task = std::move(queue_.front());
                queue_.pop();
                ++running_;
            }
            task(id);
            { std::lock_guard<std::mutex> lock(mutex_); --running_; }
            idle_.notify_one();
        }
    }
    std::mutex mutex_;
    std::condition_variable wake_, idle_;
    std::queue<Task> queue_;
    std::vector<std::thread> workers_;
    int running_ = 0;
    bool quit_ = false;
};

template <typename Derived>
struct Executor {
    template <typename Loop> BVH_ALWAYS_INLINE void for_each(size_t b, size_t e, const Loop& loop) { static_cast<Derived*>(this)->for_each(b, e, loop); }
    template <typename X, typename Reduce, typename Join>
    BVH_ALWAYS_INLINE X reduce(size_t b, size_t e, const X& init, const Reduce& r, const Join& j) { return static_cast<Derived*>(this)->reduce(b, e, init, r, j); }
};
struct SequentialExecutor : Executor<SequentialExecutor> {
    template <typename Loop> BVH_ALWAYS_INLINE void for_each(size_t b, size_t e, const Loop& loop) { loop(b, e); }
    template <typename X, typename Reduce, typename Join>
    BVH_ALWAYS_INLINE X reduce(size_t b, size_t e, const X& init, const Reduce& r, const Join&) { X x(init); r(x, b, e); return x; }
};
struct ParallelExecutor : Executor<ParallelExecutor> {
    ThreadPool& thread_pool;
    size_t parallel_threshold;
    ParallelExecutor(ThreadPool& pool, size_t threshold = 1024) : thread_pool(pool), parallel_threshold(threshold) {}

    template <typename Loop> BVH_ALWAYS_INLINE void for_each(size_t b, size_t e, const Loop& loop) {
        if (e - b < parallel_threshold) return loop(b, e);
        const size_t chunk = std::max(size_t(1), (e - b) / thread_pool.get_thread_count());
        for (size_t i = b; i < e; i += chunk) {
            const size_t j = std::min(e, i + chunk);
            thread_pool.push([=](size_t) { loop(i, j); });
        }
        thread_pool.wait();
    }
    template <typename X, typename Reduce, typename Join>
    BVH_ALWAYS_INLINE X reduce(size_t b, size_t e, const X& init, const Reduce& r, const Join& join) {
        if (e - b < parallel_threshold) { X x(init); r(x, b, e); return x; }
        const size_t threads = thread_pool.get_thread_count();
        const size_t chunk = std::max(size_t(1), (e - b) / threads);
        std::vector<X> partial(threads, init);
        for (size_t i = b; i < e; i += chunk) {
            const size_t j = std::min(e, i + chunk);
            thread_pool.push([&, i, j](size_t id) { r(partial[id], i, j); });
        }
        thread_pool.wait();
        for (size_t k = 1; k < threads; ++k) join(partial[0], std::move(partial[k]));
        return partial[0];
    }
};

// ------------------------------------------------------------------------------------------------
// Bvh (reference bvh.h)
// ------------------------------------------------------------------------------------------------
template <typename Node>
struct Bvh {
    using Index = typename Node::Index;
    using Scalar = typename Node::Scalar;
    using Ray = bvh::v2::Ray<Scalar, Node::dimension>;

    std::vector<Node> nodes;
    std::vector<size_t> prim_ids;

    Bvh() = default;
    Bvh(Bvh&&) = default;
    Bvh& operator=(Bvh&&) = default;
    bool operator==(const Bvh&) const = default;
    bool operator!=(const Bvh&) const = default;

    // siblings are adjacent and the left one sits at an odd index (the root is alone at 0)
    static BVH_ALWAYS_INLINE bool is_left_sibling(size_t id) { return (id & 1) == 1; }
    static BVH_ALWAYS_INLINE size_t get_sibling_id(size_t id) { return is_left_sibling(id) ? id + 1 : id - 1; }
    static BVH_ALWAYS_INLINE size_t get_left_sibling_id(size_t id) { return is_left_sibling(id) ? id : id - 1; }
    static BVH_ALWAYS_INLINE size_t get_right_sibling_id(size_t id) { return is_left_sibling(id) ? id + 1 : id; }
    BVH_ALWAYS_INLINE const Node& get_root() const { return nodes[0]; }

    [[nodiscard]] inline Bvh extract_bvh(size_t root_id) const {
        assert(root_id != 0);
        Bvh out;
        out.nodes.emplace_back();
        std::stack<std::pair<size_t, size_t>> todo;        // (index here, index in `out`)
        todo.emplace(root_id, 0);
        while (!todo.empty()) {
            const auto [src, dst] = todo.top();
            todo.pop();
            Node copy = nodes[src];
            if (copy.is_leaf()) {
                const size_t first = copy.index.first_id(), count = copy.index.prim_count();
                copy.index.set_first_id(out.prim_ids.size());
                out.prim_ids.insert(out.prim_ids.end(), prim_ids.begin() + first, prim_ids.begin() + first + count);
            } else {
                const size_t first = copy.index.first_id(), base = out.nodes.size();
                copy.index.set_first_id(base);
                todo.emplace(first, base);
                todo.emplace(first + 1, base + 1);
                out.nodes.resize(base + 2);
            }
            out.nodes[dst] = copy;
        }
        return out;
    }

    template <bool IsAnyHit, typename Stack, typename LeafFn, typename InnerFn>
    inline void traverse_top_down(Index start, Stack& stack, LeafFn&& leaf_fn, InnerFn&& inner_fn) const {
        Index top = start;
        for (;;) {
            bool alive = true;
            while (top.prim_count() == 0) {
                const Node& left = nodes[top.first_id()];
                const Node& right = nodes[top.first_id() + 1];
                const auto [hit_left, hit_right, swap_order] = inner_fn(left, right);
                if (hit_left) {
                    Index near_index = left.index;
                    if (hit_right) {
                        Index far_index = right.index;
                        if (swap_order) std::swap(near_index, far_index);
                        stack.push(far_index);
                    }
                    top = near_index;
                } else if (hit_right) {
                    top = right.index;
                } else if (stack.is_empty()) {
                    alive = false;
                    break;
                } else {
                    top = stack.pop();
                }
            }
            if (!alive) return;
            [[maybe_unused]] const auto was_hit = leaf_fn(top.first_id(), top.first_id() + top.prim_count());
            if constexpr (IsAnyHit) { if (was_hit) return; }
            if (stack.is_empty()) return;
            top = stack.pop();
        }
    }

    template <bool IsAnyHit, bool IsRobust, typename Stack, typename LeafFn, typename InnerFn = IgnoreArgs>
    inline void intersect(const Ray& ray, Index start, Stack& stack, LeafFn&& leaf_fn, InnerFn&& inner_fn = {}) const {
        const auto inv_dir = ray.template get_inv_dir<!IsRobust>();
        const auto inv_org = -inv_dir * ray.org;
        const auto inv_dir_pad = Ray::pad_inv_dir(inv_dir);
        const auto octant = ray.get_octant();
        traverse_top_down<IsAnyHit>(start, stack, leaf_fn, [&](const Node& left, const Node& right) {
            inner_fn(left, right);
            std::pair<Scalar, Scalar> l, r;
            if constexpr (IsRobust) {
                l = left.intersect_robust(ray, inv_dir, inv_dir_pad, octant);
                r = right.intersect_robust(ray, inv_dir, inv_dir_pad, octant);
            } else {
                l = left.intersect_fast(ray, inv_dir, inv_org, octant);
                r = right.intersect_fast(ray, inv_dir, inv_org, octant);
            }
            return std::make_tuple(l.first <= l.second, r.first <= r.second, !IsAnyHit && l.first > r.first);
        });
    }

    template <typename LeafFn = IgnoreArgs, typename InnerFn = IgnoreArgs>
    inline void traverse_bottom_up(LeafFn&& leaf_fn = {}, InnerFn&& inner_fn = {}) {
        const size_t n = nodes.size();
        std::vector<size_t> parent(n, 0);
        for (size_t i = 0; i < n; ++i) {
            if (nodes[i].is_leaf()) continue;
            parent[nodes[i].index.first_id()] = parent[nodes[i].index.first_id() + 1] = i;
        }
        std::vector<bool> done(n, false);
        for (size_t i = n; i-- > 0;) {
            if (!nodes[i].is_leaf()) continue;
            leaf_fn(nodes[i]);
            done[i] = true;
            for (size_t j = parent[i];; j = parent[j]) {
                const size_t first = nodes[j].index.first_id();
                if (done[j] || !done[first] || !done[first + 1]) break;
                inner_fn(nodes[j]);
                done[j] = true;
            }
        }
    }

    template <typename LeafFn = IgnoreArgs>
    inline void refit(LeafFn&& leaf_fn = {}) {
        traverse_bottom_up(leaf_fn, [&](Node& node) {
            const Node& l = nodes[node.index.first_id()];
            const Node& r = nodes[node.index.first_id() + 1];
            node.set_bbox(l.get_bbox().extend(r.get_bbox()));
        });
    }

    template <typename IndexType = typename Index::Type>
    inline void serialize(OutputStream& s) const {
        s.write(static_cast<IndexType>(nodes.size()));
        s.write(static_cast<IndexType>(prim_ids.size()));
        for (const Node& n : nodes) n.serialize(s);
        for (size_t id : prim_ids) s.write(static_cast<IndexType>(id));
    }
    template <typename IndexType = typename Index::Type>
    [[nodiscard]] static inline Bvh deserialize(InputStream& s) {
        Bvh b;
        b.nodes.resize(s.read<IndexType>());
        b.prim_ids.resize(s.read<IndexType>());
        for (Node& n : b.nodes) n = Node::deserialize(s);
        for (size_t& id : b.prim_ids) id = s.read<IndexType>();
        return b;
    }
};

// ------------------------------------------------------------------------------------------------
// builder front end (reference split_heuristic.h, top_down_sah_builder.h:27-40, default_builder.h)
// ------------------------------------------------------------------------------------------------
template <typename T>
class SplitHeuristic {
public:
    BVH_ALWAYS_INLINE SplitHeuristic(size_t log_cluster_size = 0, T cost_ratio = T(1))
        : log_cluster_size_(log_cluster_size), prim_offset_(make_bitmask<size_t>(log_cluster_size)), cost_ratio_(cost_ratio) {}
    BVH_ALWAYS_INLINE size_t get_prim_count(size_t size) const { return (size + prim_offset_) >> log_cluster_size_; }
    template <size_t N> BVH_ALWAYS_INLINE T get_leaf_cost(size_t b, size_t e, const BBox<T, N>& box) const { return box.get_half_area() * T(get_prim_count(e - b)); }
    template <size_t N> BVH_ALWAYS_INLINE T get_non_split_cost(size_t b, size_t e, const BBox<T, N>& box) const { return box.get_half_area() * (T(get_prim_count(e - b)) - cost_ratio_); }
private:
    size_t log_cluster_size_, prim_offset_;
    T cost_ratio_;
};

namespace detail {
template <typename T> struct CApi;
template <> struct CApi<float> {
    using Handle = bvh3f; using BBoxPod = bvh_bbox3f; using VecPod = bvh_vec3f; using NodePod = bvh_node3f;
    using RayPod = bvh_ray3f; using HitPod = bvh_hit3f; using ViewPod = bvh_device_view3f;
    static int device_view(Handle* h, ViewPod* v) { return bvh3f_get_device_view(h, v); }
    static Handle* build(const BBoxPod* b, const VecPod* c, size_t n, const bvh_build_config* cfg) { return bvh3f_build(nullptr, b, c, n, cfg); }
    static Handle* build_triangles(const float* v, size_t n, const bvh_build_config* cfg, unsigned fl) { return bvh3f_build_triangles(v, n, cfg, fl); }
    static void destroy(Handle* h) { bvh3f_destroy(h); }
    static size_t node_count(Handle* h) { return bvh3f_get_node_count(h); }
    static size_t prim_count(Handle* h) { return bvh3f_get_prim_count(h); }
    static const void* node0(Handle* h) { return bvh3f_get_node(h, 0); }
    static const size_t* prim_ids(Handle* h) { return bvh3f_get_prim_ids(h); }
    static int intersect(Handle* h, const RayPod* r, size_t n, HitPod* o, unsigned fl) { return bvh3f_intersect_rays(h, r, n, o, fl); }
};
template <> struct CApi<double> {
    using Handle = bvh3d; using BBoxPod = bvh_bbox3d; using VecPod = bvh_vec3d; using NodePod = bvh_node3d;
    using RayPod = bvh_ray3d; using HitPod = bvh_hit3d; using ViewPod = bvh_device_view3d;
    static int device_view(Handle* h, ViewPod* v) { return bvh3d_get_device_view(h, v); }
    static Handle* build(const BBoxPod* b, const VecPod* c, size_t n, const bvh_build_config* cfg) { return bvh3d_build(nullptr, b, c, n, cfg); }
    static Handle* build_triangles(const double* v, size_t n, const bvh_build_config* cfg, unsigned fl) { return bvh3d_build_triangles(v, n, cfg, fl); }
    static void destroy(Handle* h) { bvh3d_destroy(h); }
    static size_t node_count(Handle* h) { return bvh3d_get_node_count(h); }
    static size_t prim_count(Handle* h) { return bvh3d_get_prim_count(h); }
    static const void* node0(Handle* h) { return bvh3d_get_node(h, 0); }
    static const size_t* prim_ids(Handle* h) { return bvh3d_get_prim_ids(h); }
    static int intersect(Handle* h, const RayPod* r, size_t n, HitPod* o, unsigned fl) { return bvh3d_intersect_rays(h, r, n, o, fl); }
};
} // namespace detail

template <typename Node>
class DefaultBuilder {
    using Scalar = typename Node::Scalar;
    using Vec = bvh::v2::Vec<Scalar, Node::dimension>;
    using BBox = bvh::v2::BBox<Scalar, Node::dimension>;

public:
    enum class Quality { Low, Medium, High };

    struct Config {
        SplitHeuristic<Scalar> sah;
        size_t min_leaf_size = 1;
        size_t max_leaf_size = 8;
        Quality quality = Quality::High;
        size_t parallel_threshold = 1024;
    };

    /// The thread pool is accepted for source compatibility; the build runs on the GPU.
    [[nodiscard]] BVH_ALWAYS_INLINE static Bvh<Node> build(ThreadPool&, std::span<const BBox> bboxes, std::span<const Vec> centers,
                                                           const Config& config = {}) { return build(bboxes, centers, config); }

    [[nodiscard]] static Bvh<Node> build(std::span<const BBox> bboxes, std::span<const Vec> centers, const Config& config = {}) {
        static_assert(Node::dimension == 3 && Node::index_bits == sizeof(Scalar) * CHAR_BIT && Node::prim_count_bits == 4,
                      "the GPU builder supports Node<float,3> and Node<double,3> with the default index layout");
        using Api = detail::CApi<Scalar>;
        static_assert(sizeof(BBox) == sizeof(typename Api::BBoxPod) && sizeof(Vec) == sizeof(typename Api::VecPod));
        assert(bboxes.size() == centers.size());
        bvh_build_config cfg { static_cast<bvh_build_quality>(config.quality), config.min_leaf_size, config.max_leaf_size, config.parallel_threshold };
        auto* handle = Api::build(reinterpret_cast<const typename Api::BBoxPod*>(bboxes.data()),
                                  reinterpret_cast<const typename Api::VecPod*>(centers.data()), bboxes.size(), &cfg);
        if (!handle) throw std::runtime_error(std::string("bvh::v2::DefaultBuilder: ") + bvh_last_error());
        Bvh<Node> bvh;
        static_assert(std::is_trivially_copyable_v<Node>);
        bvh.nodes.resize(Api::node_count(handle));                 // the handle's mirror IS an array of Node<T,3>
        std::memcpy(bvh.nodes.data(), Api::node0(handle), bvh.nodes.size() * sizeof(Node));
        bvh.prim_ids.resize(Api::prim_count(handle));
        if (!bvh.prim_ids.empty()) std::memcpy(bvh.prim_ids.data(), Api::prim_ids(handle), bvh.prim_ids.size() * sizeof(size_t));
        Api::destroy(handle);
        return bvh;
    }
};

/// Subtree reinsertion (reference reinsertion_optimizer.h): runs in the library on the caller's node array
/// (bvh_optimize_nodes, include/bvh_b200.h) — host work, the tree is host data.
template <typename Node>
struct ReinsertionOptimizer {
    using Scalar = typename Node::Scalar;
    struct Config { Scalar batch_size_ratio = Scalar(0.05); size_t max_iter_count = 3; };
    static void optimize(ThreadPool& pool, Bvh<Node>& bvh, const Config& config = {}) { run(bvh, config, pool.get_thread_count()); }
    static void optimize(Bvh<Node>& bvh, const Config& config = {}) { run(bvh, config, 1); }
private:
    static void run(Bvh<Node>& bvh, const Config& config, size_t threads) {
        static_assert(Node::index_bits == sizeof(Scalar) * CHAR_BIT && Node::prim_count_bits == 4 && std::is_trivially_copyable_v<Node>,
                      "the library's optimizer supports the default index layout");
        if (bvh_optimize_nodes(bvh.nodes.data(), bvh.nodes.size(), int(Node::dimension), sizeof(Scalar) == 8,
                               double(config.batch_size_ratio), config.max_iter_count, threads ? threads : 1))
            throw std::runtime_error(std::string("bvh::v2::ReinsertionOptimizer: ") + bvh_last_error());
    }
};

// ------------------------------------------------------------------------------------------------
// Batched GPU path: one object owning the device BVH + BVH-order triangles
// ------------------------------------------------------------------------------------------------
namespace cuda {

template <typename T>
class Accel {
    using Api = detail::CApi<T>;
public:
    using Hit = typename Api::HitPod;
    enum Flags : unsigned { AnyHit = BVH_ANY_HIT, Robust = BVH_ROBUST, TieLastVisited = BVH_TIE_LAST_VISITED };

    Accel() = default;
    /// Builds from triangles in their original order (what callers otherwise do with
    /// Tri::get_bbox/get_center + DefaultBuilder::build + the PrecomputedTri permutation).
    explicit Accel(std::span<const Tri<T, 3>> tris, const bvh_build_config* config = nullptr) {
        static_assert(sizeof(Tri<T, 3>) == 9 * sizeof(T));
        handle_ = Api::build_triangles(reinterpret_cast<const T*>(tris.data()), tris.size(), config, 0);
        if (!handle_) throw std::runtime_error(std::string("bvh::v2::cuda::Accel: ") + bvh_last_error());
    }
    Accel(Accel&& o) noexcept : handle_(std::exchange(o.handle_, nullptr)) {}
    Accel& operator=(Accel&& o) noexcept { if (this != &o) { reset(); handle_ = std::exchange(o.handle_, nullptr); } return *this; }
    ~Accel() { reset(); }

    /// hits[i] answers rays[i]; prim_id is an original triangle index, all ones on a miss.
    void intersect(std::span<const Ray<T, 3>> rays, std::span<Hit> hits, unsigned flags = 0) const {
        static_assert(sizeof(Ray<T, 3>) == sizeof(typename Api::RayPod));
        if (hits.size() < rays.size()) throw std::invalid_argument("hits span too small");
        if (Api::intersect(handle_, reinterpret_cast<const typename Api::RayPod*>(rays.data()), rays.size(), hits.data(), flags))
            throw std::runtime_error(std::string("bvh::v2::cuda::Accel::intersect: ") + bvh_last_error());
    }
    typename Api::Handle* handle() const { return handle_; }

    using DeviceViewPod = typename Api::ViewPod;
    /// The device tree for kernels of your own (bvhNN_get_device_view; in device code wrap it with
    /// bvh::v2::cuda::DeviceView<T>::from, include/bvh/v2/cuda/intersect.cuh).
    DeviceViewPod device_view() const {
        DeviceViewPod v {};
        if (Api::device_view(handle_, &v))
            throw std::runtime_error(std::string("bvh::v2::cuda::Accel::device_view: ") + bvh_last_error());
        return v;
    }
    /// Same, for kernels whose per-thread traversal stack holds `stack_capacity` entries: throws std::length_error
    /// when the tree needs more (depth + 1).  The device never checks a stack's capacity.
    DeviceViewPod device_view(size_t stack_capacity) const {
        const DeviceViewPod v = device_view();
        if (stack_capacity < v.depth + 1)
            throw std::length_error("bvh::v2::cuda::Accel::device_view: a stack of " + std::to_string(stack_capacity) +
                                    " entries is too small for a tree of depth " + std::to_string(v.depth));
        return v;
    }

private:
    void reset() { if (handle_) Api::destroy(handle_); handle_ = nullptr; }
    typename Api::Handle* handle_ = nullptr;
};

} // namespace cuda
} // namespace bvh::v2

#endif
