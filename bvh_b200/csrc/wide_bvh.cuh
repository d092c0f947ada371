// bvh_b200/csrc/wide_bvh.cuh — the compressed 4-wide acceleration structure used by the fast traversal
// path (float only).
//
// Why it exists: with divergent rays the binary traversal is bound by the L1 data pipe — every lane's
// fetch of a 64-byte sibling pair costs two wavefronts (profiles/: l1tex__data_pipe_lsu_wavefronts at
// ~87 % of peak at 2.6 Grays/s).  A 4-wide node with 8-bit quantised child boxes is ALSO 64 bytes, but one
// step through it replaces about two binary steps, so a ray needs roughly half as many wavefronts.
//
// It is derived on the device from the reference-layout binary tree (which stays authoritative: host
// mirror, exact-order traversal, save/load all use the binary tree), by collapsing each node with its
// larger grandchildren.  Child boxes are stored relative to the node's own box on a power-of-two grid and
// rounded OUTWARDS, so the wide tree is conservative: every ray/triangle pair the binary traversal tests
// is also tested here, the triangle test itself (core.cuh tri_test) is the exact one, and the closest hit
// under the canonical tie-break is therefore the same hit, bit for bit.  What differs is the visit order,
// so this path is not used when the caller asks for the reference's order-dependent behaviour
// (BVH_TIE_LAST_VISITED, per-ray statistics) — those run on the binary tree.
#pragma once

#include "core.cuh"

namespace bvhb200 {

// One 4-wide node: 64 bytes, 64-byte aligned (two 256-bit loads from one line).
//   origin[3]            the node's box minimum
//   exp[3]               biased IEEE exponents: cell size on axis a = 2^(exp[a]-127); 0 means a flat axis
//   count                number of used child slots (1..4)
//   qlo[a][c], qhi[a][c] child c's box on axis a in cells from the origin (lo rounded down, hi up)
//   child[c]             reference-style packed index: low 4 bits = primitive count (leaf) or 0 (inner);
//                        leaf: high bits = first BVH-order primitive; inner: high bits = index of the
//                        child WideNode.  Unused slots have qlo = 255, qhi = 0 (never hit).
struct alignas(64) WideNode {
    float origin[3];
    uint8_t exp[3];
    uint8_t count;
    uint8_t qlo[3][4];
    uint8_t qhi[3][4];
    uint32_t child[4];
    uint32_t pad[2];
};
static_assert(sizeof(WideNode) == 64, "wide node size");

// Smallest power-of-two cell such that `extent` spans at most 255 cells; returned as a biased exponent.
BVH_HD uint8_t wide_cell_exponent(float extent) {
    if (!(extent > 0.f)) return 0;
    const float cell = extent / 255.f;
    uint32_t bits = Real<float>::bits(cell);
    uint32_t e = bits >> 23;
    if (bits & 0x7FFFFFu) e += 1;                 // round the cell size up to a power of two
    if (e == 0) e = 1;                             // denormal cell: use the smallest normal power of two
    if (e > 254) e = 254;
    return (uint8_t)e;
}
BVH_HD float wide_cell_size(uint8_t e) { return Real<float>::from_bits((uint32_t)e << 23); }

// Quantise [lo, hi] relative to origin on a grid of `cell`; outward rounding verified in position space.
BVH_HD void wide_quantize(float lo, float hi, float origin, uint8_t e, uint8_t& qlo, uint8_t& qhi) {
    if (e == 0) { qlo = 0; qhi = 0; return; }
    const float cell = wide_cell_size(e), inv = 1.f / cell;
    int a = (int)floorf((lo - origin) * inv), b = (int)ceilf((hi - origin) * inv);
    if (a < 0) a = 0;
    if (a > 255) a = 255;
    if (b < 0) b = 0;
    if (b > 255) b = 255;
    while (a > 0 && origin + (float)a * cell > lo) --a;
    while (b < 255 && origin + (float)b * cell < hi) ++b;
    qlo = (uint8_t)a; qhi = (uint8_t)b;
}


// Gathers the (up to four) binary nodes that become the children of the wide node representing the binary
// node stored at device slot `self_slot`: its two children, with the larger-area inner ones replaced by
// their own children.  Returns the number of slots used.
BVH_HD int wide_gather_children(const DevNode<float>* __restrict__ nodes, uint32_t self_slot, uint32_t slot[4]) {
    const DevNode<float>& self = nodes[self_slot];
    if (index_count(self.index) != 0) { slot[0] = self_slot; return 1; }     // the root is a leaf
    slot[0] = (uint32_t)index_first(self.index) + 1; slot[1] = slot[0] + 1;
    int used = 2;
    for (int round = 0; round < 2 && used < 4; ++round) {
        int best = -1; float best_area = -1.f;
        for (int c = 0; c < used; ++c) {
            const DevNode<float>& n = nodes[slot[c]];
            if (index_count(n.index) != 0) continue;
            const float mn[3] = { n.bounds[0], n.bounds[2], n.bounds[4] }, mx[3] = { n.bounds[1], n.bounds[3], n.bounds[5] };
            const float area = half_area(mn, mx);
            if (area > best_area) { best_area = area; best = c; }
        }
        if (best < 0) break;
        const uint32_t first = (uint32_t)index_first(nodes[slot[best]].index) + 1;
        slot[best] = first;
        slot[used++] = first + 1;
    }
    return used;
}

// Fills everything of a wide node except the references of inner children (child[c] = 0 for those; the
// caller allocates their wide indices).  is_inner[c] tells which slots are inner.
BVH_HD void wide_encode(const DevNode<float>* __restrict__ nodes, const uint32_t slot[4], int used, WideNode& w, bool is_inner[4]) {
    float lo[3] = { FLT_MAX, FLT_MAX, FLT_MAX }, hi[3] = { -FLT_MAX, -FLT_MAX, -FLT_MAX };
    for (int c = 0; c < used; ++c)
        for (int a = 0; a < 3; ++a) {
            lo[a] = robust_min(nodes[slot[c]].bounds[2 * a], lo[a]);
            hi[a] = robust_max(nodes[slot[c]].bounds[2 * a + 1], hi[a]);
        }
    for (int a = 0; a < 3; ++a) {
        w.origin[a] = lo[a];
        uint8_t e = wide_cell_exponent(hi[a] - lo[a]);
        // hi - lo and origin + 255 * cell are both rounded: make sure cell 255 really reaches the far side, so that
        // wide_quantize can always round a child's upper bound outwards (the wide tree must stay conservative)
        while (e != 0 && e < 254 && lo[a] + 255.f * wide_cell_size(e) < hi[a]) ++e;
        w.exp[a] = e;
    }
    w.count = (uint8_t)used;
    w.pad[0] = w.pad[1] = 0;
    for (int c = 0; c < 4; ++c) {
        is_inner[c] = false;
        if (c >= used) {
            for (int a = 0; a < 3; ++a) { w.qlo[a][c] = 255; w.qhi[a][c] = 0; }
            w.child[c] = 0xFFFFFFFFu;
            continue;
        }
        const DevNode<float>& n = nodes[slot[c]];
        for (int a = 0; a < 3; ++a) wide_quantize(n.bounds[2 * a], n.bounds[2 * a + 1], w.origin[a], w.exp[a], w.qlo[a][c], w.qhi[a][c]);
        if (index_count(n.index) != 0) w.child[c] = n.index;                 // leaf: first << 4 | count
        else { w.child[c] = 0; is_inner[c] = true; }
    }
}

// Per-ray constants of the wide traversal: inverse direction shrunk by 2 ulp for near planes and grown by
// 2 ulp for far planes, so that rounding in the dequantisation can only make a child box larger.
BVH_HD void wide_ray_setup(RayCtx<float>& r) {
    r.oct = 0;
    for (int k = 0; k < 3; ++k) {
        const float inv = safe_inverse(r.dir[k]);
        r.inv_dir[k] = Real<float>::from_bits(Real<float>::bits(inv) - 2u);
        r.aux[k] = add_ulp_magnitude(inv, 2);
        r.oct |= (Real<float>::sign(r.dir[k]) ? 1u : 0u) << k;
    }
}

BVH_HD float wide_fmax(float a, float b) {        // returns b when a is a NaN (a 0 * inf slab is ignored)
#if defined(__CUDA_ARCH__)
    return fmaxf(a, b);
#else
    return a > b ? a : b;
#endif
}
BVH_HD float wide_fmin(float a, float b) {
#if defined(__CUDA_ARCH__)
    return fminf(a, b);
#else
    return a < b ? a : b;
#endif
}

// Byte c of a packed word as a float: a plain int-to-float conversion (I2F, on the XU pipe, which nothing else in this
// kernel uses).  Byte permutes into the mantissa of a power of two were measured slower on an earlier GPU: they cost an
// extra issue slot per value or load the ALU pipe that also carries the kernel's min/max, compares and selects.
BVH_HD float wide_byte_to_float(uint32_t word, int c) { return (float)((word >> (8 * c)) & 0xFFu); }

// One inner step through the wide node whose 16 words are in w (layout of WideNode).  Dequantises the four
// child boxes straight into ray-parameter space, t = q * (cell * inv_dir) + (origin - org) * inv_dir,
// visits the nearest hit child next and pushes the others far-to-near (any-hit: no ordering).  Returns
// false when nothing was hit and the stack is empty.
template <bool kAny, typename Stack>
BVH_HD bool wide_step(const uint32_t (&w)[16], const RayCtx<float>& r, uint32_t& top, Stack& stack) {
    using R = Real<float>;
    float s[3], sp[3], b[3], bp[3];
    for (int k = 0; k < 3; ++k) {
        const float cell = R::from_bits(((w[3] >> (8 * k)) & 0xFFu) << 23);
        const float d = R::sub(R::from_bits(w[k]), r.org[k]);
        s[k] = R::mul(cell, r.inv_dir[k]);  b[k] = R::mul(d, r.inv_dir[k]);
        sp[k] = R::mul(cell, r.aux[k]);     bp[k] = R::mul(d, r.aux[k]);
    }
    uint32_t qn[3], qf[3];
    for (int k = 0; k < 3; ++k) {
        const bool neg = (r.oct >> k) & 1u;
        qn[k] = neg ? w[7 + k] : w[4 + k];          // words 4..6 = qlo x,y,z ; 7..9 = qhi x,y,z
        qf[k] = neg ? w[4 + k] : w[7 + k];
    }
    const float inf = R::from_bits(0x7F800000u);
    const uint32_t used = w[3] >> 24;                // child slots in use (unused ones carry an inverted box, but a ray whose
                                                     // direction has a zero component turns slab values into NaNs that are ignored)
    float t0[4]; uint32_t ref[4];
    for (int c = 0; c < 4; ++c) {
        float tn = r.tmin, tf = r.tmax;
        for (int k = 0; k < 3; ++k) {
            tn = wide_fmax(R::fma(wide_byte_to_float(qn[k], c), s[k], b[k]), tn);
            tf = wide_fmin(R::fma(wide_byte_to_float(qf[k], c), sp[k], bp[k]), tf);
        }
        ref[c] = w[10 + c];
        t0[c] = ((uint32_t)c < used && tn <= tf) ? tn : inf;             // +inf marks a miss
    }
    if (!kAny) {
        // sort the four (t0, ref) pairs by t0, nearest first (5 compare-exchanges)
#define BVH_CSWAP(i, j) { const bool sw = t0[j] < t0[i]; const float ta = sw ? t0[j] : t0[i], tb = sw ? t0[i] : t0[j]; \
                          const uint32_t ra = sw ? ref[j] : ref[i], rb = sw ? ref[i] : ref[j]; t0[i] = ta; t0[j] = tb; ref[i] = ra; ref[j] = rb; }
        BVH_CSWAP(0, 1) BVH_CSWAP(2, 3) BVH_CSWAP(0, 2) BVH_CSWAP(1, 3) BVH_CSWAP(1, 2)
#undef BVH_CSWAP
        if (t0[0] == inf) {
            if (!stack.try_pop(top)) return false;
        } else {
            if (t0[3] != inf) stack.push(ref[3]);
            if (t0[2] != inf) stack.push(ref[2]);
            if (t0[1] != inf) stack.push(ref[1]);
            top = ref[0];
        }
    } else {
        uint32_t next = 0xFFFFFFFFu;
        for (int c = 3; c >= 0; --c)
            if (t0[c] != inf) { if (next != 0xFFFFFFFFu) stack.push(next); next = ref[c]; }
        if (next == 0xFFFFFFFFu) {
            if (!stack.try_pop(top)) return false;
        } else top = next;
    }
    return true;
}

} // namespace bvhb200
