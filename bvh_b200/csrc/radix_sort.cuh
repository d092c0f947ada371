// bvh_b200/csrc/radix_sort.cuh — hand-written LSD radix sort of (Morton key, primitive id) pairs.
//
// 8-bit digits, stable, three kernels per pass:
//   rs_tile_hist   per-tile digit histogram, stored digit-major  [digit][tile]
//   rs_scan_bins   one warp per digit: exclusive scan of that digit's counts over the tiles (= keys with
//                  the same digit in earlier tiles) and the digit's total
//   rs_scatter     scans the 256 digit totals (= keys with a smaller digit anywhere), re-reads the tile,
//                  ranks keys of equal digit stably (warp-level multi-split from eight ballots per key, then
//                  a per-digit prefix across the tile's warps) and scatters
// A tile is 256 threads x 8 keys = 2048 keys, warp-striped so every load instruction of a warp
// reads 32 consecutive keys (128 B / 256 B, fully coalesced).  No stage is a single serial block.
//
// Algorithmic HBM bytes per key per pass (32-bit key, 32-bit value): hist 4 + scatter read 8 +
// scatter write 8 = 20 (the first pass synthesises the identity permutation instead of reading it).
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

namespace bvhb200 {

constexpr int kRsBlock = 256;
constexpr int kRsItems = 8;
constexpr int kRsTile = kRsBlock * kRsItems;     // 2048 keys per tile
constexpr int kRsBins = 256;
constexpr int kRsWarps = kRsBlock / 32;          // 8
constexpr int kRsScanWarps = 8;                  // digits scanned per block of rs_scan_bins_kernel
static_assert(kRsBlock == kRsBins, "thread d owns digit d");

template <typename K>
__global__ void __launch_bounds__(kRsBlock)
rs_tile_hist_kernel(const K* __restrict__ keys, uint32_t n, int shift,
                    uint32_t* __restrict__ tile_hist, uint32_t num_tiles) {
    __shared__ uint32_t hist[kRsBins];
    const uint32_t tile = blockIdx.x;
    hist[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t base = tile * (uint32_t)kRsTile;
    #pragma unroll
    for (int k = 0; k < kRsItems; ++k) {
        const uint32_t idx = base + k * kRsBlock + threadIdx.x;
        if (idx < n) atomicAdd(&hist[(uint32_t)(keys[idx] >> shift) & 255u], 1u);
    }
    __syncthreads();
    tile_hist[(size_t)threadIdx.x * num_tiles + tile] = hist[threadIdx.x];
}

// One warp per digit: exclusive scan of that digit's per-tile counts (a contiguous row of the
// digit-major histogram), in place, plus the digit's total.  The 256 totals are scanned by every
// scatter block itself.
static __global__ void __launch_bounds__(kRsScanWarps * 32)
rs_scan_bins_kernel(uint32_t* __restrict__ tile_hist, uint32_t num_tiles, uint32_t* __restrict__ bin_totals) {
    const unsigned lane = threadIdx.x & 31u;
    const uint32_t bin = blockIdx.x * kRsScanWarps + (threadIdx.x >> 5);
    uint32_t* row = tile_hist + (size_t)bin * num_tiles;
    uint32_t running = 0;
    for (uint32_t base = 0; base < num_tiles; base += 32) {
        const uint32_t i = base + lane;
        const uint32_t v = i < num_tiles ? row[i] : 0u;
        uint32_t incl = v;
        #pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, incl, o);
            if (lane >= (unsigned)o) incl += x;
        }
        if (i < num_tiles) row[i] = running + incl - v;
        running += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
    if (lane == 0) bin_totals[bin] = running;
}

template <typename K, bool kIota>
__global__ void __launch_bounds__(kRsBlock)
rs_scatter_kernel(const K* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                  K* __restrict__ keys_out, uint32_t* __restrict__ vals_out, uint32_t n, int shift,
                  const uint32_t* __restrict__ tile_offsets, uint32_t num_tiles,
                  const uint32_t* __restrict__ bin_totals) {
    __shared__ uint32_t warp_hist[kRsWarps][kRsBins];     // 8 KB
    __shared__ uint32_t bin_base[kRsBins];
    __shared__ uint32_t scan_tmp[kRsWarps];
    const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned lt = (1u << lane) - 1u;
    const uint32_t tile = blockIdx.x;

    #pragma unroll
    for (int w = 0; w < kRsWarps; ++w) warp_hist[w][tid] = 0;

    // exclusive scan of the 256 digit totals (thread d owns digit d) -> start of digit d in the output
    const uint32_t total = bin_totals[tid];
    uint32_t incl = total;
    #pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= (unsigned)o) incl += x;
    }
    if (lane == 31) scan_tmp[warp] = incl;
    __syncthreads();
    uint32_t warp_prefix = 0;
    #pragma unroll
    for (int w = 0; w < kRsWarps; ++w) if (w < (int)warp) warp_prefix += scan_tmp[w];
    const uint32_t digit_start = warp_prefix + incl - total;

    const uint32_t warp_base = tile * (uint32_t)kRsTile + warp * (32u * kRsItems);
    K key[kRsItems];
    uint32_t val[kRsItems];
    uint32_t rank[kRsItems];
    #pragma unroll
    for (int j = 0; j < kRsItems; ++j) {
        const uint32_t idx = warp_base + j * 32 + lane;
        const bool valid = idx < n;
        key[j] = valid ? keys_in[idx] : (K)0;
        val[j] = kIota ? idx : (valid ? vals_in[idx] : 0u);
    }
    #pragma unroll
    for (int j = 0; j < kRsItems; ++j) {
        const uint32_t idx = warp_base + j * 32 + lane;
        const bool valid = idx < n;
        const uint32_t d = valid ? ((uint32_t)(key[j] >> shift) & 255u) : 256u;
        // lanes holding the same digit: AND of eight ballots (much cheaper than __match_any_sync, which
        // iterates over the distinct values in the warp — up to 32 of them here)
        unsigned peers = __ballot_sync(0xFFFFFFFFu, valid);
        if (!valid) peers = ~peers;
        #pragma unroll
        for (int bit = 0; bit < 8; ++bit) {
            const unsigned vote = __ballot_sync(0xFFFFFFFFu, (d >> bit) & 1u);
            peers &= ((d >> bit) & 1u) ? vote : ~vote;
        }
        const uint32_t r = __popc(peers & lt);
        uint32_t base = 0;
        if (valid) base = warp_hist[warp][d];
        __syncwarp();
        if (valid && r == 0) warp_hist[warp][d] = base + __popc(peers);
        __syncwarp();
        rank[j] = base + r;
    }
    __syncthreads();
    {
        uint32_t running = 0;
        #pragma unroll
        for (int w = 0; w < kRsWarps; ++w) {
            const uint32_t c = warp_hist[w][tid];
            warp_hist[w][tid] = running;
            running += c;
        }
        bin_base[tid] = digit_start + tile_offsets[(size_t)tid * num_tiles + tile];
    }
    __syncthreads();
    #pragma unroll
    for (int j = 0; j < kRsItems; ++j) {
        const uint32_t idx = warp_base + j * 32 + lane;
        if (idx < n) {
            const uint32_t d = (uint32_t)(key[j] >> shift) & 255u;
            const uint32_t pos = bin_base[d] + warp_hist[warp][d] + rank[j];
            keys_out[pos] = key[j];
            vals_out[pos] = val[j];
        }
    }
}

// ---- one-sweep variant --------------------------------------------------------------------------------------
// ONE kernel per pass.  The digit totals of every pass are known before the first pass (a histogram does not depend
// on the order of the keys: lbvh_build.cu's morton_kernel counts the digits of each key it produces), so a pass only
// needs, per tile and digit, the number of keys with that digit in EARLIER tiles.  Tiles are handed out in order by
// a ticket counter; a tile publishes its per-digit counts in a descriptor row (flag AGGREGATE), then looks back over
// its predecessors' rows, adding counts until it meets a row already flagged INCLUSIVE, and publishes its own
// inclusive prefixes (decoupled look-back: a tile only ever waits for tiles that started before it).  Compared with
// the three-kernel pass above this drops the histogram pass over the keys (4 bytes per key and pass) and two of
// three launches: 4 + 8 + 8 -> 8 + 8 bytes per key and pass.
// Descriptor word: bits 31..30 = 0 not ready, 1 aggregate, 2 inclusive prefix; bits 29..0 = count.
constexpr uint32_t kOsAggregate = 1u << 30, kOsInclusive = 2u << 30, kOsCountMask = (1u << 30) - 1u;
constexpr int kOsWindow = 8;                    // descriptors fetched together by a looking-back thread
constexpr uint32_t kOsMaxPolls = 1u << 24;      // look-back polls of one descriptor before a tile gives up (a hang becomes an error)

__device__ __forceinline__ uint32_t os_load(const uint32_t* p) { return *reinterpret_cast<const volatile uint32_t*>(p); }
__device__ __forceinline__ void os_store(uint32_t* p, uint32_t v) { *reinterpret_cast<volatile uint32_t*>(p) = v; }

template <typename K, bool kIota>
__global__ void __launch_bounds__(kRsBlock)
rs_onesweep_kernel(const K* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                   K* __restrict__ keys_out, uint32_t* __restrict__ vals_out, uint32_t n, int shift,
                   const uint32_t* __restrict__ digit_totals, uint32_t* __restrict__ desc, uint32_t* __restrict__ ticket,
                   uint32_t* __restrict__ status) {
    __shared__ uint32_t warp_hist[kRsWarps][kRsBins];     // 8 KB
    __shared__ uint32_t bin_base[kRsBins];
    __shared__ uint32_t scan_tmp[kRsWarps];
    __shared__ uint32_t tile_shared;
    const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned lt = (1u << lane) - 1u;
    if (tid == 0) tile_shared = atomicAdd(ticket, 1u);    // tiles in order of arrival: every predecessor is running or done
    #pragma unroll
    for (int w = 0; w < kRsWarps; ++w) warp_hist[w][tid] = 0;

    // exclusive scan of the 256 digit totals (thread d owns digit d) -> start of digit d in the output
    const uint32_t total = digit_totals[tid];
    uint32_t incl = total;
    #pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= (unsigned)o) incl += x;
    }
    if (lane == 31) scan_tmp[warp] = incl;
    __syncthreads();
    const uint32_t tile = tile_shared;
    uint32_t warp_prefix = 0;
    #pragma unroll
    for (int w = 0; w < kRsWarps; ++w) if (w < (int)warp) warp_prefix += scan_tmp[w];
    const uint32_t digit_start = warp_prefix + incl - total;

    const uint32_t warp_base = tile * (uint32_t)kRsTile + warp * (32u * kRsItems);
    K key[kRsItems];
    uint32_t val[kRsItems];
    uint32_t rank[kRsItems];
    #pragma unroll
    for (int j = 0; j < kRsItems; ++j) {
        const uint32_t idx = warp_base + j * 32 + lane;
        const bool valid = idx < n;
        key[j] = valid ? keys_in[idx] : (K)0;
        val[j] = kIota ? idx : (valid ? vals_in[idx] : 0u);
    }
    #pragma unroll
    for (int j = 0; j < kRsItems; ++j) {
        const uint32_t idx = warp_base + j * 32 + lane;
        const bool valid = idx < n;
        const uint32_t d = valid ? ((uint32_t)(key[j] >> shift) & 255u) : 256u;
        unsigned peers = __ballot_sync(0xFFFFFFFFu, valid);
        if (!valid) peers = ~peers;
        #pragma unroll
        for (int bit = 0; bit < 8; ++bit) {
            const unsigned vote = __ballot_sync(0xFFFFFFFFu, (d >> bit) & 1u);
            peers &= ((d >> bit) & 1u) ? vote : ~vote;
        }
        const uint32_t r = __popc(peers & lt);
        uint32_t base = 0;
        if (valid) base = warp_hist[warp][d];
        __syncwarp();
        if (valid && r == 0) warp_hist[warp][d] = base + __popc(peers);
        __syncwarp();
        rank[j] = base + r;
    }
    __syncthreads();
    {
        uint32_t count = 0;
        #pragma unroll
        for (int w = 0; w < kRsWarps; ++w) {
            const uint32_t c = warp_hist[w][tid];
            warp_hist[w][tid] = count;
            count += c;
        }
        // publish, look back, publish again (thread d: digit d)
        uint32_t before = 0;
        uint32_t* mine = desc + (size_t)tile * kRsBins + tid;
        if (tile == 0) {
            os_store(mine, count | kOsInclusive);
        } else {
            os_store(mine, count | kOsAggregate);
            // Look back in windows of kOsWindow descriptors: the loads of a window are independent (all in flight at
            // once), then the window is consumed nearest first.  With every tile of a pass resident at the same time
            // most predecessors still show an AGGREGATE when a tile starts to look, so the walk is long; one load per
            // step made a pass no faster than the three-kernel form.
            bool done = false;
            for (uint32_t hi = tile; hi > 0 && !done;) {                   // predecessors hi-1, hi-2, ...
                const uint32_t span = hi < (uint32_t)kOsWindow ? hi : (uint32_t)kOsWindow;
                uint32_t v[kOsWindow];
                #pragma unroll
                for (int k = 0; k < kOsWindow; ++k)
                    v[k] = (uint32_t)k < span ? os_load(desc + (size_t)(hi - 1 - k) * kRsBins + tid) : kOsInclusive;
                #pragma unroll
                for (int k = 0; k < kOsWindow; ++k) {
                    if (done || (uint32_t)k >= span) continue;
                    uint32_t polls = 0;
                    while ((v[k] >> 30) == 0u && ++polls < kOsMaxPolls) v[k] = os_load(desc + (size_t)(hi - 1 - k) * kRsBins + tid);
                    if ((v[k] >> 30) == 0u) { atomicExch(status, 1u); done = true; continue; }   // a predecessor never published: give up (the caller reports it)
                    before += v[k] & kOsCountMask;
                    if ((v[k] >> 30) == 2u) done = true;
                }
                hi -= span;
            }
            os_store(mine, ((before + count) & kOsCountMask) | kOsInclusive);
        }
        bin_base[tid] = digit_start + before;
    }
    __syncthreads();
    #pragma unroll
    for (int j = 0; j < kRsItems; ++j) {
        const uint32_t idx = warp_base + j * 32 + lane;
        if (idx < n) {
            const uint32_t d = (uint32_t)(key[j] >> shift) & 255u;
            const uint32_t pos = bin_base[d] + warp_hist[warp][d] + rank[j];
            keys_out[pos] = key[j];
            vals_out[pos] = val[j];
        }
    }
}

constexpr int kOsStatusWord = 32;               // state[32]: set to 1 when a look-back gave up
// Words of the one-sweep state for n keys and `passes` passes: [0, 64) tickets, then passes x 256 digit totals,
// then passes x tiles x 256 descriptor words.  The caller zeroes it and has the digit totals filled in (digit d of
// pass p at state[64 + 256 * p + d]) before radix_sort_onesweep runs.
inline size_t onesweep_state_words(uint32_t n, int passes) {
    const size_t tiles = (n + kRsTile - 1) / kRsTile;
    return 64 + (size_t)passes * kRsBins + (size_t)passes * tiles * kRsBins;
}
inline int radix_passes(int key_bits) { int p = (key_bits + 7) / 8; return (p & 1) ? p + 1 : p; }   // even: the result lands in buffer A

template <typename K>
inline cudaError_t radix_sort_onesweep(K* keys_a, uint32_t* vals_a, K* keys_b, uint32_t* vals_b,
                                       uint32_t* state, uint32_t n, int key_bits, cudaStream_t stream) {
    const uint32_t num_tiles = (n + kRsTile - 1) / kRsTile;
    const int passes = radix_passes(key_bits);
    uint32_t* tickets = state;
    uint32_t* totals = state + 64;
    uint32_t* desc = totals + (size_t)passes * kRsBins;
    K* kin = keys_a; K* kout = keys_b;
    uint32_t* vin = vals_a; uint32_t* vout = vals_b;
    for (int pass = 0; pass < passes; ++pass) {
        uint32_t* d = desc + (size_t)pass * num_tiles * kRsBins;
        if (pass == 0)
            rs_onesweep_kernel<K, true><<<num_tiles, kRsBlock, 0, stream>>>(kin, vin, kout, vout, n, pass * 8, totals + pass * kRsBins, d, tickets + pass, tickets + kOsStatusWord);
        else
            rs_onesweep_kernel<K, false><<<num_tiles, kRsBlock, 0, stream>>>(kin, vin, kout, vout, n, pass * 8, totals + pass * kRsBins, d, tickets + pass, tickets + kOsStatusWord);
        K* tk = kin; kin = kout; kout = tk;
        uint32_t* tv = vin; vin = vout; vout = tv;
    }
    return cudaGetLastError();
}

// Sorts n (key, value) pairs by the low `key_bits` bits of the key.  keys_a/vals_a hold the input
// (vals_a is ignored: the value of element i is i) and, because the number of passes is even for
// 30- and 63-bit keys, also the output.  tile_hist needs 256 * ceil(n / 2048) + 256 uint32.
template <typename K>
inline cudaError_t radix_sort_pairs(K* keys_a, uint32_t* vals_a, K* keys_b, uint32_t* vals_b,
                                    uint32_t* tile_hist, uint32_t n, int key_bits, cudaStream_t stream) {
    const uint32_t num_tiles = (n + kRsTile - 1) / kRsTile;
    uint32_t* bin_totals = tile_hist + (size_t)num_tiles * kRsBins;
    int passes = (key_bits + 7) / 8;
    if (passes & 1) ++passes;                              // keep the result in buffer A
    K* kin = keys_a; K* kout = keys_b;
    uint32_t* vin = vals_a; uint32_t* vout = vals_b;
    for (int pass = 0; pass < passes; ++pass) {
        const int shift = pass * 8;
        rs_tile_hist_kernel<K><<<num_tiles, kRsBlock, 0, stream>>>(kin, n, shift, tile_hist, num_tiles);
        rs_scan_bins_kernel<<<kRsBins / kRsScanWarps, kRsScanWarps * 32, 0, stream>>>(tile_hist, num_tiles, bin_totals);
        if (pass == 0)
            rs_scatter_kernel<K, true><<<num_tiles, kRsBlock, 0, stream>>>(kin, vin, kout, vout, n, shift, tile_hist, num_tiles, bin_totals);
        else
            rs_scatter_kernel<K, false><<<num_tiles, kRsBlock, 0, stream>>>(kin, vin, kout, vout, n, shift, tile_hist, num_tiles, bin_totals);
        K* tk = kin; kin = kout; kout = tk;
        uint32_t* tv = vin; vin = vout; vout = tv;
    }
    return cudaGetLastError();
}

} // namespace bvhb200
