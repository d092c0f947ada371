// bvh_b200/csrc/c_api.cu — the extern "C" boundary (include/bvh/v2/c_api/bvh.h + include/bvh_b200.h).
//
// A handle (struct bvh3f / bvh3d) owns
//   * the device-resident BVH (engine.h: DeviceBvh) that the batched entry points trace against, and
//   * a lazily synchronised HOST MIRROR in the reference's exact layout — vector of Node<T,3>
//     (28 / 56 bytes: six bounds + packed index, reference node.h:31-37) plus size_t prim_ids
//     (reference bvh.h:17-23) — which is what the reference's per-node accessors, refit, save/load and
//     the per-ray callback API operate on (reference c_api/bvh_impl.h:118-250).
// A GPU build leaves the mirror empty until a legacy accessor asks for it; a mirror that may have been
// edited through bvhNN_get_node / bvhNN_load is re-uploaded before the next batched call.
#define BVH_BUILD_API
#include <bvh_b200.h>
#include <bvh_b200_device.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

#include "engine.h"
#include "reinsertion.h"

namespace bvhb200 {

// ---- errors, allocation ---------------------------------------------------------------------
static thread_local std::string g_error;
void set_error(const std::string& msg) { g_error = msg; }
const char* last_error() { return g_error.c_str(); }

Tunables& tunables() {
    static Tunables t;
    static std::once_flag once;
    std::call_once(once, [] {
        auto env = [] (const char* name, long fallback) { const char* e = getenv(name); return e ? atol(e) : fallback; };
        t.morton_bits = (int)env("BVH_B200_MORTON_BITS", 0);
        t.sah_treelets = (int)env("BVH_B200_SAH_TREELETS", -1);
        if (const char* e = getenv("BVH_B200_HIERARCHY")) {
            const std::string v = e;
            t.hierarchy = v == "global" ? 0 : v == "thread64" ? 64 : v == "thread256" ? 256 : 128;
        }
        t.e2e_chunks = (int)env("BVH_B200_E2E_CHUNKS", 0);
        t.variant = (int)env("BVH_B200_VARIANT", 0);
        t.use_wide = (int)env("BVH_B200_USE_WIDE", 0);
        { const long m = env("BVH_B200_REFILL_MIN", 0); t.refill_min = m < 1 ? 0u : m > 32 ? 32u : (uint32_t)m; }   // 0: auto
        if (getenv("BVH_B200_INNER_BUDGET")) {                  // unset: auto
            const long budget = env("BVH_B200_INNER_BUDGET", 0);
            t.inner_budget = budget <= 0 ? 0xFFFFFFFFu : (uint32_t)budget;
        }
        const long wbudget = env("BVH_B200_WIDE_BUDGET", 4);
        t.wide_budget = wbudget <= 0 ? 0xFFFFFFFFu : (uint32_t)wbudget;
        t.watchdog = (uint32_t)env("BVH_B200_WATCHDOG", 1l << 26);
        t.stack_round = (int)env("BVH_B200_STACK_ROUND", 2);
        t.chunk_rays = (uint32_t)env("BVH_B200_CHUNK_RAYS", 64);
        t.smem_carveout = (int)env("BVH_B200_SMEM_CARVEOUT", -1);
        t.gather_staging = (int)env("BVH_B200_GATHER_STAGING", 1);
        t.sort_onesweep = (int)env("BVH_B200_SORT_ONESWEEP", 1);
        t.treelet_blocks = (int)env("BVH_B200_TREELET_BLOCKS", 3);
    });
    return t;
}

static thread_local int g_device = 0;
static thread_local cudaStream_t g_user_stream = nullptr;
static thread_local bool g_have_user_stream = false;

// One PRIVATE memory pool per device (stream-ordered allocation): freed blocks stay cached in it so that
// rebuilds never go back to the driver, without touching the process-wide default pool of the host
// application (bvh_cuda_trim() hands the cached memory back).
static std::mutex g_pool_mutex;
static cudaMemPool_t g_pools[64] = {};

int prepare_device(int device) {
    if (device < 0 || device >= 64) { set_error("device index out of range"); return -1; }
    std::lock_guard<std::mutex> lock(g_pool_mutex);
    if (!g_pools[device]) {
        cudaMemPoolProps props = {};
        props.allocType = cudaMemAllocationTypePinned;
        props.handleTypes = cudaMemHandleTypeNone;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = device;
        cudaMemPool_t pool;
        BVH_CUDA_TRY(cudaMemPoolCreate(&pool, &props));
        unsigned long long threshold = ~0ull;
        BVH_CUDA_TRY(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold));
        g_pools[device] = pool;
    }
    return 0;
}

int device_alloc(void** ptr, size_t bytes, cudaStream_t stream) {
    *ptr = nullptr;
    int device = 0;
    BVH_CUDA_TRY(cudaGetDevice(&device));
    cudaMemPool_t pool = nullptr;
    if (device >= 0 && device < 64) { std::lock_guard<std::mutex> lock(g_pool_mutex); pool = g_pools[device]; }
    if (!pool) { if (prepare_device(device)) return -1; std::lock_guard<std::mutex> lock(g_pool_mutex); pool = g_pools[device]; }
    BVH_CUDA_TRY(cudaMallocFromPoolAsync(ptr, bytes ? bytes : 16, pool, stream));
    return 0;
}
void device_free(void* ptr, cudaStream_t stream) { if (ptr) cudaFreeAsync(ptr, stream); }

// Every entry point runs on the handle's device and puts the caller's current device back afterwards.
struct DeviceGuard {
    int prev = -1, dev;
    bool ok = true;
    explicit DeviceGuard(int device) : dev(device) {
        if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; }
        if (prev != dev && cudaSetDevice(dev) != cudaSuccess) {
            set_error(std::string("cudaSetDevice: ") + cudaGetErrorString(cudaGetLastError()));
            ok = false;
        }
    }
    ~DeviceGuard() { if (prev >= 0 && prev != dev) cudaSetDevice(prev); }
};
#define BVH_ON_DEVICE(device) DeviceGuard device_guard__(device); if (!device_guard__.ok) return -1

// ---- host mirror ------------------------------------------------------------------------------
template <typename T> struct HostNode { T bounds[6]; typename Real<T>::UInt index; };
static_assert(sizeof(HostNode<float>) == 28 && sizeof(HostNode<double>) == 56, "reference Node<T,3> layout");

template <typename T> struct Handle {
    using U = typename Real<T>::UInt;
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    DeviceBvh<T> dev;
    bool device_valid = false;

    std::vector<HostNode<T>> nodes;           // reference layout
    std::vector<size_t> prim_ids;
    bool host_valid = false;
    bool maybe_edited = false;                // a mutable node pointer was handed out since the last upload
    uint64_t synced_hash = 0;
    uint64_t synced_ids_hash = 0;             // hash of prim_ids the device triangles were permuted with

    // staging and side streams for host-pointer batches
    static constexpr size_t kMaxChunks = 16;
    static constexpr size_t kDefaultChunks = 8;   // measured: 8 chunks of a 10M-ray batch overlap best
    cudaStream_t copy_in = nullptr, copy_out = nullptr;
    cudaEvent_t events[1 + 2 * kMaxChunks] = {};
    void* d_rays = nullptr; size_t d_rays_bytes = 0;
    void* d_hits = nullptr; size_t d_hits_bytes = 0;
    void* d_stats = nullptr; size_t d_stats_bytes = 0;
    // Batched calls on one handle share its stream, staging buffers and the kernels' cursor/status words:
    // concurrent callers are serialised (the reference's per-ray calls are const and run on the host mirror).
    std::mutex batch_mutex;
    std::mutex mirror_mutex;                      // the lazy download of the mirror (first legacy call) happens once
};

template <typename T> int init_handle(Handle<T>& h) {
    h.device = g_device;                        // (the caller holds a DeviceGuard on g_device)
    if (prepare_device(h.device)) return -1;
    h.dev.device = h.device;
    if (g_have_user_stream) { h.stream = g_user_stream; h.own_stream = false; }
    else { BVH_CUDA_TRY(cudaStreamCreateWithFlags(&h.stream, cudaStreamNonBlocking)); h.own_stream = true; }
    return 0;
}

template <typename T> void destroy_handle(Handle<T>* h) {
    if (!h) return;
    DeviceGuard guard(h->device);
    release(h->dev, h->stream);
    device_free(h->d_rays, h->stream); device_free(h->d_hits, h->stream); device_free(h->d_stats, h->stream);
    cudaStreamSynchronize(h->stream);
    if (h->copy_in) {
        cudaStreamDestroy(h->copy_in); cudaStreamDestroy(h->copy_out);
        for (auto& e : h->events) if (e) cudaEventDestroy(e);
    }
    if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

static uint64_t hash_bytes(const void* data, size_t size, uint64_t seed) {
    // FNV-1a over 64-bit words (the tail bytewise); only used to detect edits of the mirror
    uint64_t h = 1469598103934665603ull ^ seed;
    const unsigned char* p = static_cast<const unsigned char*>(data);
    size_t words = size / 8;
    for (size_t i = 0; i < words; ++i) { uint64_t w; std::memcpy(&w, p + 8 * i, 8); h = (h ^ w) * 1099511628211ull; }
    for (size_t i = words * 8; i < size; ++i) h = (h ^ p[i]) * 1099511628211ull;
    return h;
}

template <typename T> uint64_t ids_hash(const Handle<T>& h) {
    return hash_bytes(h.prim_ids.data(), h.prim_ids.size() * sizeof(size_t), h.prim_ids.size());
}

template <typename T> uint64_t mirror_hash(const Handle<T>& h) {
    uint64_t a = hash_bytes(h.nodes.data(), h.nodes.size() * sizeof(HostNode<T>), h.nodes.size());
    return hash_bytes(h.prim_ids.data(), h.prim_ids.size() * sizeof(size_t), a);
}

// Device -> mirror.  The device array is dense and in the reference's numbering (root at 0, children of a node
// adjacent, left child at an odd index, bvh.h:34-54), shifted by one slot: the export kernels strip the padding
// on the device and the records land in the mirror with one copy per array.
template <typename T> int download_mirror(Handle<T>& h) {
    std::lock_guard<std::mutex> lock(h.mirror_mutex);       // concurrent bvhNN_intersect_ray* callers (bvh_impl.h:244)
    if (h.host_valid) return 0;
    if (!h.device_valid) { set_error("handle holds no BVH"); return -1; }
    BVH_ON_DEVICE(h.device);
    static_assert(sizeof(size_t) == sizeof(unsigned long long), "prim ids are copied as 64-bit words");
    const size_t node_count = h.dev.node_slots - 1, prim_count = h.dev.prim_count;
    void* d_nodes = nullptr; void* d_ids = nullptr;
    if (device_alloc(&d_nodes, node_count * sizeof(HostNode<T>), h.stream)) return -1;
    if (device_alloc(&d_ids, prim_count * sizeof(unsigned long long), h.stream)) { device_free(d_nodes, h.stream); return -1; }
    int rc = export_reference_arrays(h.dev, d_nodes, static_cast<unsigned long long*>(d_ids), h.stream);
    if (!rc) {
        try { h.nodes.resize(node_count); h.prim_ids.resize(prim_count); }
        catch (const std::exception&) { set_error("download: out of host memory"); rc = -1; }
    }
    cudaError_t err = cudaSuccess;
    if (!rc) err = cudaMemcpyAsync(h.nodes.data(), d_nodes, node_count * sizeof(HostNode<T>), cudaMemcpyDeviceToHost, h.stream);
    if (!rc && err == cudaSuccess) err = cudaMemcpyAsync(h.prim_ids.data(), d_ids, prim_count * sizeof(size_t), cudaMemcpyDeviceToHost, h.stream);
    if (!rc && err == cudaSuccess) err = cudaStreamSynchronize(h.stream);
    device_free(d_nodes, h.stream); device_free(d_ids, h.stream);
    if (rc) return -1;
    if (err != cudaSuccess) { set_error(std::string("download: ") + cudaGetErrorString(err)); return -1; }
    h.host_valid = true;
    h.maybe_edited = false;
    h.synced_ids_hash = ids_hash(h);
    return 0;
}

// Mirror -> device: reference node i goes to device slot i + 1, padded to 32 / 64 bytes.
template <typename T> int upload_mirror(Handle<T>& h) {
    BVH_ON_DEVICE(h.device);
    const size_t node_count = h.nodes.size();
    if (node_count == 0) { set_error("upload: empty BVH"); return -1; }
    std::vector<DevNode<T>> dev_nodes(node_count + 1);
    std::memset(dev_nodes.data(), 0, sizeof(DevNode<T>));
    for (size_t i = 0; i < node_count; ++i) {
        std::memcpy(dev_nodes[i + 1].bounds, h.nodes[i].bounds, sizeof(h.nodes[i].bounds));
        dev_nodes[i + 1].index = h.nodes[i].index;
        dev_nodes[i + 1].pad = 0;
    }
    std::vector<uint32_t> ids(h.prim_ids.size());
    for (size_t i = 0; i < ids.size(); ++i) {
        if (h.prim_ids[i] >= ids.size()) { set_error("upload: primitive id out of range"); return -1; }
        ids[i] = (uint32_t)h.prim_ids[i];
    }

    // depth = longest chain of inner nodes (bounds the traversal stack); also validates child indices
    uint32_t depth = 0;
    {
        std::vector<std::pair<size_t, uint32_t>> stack;
        stack.emplace_back(0, 0);
        size_t visited = 0;
        while (!stack.empty()) {
            auto [i, d] = stack.back();
            stack.pop_back();
            if (++visited > node_count) { set_error("upload: the node graph is not a tree"); return -1; }
            if (const uint32_t leaf_count = index_count(h.nodes[i].index)) {
                // the kernels index tris[first .. first + count) and prim_ids[slot] without further checks
                if ((size_t)index_first(h.nodes[i].index) + leaf_count > ids.size()) { set_error("upload: leaf range exceeds the primitive count"); return -1; }
                continue;
            }
            const size_t first = (size_t)index_first(h.nodes[i].index);
            if (first == 0 || first + 1 >= node_count) { set_error("upload: child index out of range"); return -1; }
            depth = std::max(depth, d + 1);
            stack.emplace_back(first, d + 1);
            stack.emplace_back(first + 1, d + 1);
        }
    }

    const bool had_tris = h.dev.tris != nullptr && h.dev.prim_count == ids.size();
    DevTri<T>* keep_tris = had_tris ? h.dev.tris : nullptr;
    if (had_tris) h.dev.tris = nullptr;
    release(h.dev, h.stream);
    h.dev.device = h.device;
    h.dev.prim_count = (uint32_t)ids.size();
    h.dev.node_slots = dev_nodes.size();
    h.dev.depth = depth;
    h.dev.compact = true;
    h.dev.tris = keep_tris;
    if (device_alloc(reinterpret_cast<void**>(&h.dev.nodes), dev_nodes.size() * sizeof(DevNode<T>), h.stream)) return -1;
    if (device_alloc(reinterpret_cast<void**>(&h.dev.prim_ids), ids.size() * sizeof(uint32_t), h.stream)) return -1;
    BVH_CUDA_TRY(cudaMemcpyAsync(h.dev.nodes, dev_nodes.data(), dev_nodes.size() * sizeof(DevNode<T>), cudaMemcpyHostToDevice, h.stream));
    BVH_CUDA_TRY(cudaMemcpyAsync(h.dev.prim_ids, ids.data(), ids.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, h.stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(h.stream));
    if (rebuild_wide(h.dev, h.stream)) return -1;
    h.device_valid = true;
    h.maybe_edited = false;
    h.synced_hash = mirror_hash(h);
    h.synced_ids_hash = ids_hash(h);
    return 0;
}

// Called before any batched call: make the device copy current.
template <typename T> int ensure_device(Handle<T>& h) {
    if (h.device_valid && !(h.host_valid && h.maybe_edited)) return 0;
    if (!h.host_valid) { set_error("handle holds no BVH"); return -1; }
    if (h.device_valid && mirror_hash(h) == h.synced_hash) { h.maybe_edited = false; return 0; }
    // if the primitive order was edited the BVH-order triangles are stale: drop them
    if (h.device_valid && h.dev.tris && ids_hash(h) != h.synced_ids_hash) { device_free(h.dev.tris, h.stream); h.dev.tris = nullptr; }
    return upload_mirror(h);
}

// ---- reference semantics on the mirror ---------------------------------------------------------
// Bvh::refit with no leaf function (reference bvh.h:184-218; c_api/bvh_impl.h:218-221).
template <typename T, int kDim, typename NodeVec> void refit_nodes(NodeVec& nodes) {
    const size_t n = nodes.size();
    std::vector<size_t> parents(n, 0);
    std::vector<unsigned char> seen(n, 0);
    for (size_t i = 0; i < n; ++i) {
        if (index_count(nodes[i].index) != 0) continue;
        const size_t first = (size_t)index_first(nodes[i].index);
        if (first + 1 < n) { parents[first] = i; parents[first + 1] = i; }
    }
    for (size_t i = n; i-- > 0;) {
        if (index_count(nodes[i].index) == 0) continue;
        seen[i] = 1;
        for (size_t j = parents[i];; j = parents[j]) {
            auto& node = nodes[j];
            const size_t first = (size_t)index_first(node.index);
            if (seen[j] || index_count(node.index) != 0 || first + 1 >= n || !seen[first] || !seen[first + 1]) break;
            const auto& l = nodes[first];
            const auto& r = nodes[first + 1];
            for (int k = 0; k < kDim; ++k) {
                node.bounds[2 * k]     = robust_min(l.bounds[2 * k], r.bounds[2 * k]);
                node.bounds[2 * k + 1] = robust_max(l.bounds[2 * k + 1], r.bounds[2 * k + 1]);
            }
            seen[j] = 1;
            if (j == 0) break;
        }
    }
}
template <typename T> void refit_mirror(Handle<T>& h) { refit_nodes<T, 3>(h.nodes); }

// Bvh::intersect for one ray with a host callback (reference bvh.h:124-182, c_api/bvh_impl.h:235-250).
// `nodes` is the mirror in the reference layout (Node<T, kDim>), `ray` = org[kDim] dir[kDim] tmin tmax.
template <typename T, bool kAny, bool kRobust, int kDim, typename NodeVec, typename Callback>
void intersect_nodes(const NodeVec& nodes, const T* ray, const Callback* cb) {
    using U = typename Real<T>::UInt;
    RayCtx<T> r;
    for (int k = 0; k < 3; ++k) { r.org[k] = 0; r.dir[k] = 0; r.inv_dir[k] = 0; r.aux[k] = 0; }
    for (int k = 0; k < kDim; ++k) { r.org[k] = ray[k]; r.dir[k] = ray[kDim + k]; }
    r.tmin = ray[2 * kDim]; r.tmax = ray[2 * kDim + 1];
    ray_prologue<T, kRobust, kDim>(r);
    // SmallStack<Index, 64> (bvh_impl.h:241) that spills to the heap instead of asserting (stack.h:21): an LBVH
    // over 63-bit keys with duplicate runs can be up to 91 levels deep.
    U fixed[64];
    std::vector<U> spill;
    U* stack = fixed;
    size_t capacity = 64, sp = 0;
    auto push = [&] (U v) {
        if (sp == capacity) {
            if (stack == fixed) spill.assign(fixed, fixed + sp);
            spill.resize(2 * capacity);                     // (keeps the entries already spilled)
            stack = spill.data(); capacity *= 2;
        }
        stack[sp++] = v;
    };
    U top = nodes[0].index;
    for (;;) {
        bool alive = true;
        while (index_count(top) == 0) {
            const auto& left = nodes[(size_t)index_first(top)];
            const auto& right = nodes[(size_t)index_first(top) + 1];
            T l0, l1, r0, r1;
            node_test<T, kRobust, kDim>(left.bounds, r, l0, l1);
            node_test<T, kRobust, kDim>(right.bounds, r, r0, r1);
            const bool hl = l0 <= l1, hr = r0 <= r1;
            if (hl) {
                U near_i = left.index;
                if (hr) {
                    U far_i = right.index;
                    if (!kAny && l0 > r0) std::swap(near_i, far_i);
                    push(far_i);
                }
                top = near_i;
            } else if (hr) top = right.index;
            else { if (sp == 0) { alive = false; break; } top = stack[--sp]; }
        }
        if (!alive) break;
        const size_t begin = (size_t)index_first(top), end = begin + index_count(top);
        const bool was_hit = cb->user_fn(cb->user_data, &r.tmax, begin, end);
        if (kAny && was_hit) break;
        if (sp == 0) break;
        top = stack[--sp];
    }
}

template <typename T, bool kAny, bool kRobust, typename Callback>
void intersect_mirror(const Handle<T>& h, const T* ray8, const Callback* cb) {
    intersect_nodes<T, kAny, kRobust, 3>(h.nodes, ray8, cb);
}

template <typename T> BuildOptions translate_config(const bvh_build_config* config) {
    BuildOptions o;                                         // defaults of DefaultBuilder::Config
    if (config) {
        o.quality = (int)config->quality;
        o.min_leaf = (uint32_t)std::min<size_t>(config->min_leaf_size ? config->min_leaf_size : 1, 15);
        o.max_leaf = (uint32_t)std::min<size_t>(config->max_leaf_size ? config->max_leaf_size : 1, 15);
    }
    return o;
}

// Copies a host array to the device (or passes a device pointer through).
template <typename X> struct DeviceInput {
    const X* ptr = nullptr;
    void* owned = nullptr;
    cudaStream_t stream;
    explicit DeviceInput(cudaStream_t s) : stream(s) {}
    ~DeviceInput() { device_free(owned, stream); }
    int set(const X* src, size_t count, bool is_device) {
        if (is_device) { ptr = src; return 0; }
        if (device_alloc(&owned, count * sizeof(X), stream)) return -1;
        BVH_CUDA_TRY(cudaMemcpyAsync(owned, src, count * sizeof(X), cudaMemcpyHostToDevice, stream));
        ptr = static_cast<const X*>(owned);
        return 0;
    }
};

template <typename T>
Handle<T>* build_handle(const T* verts, const T* bboxes, const T* centers, size_t n,
                        const bvh_build_config* config, bool device_ptrs) {
    if (n == 0 || n > 0xFFFFFFFFull) { set_error("build: prim_count out of range"); return nullptr; }
    DeviceGuard guard(g_device);
    if (!guard.ok) return nullptr;
    auto h = new Handle<T>();
    if (init_handle(*h)) { delete h; return nullptr; }
    int rc = 0;
    {
        DeviceInput<T> dv(h->stream), db(h->stream), dc(h->stream);
        if (verts) rc = dv.set(verts, 9 * n, device_ptrs);
        else { rc = db.set(bboxes, 6 * n, device_ptrs); if (!rc) rc = dc.set(centers, 3 * n, device_ptrs); }
        if (!rc) rc = build_lbvh<T>(h->dev, dv.ptr, db.ptr, dc.ptr, (uint32_t)n, translate_config<T>(config), h->stream);
    }
    if (rc) { destroy_handle(h); return nullptr; }
    h->device_valid = true;
    return h;
}

template <typename T> int ensure_staging(Handle<T>& h, void** buf, size_t* cap, size_t bytes) {
    if (*cap >= bytes) return 0;
    device_free(*buf, h.stream);
    *buf = nullptr; *cap = 0;
    if (device_alloc(buf, bytes, h.stream)) return -1;
    *cap = bytes;
    return 0;
}

static unsigned translate_flags(unsigned flags) {
    unsigned tf = 0;
    if (flags & BVH_ANY_HIT) tf |= kTraceAnyHit;
    if (flags & BVH_ROBUST) tf |= kTraceRobust;
    if (flags & BVH_TIE_LAST_VISITED) tf |= kTraceLastVisited;
    if (flags & BVH_KERNEL_SIMPLE) tf |= kTraceSimple;
    if (flags & BVH_KERNEL_NO_TMA) tf |= kTraceNoTma;
    if (flags & BVH_KERNEL_TMA) tf |= kTraceTma;
    if (flags & BVH_KERNEL_PAIR) tf |= kTracePair;
    if (flags & BVH_KERNEL_WIDE) tf |= kTraceWide;
    if (flags & BVH_SORT_RAYS) tf |= kTraceSortRays;
    return tf;
}

template <typename T, typename RayPod, typename HitPod>
int intersect_batch(Handle<T>* h, const RayPod* rays, size_t n, HitPod* hits, bvh_ray_stats* stats, unsigned flags) {
    static_assert(sizeof(RayPod) == sizeof(DevRay<T>) && sizeof(HitPod) == sizeof(DevHit<T>), "POD layouts");
    if (!h) { set_error("null handle"); return -1; }
    if (n == 0) return 0;
    std::lock_guard<std::mutex> lock(h->batch_mutex);
    BVH_ON_DEVICE(h->device);
    if (ensure_device(*h)) return -1;
    const unsigned tf = translate_flags(flags);
    if (flags & BVH_DEVICE_POINTERS) {
        return trace_rays<T>(h->dev, reinterpret_cast<const DevRay<T>*>(rays), reinterpret_cast<DevHit<T>*>(hits), n, tf,
                             reinterpret_cast<uint32_t*>(stats), h->stream);
    }
    // Host buffers: the batch is cut into chunks and software-pipelined over three streams — H2D of
    // chunk k+1 (copy-in stream), traversal of chunk k (the handle's stream) and D2H of chunk k-1
    // (copy-out stream) overlap, so a PCIe-bound call costs about max(H2D, trace, D2H), not their sum.
    if (ensure_staging(*h, &h->d_rays, &h->d_rays_bytes, n * sizeof(RayPod))) return -1;
    if (ensure_staging(*h, &h->d_hits, &h->d_hits_bytes, n * sizeof(HitPod))) return -1;
    if (stats && ensure_staging(*h, &h->d_stats, &h->d_stats_bytes, n * sizeof(bvh_ray_stats))) return -1;
    if (!h->copy_in) {
        BVH_CUDA_TRY(cudaStreamCreateWithFlags(&h->copy_in, cudaStreamNonBlocking));
        BVH_CUDA_TRY(cudaStreamCreateWithFlags(&h->copy_out, cudaStreamNonBlocking));
        for (auto& e : h->events) BVH_CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    auto d_rays = static_cast<DevRay<T>*>(h->d_rays);
    auto d_hits = static_cast<DevHit<T>*>(h->d_hits);
    auto d_stats = static_cast<uint32_t*>(h->d_stats);
    constexpr size_t kMinChunk = 1u << 20;                   // 1M rays = 32 MB of float rays per chunk
    size_t chunks = n / kMinChunk;
    if (chunks > Handle<T>::kDefaultChunks) chunks = Handle<T>::kDefaultChunks;
    if (const int forced = tunables().e2e_chunks.load()) chunks = (size_t)(forced > 0 ? forced : 1);   // experiments only
    if (chunks < 1) chunks = 1;
    if (chunks > Handle<T>::kMaxChunks) chunks = Handle<T>::kMaxChunks;
    // the staging buffers may still be in use by earlier work on the handle's stream
    BVH_CUDA_TRY(cudaEventRecord(h->events[0], h->stream));
    BVH_CUDA_TRY(cudaStreamWaitEvent(h->copy_in, h->events[0], 0));
    // Equal chunks (chunk sizes tapering towards the end were no faster on an earlier GPU).  Upload and download share
    // the PCIe link: the call is bound by the combined copy traffic whatever the schedule.
    for (size_t c = 0; c < chunks; ++c) {
        const size_t b = n * c / chunks, e = n * (c + 1) / chunks;
        cudaEvent_t in_done = h->events[1 + 2 * c], tr_done = h->events[2 + 2 * c];
        BVH_CUDA_TRY(cudaMemcpyAsync(d_rays + b, rays + b, (e - b) * sizeof(RayPod), cudaMemcpyHostToDevice, h->copy_in));
        BVH_CUDA_TRY(cudaEventRecord(in_done, h->copy_in));
        BVH_CUDA_TRY(cudaStreamWaitEvent(h->stream, in_done, 0));
        if (trace_rays<T>(h->dev, d_rays + b, d_hits + b, e - b, tf, stats ? d_stats + 3 * b : nullptr, h->stream)) return -1;
        BVH_CUDA_TRY(cudaEventRecord(tr_done, h->stream));
        BVH_CUDA_TRY(cudaStreamWaitEvent(h->copy_out, tr_done, 0));
        BVH_CUDA_TRY(cudaMemcpyAsync(hits + b, d_hits + b, (e - b) * sizeof(HitPod), cudaMemcpyDeviceToHost, h->copy_out));
        if (stats) BVH_CUDA_TRY(cudaMemcpyAsync(stats + b, d_stats + 3 * b, (e - b) * sizeof(bvh_ray_stats), cudaMemcpyDeviceToHost, h->copy_out));
    }
    BVH_CUDA_TRY(cudaStreamSynchronize(h->copy_out));
    return check_trace_status(h->dev, h->stream);
}

// reference bvh.h:220-242 / node.h:90-102: [node_count][prim_count] nodes (6 bounds + index) prim ids
template <typename T> void save_mirror(Handle<T>& h, FILE* file) {
    using U = typename Real<T>::UInt;
    if (download_mirror(h)) return;
    U v = (U)h.nodes.size(); fwrite(&v, sizeof v, 1, file);
    v = (U)h.prim_ids.size(); fwrite(&v, sizeof v, 1, file);
    for (const auto& n : h.nodes) { fwrite(n.bounds, sizeof(T), 6, file); fwrite(&n.index, sizeof(U), 1, file); }
    for (size_t id : h.prim_ids) { v = (U)id; fwrite(&v, sizeof v, 1, file); }
}

template <typename T> Handle<T>* load_mirror(FILE* file) {
    using U = typename Real<T>::UInt;
    DeviceGuard guard(g_device);
    if (!guard.ok) return nullptr;
    auto h = new Handle<T>();
    if (init_handle(*h)) { delete h; return nullptr; }
    U node_count = 0, prim_count = 0;                       // short reads give defaults (stream.h:13-18)
    if (fread(&node_count, sizeof(U), 1, file) != 1) node_count = 0;
    if (fread(&prim_count, sizeof(U), 1, file) != 1) prim_count = 0;
    // A corrupt header must not turn into a multi-gigabyte resize: the counts are bounded by what the file
    // still holds (seekable streams) and allocation failures never cross the C boundary.
    const long here = ftell(file);
    if (here >= 0 && fseek(file, 0, SEEK_END) == 0) {
        const long end = ftell(file);
        fseek(file, here, SEEK_SET);
        const double need = (double)node_count * (6 * sizeof(T) + sizeof(U)) + (double)prim_count * sizeof(U);
        if (end >= here && need > (double)(end - here)) {
            set_error("load: the header announces more nodes / primitives than the file holds");
            destroy_handle(h);
            return nullptr;
        }
    }
    try {
        h->nodes.resize((size_t)node_count);
        h->prim_ids.resize((size_t)prim_count);
    } catch (const std::exception&) {
        set_error("load: out of memory for the announced node / primitive counts");
        destroy_handle(h);
        return nullptr;
    }
    for (auto& n : h->nodes) {
        std::memset(&n, 0, sizeof n);
        if (fread(n.bounds, sizeof(T), 6, file) != 6) std::memset(n.bounds, 0, sizeof n.bounds);
        if (fread(&n.index, sizeof(U), 1, file) != 1) n.index = 0;
    }
    for (auto& id : h->prim_ids) { U v = 0; if (fread(&v, sizeof(U), 1, file) != 1) v = 0; id = (size_t)v; }
    h->host_valid = true;
    h->device_valid = false;
    return h;
}

// ---- 2-D suffixes (reference c_api/bvh.cpp:7-25 instantiates bvh2f / bvh2d next to the 3-D ones) ----------
// The reference has no 2-D primitive type: leaves are intersected by the caller's callback, one ray per call,
// so there is no batched device traversal to offer here.  What the GPU does is the BUILD: the boxes are lifted
// to z = 0, the LBVH pipeline runs as for 3-D (the z bits of the Morton keys are all zero, so the order is the
// 2-D Z-curve), and the result comes back as a host tree of the reference's Node<T, 2> (4 bounds + index,
// 20 / 40 bytes) on which every other entry point works exactly as the reference's does.
template <typename T> struct HostNode2 { T bounds[4]; typename Real<T>::UInt index; };
static_assert(sizeof(HostNode2<float>) == 20 && sizeof(HostNode2<double>) == 40, "reference Node<T,2> layout");

template <typename T> struct Handle2 {
    std::vector<HostNode2<T>> nodes;
    std::vector<size_t> prim_ids;
};

template <typename T>
Handle2<T>* build_handle2(const T* bboxes4, const T* centers2, size_t n, const bvh_build_config* config) {
    if (n == 0) { set_error("build: prim_count out of range"); return nullptr; }
    std::vector<T> boxes(6 * n), centers(3 * n);
    for (size_t i = 0; i < n; ++i) {                       // bvh_bbox2 = {min.x, min.y, max.x, max.y}
        boxes[6 * i + 0] = bboxes4[4 * i + 0]; boxes[6 * i + 1] = bboxes4[4 * i + 1]; boxes[6 * i + 2] = 0;
        boxes[6 * i + 3] = bboxes4[4 * i + 2]; boxes[6 * i + 4] = bboxes4[4 * i + 3]; boxes[6 * i + 5] = 0;
        centers[3 * i + 0] = centers2[2 * i + 0]; centers[3 * i + 1] = centers2[2 * i + 1]; centers[3 * i + 2] = 0;
    }
    Handle<T>* lifted = build_handle<T>(nullptr, boxes.data(), centers.data(), n, config, false);
    if (!lifted) return nullptr;
    if (download_mirror(*lifted)) { destroy_handle(lifted); return nullptr; }
    auto h = new Handle2<T>();
    h->nodes.resize(lifted->nodes.size());
    for (size_t i = 0; i < h->nodes.size(); ++i) {
        std::memcpy(h->nodes[i].bounds, lifted->nodes[i].bounds, 4 * sizeof(T));
        h->nodes[i].index = lifted->nodes[i].index;
    }
    h->prim_ids = lifted->prim_ids;
    destroy_handle(lifted);
    return h;
}

template <typename T> void save_nodes2(const Handle2<T>& h, FILE* file) {
    using U = typename Real<T>::UInt;
    U v = (U)h.nodes.size(); fwrite(&v, sizeof v, 1, file);
    v = (U)h.prim_ids.size(); fwrite(&v, sizeof v, 1, file);
    for (const auto& n : h.nodes) { fwrite(n.bounds, sizeof(T), 4, file); fwrite(&n.index, sizeof(U), 1, file); }
    for (size_t id : h.prim_ids) { v = (U)id; fwrite(&v, sizeof v, 1, file); }
}

template <typename T> Handle2<T>* load_nodes2(FILE* file) {
    using U = typename Real<T>::UInt;
    auto h = new Handle2<T>();
    U node_count = 0, prim_count = 0;
    if (fread(&node_count, sizeof(U), 1, file) != 1) node_count = 0;
    if (fread(&prim_count, sizeof(U), 1, file) != 1) prim_count = 0;
    h->nodes.resize((size_t)node_count);
    h->prim_ids.resize((size_t)prim_count);
    for (auto& n : h->nodes) {
        std::memset(&n, 0, sizeof n);
        if (fread(n.bounds, sizeof(T), 4, file) != 4) std::memset(n.bounds, 0, sizeof n.bounds);
        if (fread(&n.index, sizeof(U), 1, file) != 1) n.index = 0;
    }
    for (auto& id : h->prim_ids) { U v = 0; if (fread(&v, sizeof(U), 1, file) != 1) v = 0; id = (size_t)v; }
    return h;
}

// bvhNN_optimize (reference c_api/bvh_impl.h:223-233): with a pool the search runs on the pool's thread count
// (0 = hardware concurrency, thread_pool.h:82-86), without one it is serial (SequentialExecutor).
static size_t optimizer_threads(size_t requested) {
    if (requested != 0) return requested;
    const unsigned hw = std::thread::hardware_concurrency();
    return hw ? hw : 1;
}
template <typename T, int kDim, typename NodeVec>
bool optimize_nodes(NodeVec& nodes, double ratio, size_t iters, size_t threads) {
    using NodeT = typename NodeVec::value_type;
    try {
        if (!Reinserter<T, kDim, NodeT>(nodes, threads).run((T)ratio, iters)) { set_error("optimize: the node array is not a well-formed tree"); return false; }
    } catch (const std::exception& e) { set_error(std::string("optimize: ") + e.what()); return false; }
    return true;
}

} // namespace bvhb200

using namespace bvhb200;

// ---- exported symbols ---------------------------------------------------------------------------
extern "C" {

BVH_EXPORT const char* bvh_last_error(void) { return last_error(); }
BVH_EXPORT int bvh_cuda_device_count(void) {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess) { cudaGetLastError(); return 0; }
    return count;
}
BVH_EXPORT int bvh_cuda_set_device(int device) {
    if (device < 0 || device >= bvh_cuda_device_count()) { set_error("no such CUDA device"); return -1; }
    g_device = device;
    return 0;
}
BVH_EXPORT void bvh_cuda_set_stream(void* cuda_stream) {
    g_user_stream = static_cast<cudaStream_t>(cuda_stream);
    g_have_user_stream = true;
}
BVH_EXPORT void bvh_cuda_reset_stream(void) { g_user_stream = nullptr; g_have_user_stream = false; }
BVH_EXPORT void* bvh_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes ? bytes : 16) != cudaSuccess) { set_error("cudaMallocHost failed"); cudaGetLastError(); return nullptr; }
    return p;
}
BVH_EXPORT void bvh_host_free(void* ptr) { if (ptr) cudaFreeHost(ptr); }
BVH_EXPORT int bvh_set_option(const char* name, long value) {
    if (!name) { set_error("set_option: null name"); return -1; }
    Tunables& t = tunables();
    const std::string n = name;
    if (n == "morton_bits") t.morton_bits = (int)value;
    else if (n == "sah_treelets") t.sah_treelets = (int)value;
    else if (n == "hierarchy") t.hierarchy = (int)value;
    else if (n == "e2e_chunks") t.e2e_chunks = (int)value;
    else if (n == "variant") t.variant = (int)value;
    else if (n == "use_wide") t.use_wide = (int)value;
    else if (n == "chunk_rays") t.chunk_rays = value < 32 ? 32u : (uint32_t)value;
    else if (n == "stack_round") t.stack_round = value < 1 ? 1 : (int)value;
    else if (n == "smem_carveout") t.smem_carveout = (int)value;
    else if (n == "refill_min") t.refill_min = value < 1 ? 0u : value > 32 ? 32u : (uint32_t)value;     // 0: auto
    else if (n == "inner_budget") t.inner_budget = value <= 0 ? 0xFFFFFFFFu : (uint32_t)value;
    else if (n == "wide_budget") t.wide_budget = value <= 0 ? 0xFFFFFFFFu : (uint32_t)value;
    else if (n == "watchdog") t.watchdog = (uint32_t)value;
    else if (n == "gather_staging") t.gather_staging = (int)value;
    else if (n == "sort_onesweep") t.sort_onesweep = (int)value;
    else if (n == "treelet_blocks") t.treelet_blocks = (int)value;
    else { set_error("set_option: unknown option " + n); return -1; }
    return 0;
}
BVH_EXPORT int bvh_cuda_trim(int device) {
    if (device < 0 || device >= 64) { set_error("no such CUDA device"); return -1; }
    cudaMemPool_t pool;
    { std::lock_guard<std::mutex> lock(g_pool_mutex); pool = g_pools[device]; }
    if (pool) BVH_CUDA_TRY(cudaMemPoolTrimTo(pool, 0));
    return 0;
}

// The pool is an API token only: CUDA streams do the work that ThreadPool does in the reference.
struct bvh_thread_pool { size_t thread_count; };
static size_t pool_threads(const bvh_thread_pool* pool) { return pool ? optimizer_threads(pool->thread_count) : 1; }
BVH_EXPORT int bvh_optimize_nodes(void* nodes, size_t node_count, int dim, int is_double, double ratio, size_t iters, size_t threads) {
    if (!nodes && node_count) { set_error("optimize: null node array"); return -1; }
    if (dim != 2 && dim != 3) { set_error("optimize: dim must be 2 or 3"); return -1; }
    // the Reinserter works on a std::vector; the caller's array is copied in and out (host memory, O(node_count))
    auto run = [&] (auto tag_node, auto tag_scalar, auto tag_dim) {
        using NodeT = decltype(tag_node); using T = decltype(tag_scalar); constexpr int D = decltype(tag_dim)::value;
        std::vector<NodeT> v(static_cast<NodeT*>(nodes), static_cast<NodeT*>(nodes) + node_count);
        if (!optimize_nodes<T, D>(v, ratio, iters, optimizer_threads(threads))) return -1;
        std::memcpy(nodes, v.data(), node_count * sizeof(NodeT));
        return 0;
    };
    try {
        if (dim == 3) return is_double ? run(HostNode<double>{}, double{}, std::integral_constant<int, 3>{})
                                       : run(HostNode<float>{}, float{}, std::integral_constant<int, 3>{});
        return is_double ? run(HostNode2<double>{}, double{}, std::integral_constant<int, 2>{})
                         : run(HostNode2<float>{}, float{}, std::integral_constant<int, 2>{});
    } catch (const std::exception& e) { set_error(std::string("optimize: ") + e.what()); return -1; }
}
BVH_EXPORT struct bvh_thread_pool* bvh_thread_pool_create(size_t thread_count) { return new bvh_thread_pool { thread_count }; }
BVH_EXPORT void bvh_thread_pool_destroy(struct bvh_thread_pool* pool) { delete pool; }

#define H(T, bvh) (reinterpret_cast<Handle<T>*>(bvh))
#define HC(T, bvh) (const_cast<Handle<T>*>(reinterpret_cast<const Handle<T>*>(bvh)))
#define N(T, node) (reinterpret_cast<HostNode<T>*>(node))
#define NC(T, node) (reinterpret_cast<const HostNode<T>*>(node))

#define BVH_IMPL_3D(T, S, CALLBACK)                                                                               \
    BVH_EXPORT struct bvh##S* bvh##S##_build(struct bvh_thread_pool*, const struct bvh_bbox##S* bboxes,            \
            const struct bvh_vec##S* centers, size_t prim_count, const struct bvh_build_config* config) {          \
        return reinterpret_cast<bvh##S*>(build_handle<T>(nullptr, reinterpret_cast<const T*>(bboxes),              \
            reinterpret_cast<const T*>(centers), prim_count, config, false));                                      \
    }                                                                                                              \
    BVH_EXPORT struct bvh##S* bvh##S##_build_triangles(const T* vertices, size_t prim_count,                       \
            const struct bvh_build_config* config, unsigned flags) {                                               \
        return reinterpret_cast<bvh##S*>(build_handle<T>(vertices, nullptr, nullptr, prim_count, config,           \
            (flags & BVH_DEVICE_POINTERS) != 0));                                                                  \
    }                                                                                                              \
    BVH_EXPORT void bvh##S##_destroy(struct bvh##S* bvh) { destroy_handle(H(T, bvh)); }                            \
    BVH_EXPORT void bvh##S##_save(const struct bvh##S* bvh, FILE* file) { save_mirror(*HC(T, bvh), file); }        \
    BVH_EXPORT struct bvh##S* bvh##S##_load(FILE* file) { return reinterpret_cast<bvh##S*>(load_mirror<T>(file)); } \
    BVH_EXPORT struct bvh_node##S* bvh##S##_get_node(struct bvh##S* bvh, size_t node_id) {                         \
        auto h = H(T, bvh);                                                                                        \
        if (download_mirror(*h) || node_id >= h->nodes.size()) return nullptr;                                     \
        if (!h->maybe_edited && h->device_valid) h->synced_hash = mirror_hash(*h);                                 \
        h->maybe_edited = true;                                                                                    \
        return reinterpret_cast<bvh_node##S*>(&h->nodes[node_id]);                                                 \
    }                                                                                                              \
    BVH_EXPORT size_t bvh##S##_get_prim_id(const struct bvh##S* bvh, size_t i) {                                   \
        auto h = HC(T, bvh);                                                                                       \
        if (download_mirror(*h) || i >= h->prim_ids.size()) return BVH_INVALID_PRIM_ID;                            \
        return h->prim_ids[i];                                                                                     \
    }                                                                                                              \
    BVH_EXPORT size_t bvh##S##_get_prim_count(const struct bvh##S* bvh) {                                          \
        auto h = HC(T, bvh);                                                                                       \
        return h->host_valid ? h->prim_ids.size() : h->dev.prim_count;                                             \
    }                                                                                                              \
    BVH_EXPORT size_t bvh##S##_get_node_count(const struct bvh##S* bvh) {                                          \
        auto h = HC(T, bvh);                                                                                       \
        return download_mirror(*h) ? 0 : h->nodes.size();                                                          \
    }                                                                                                              \
    BVH_EXPORT bool bvh_node##S##_is_leaf(const struct bvh_node##S* node) { return index_count(NC(T, node)->index) != 0; } \
    BVH_EXPORT size_t bvh_node##S##_get_prim_count(const struct bvh_node##S* node) { return index_count(NC(T, node)->index); } \
    BVH_EXPORT void bvh_node##S##_set_prim_count(struct bvh_node##S* node, size_t count) {                         \
        using U = Real<T>::UInt;                                                                                   \
        N(T, node)->index = make_index<U>(index_first(N(T, node)->index), (uint32_t)(count & kMaxLeafPrims));      \
    }                                                                                                              \
    BVH_EXPORT size_t bvh_node##S##_get_first_id(const struct bvh_node##S* node) { return (size_t)index_first(NC(T, node)->index); } \
    BVH_EXPORT void bvh_node##S##_set_first_id(struct bvh_node##S* node, size_t first_id) {                        \
        using U = Real<T>::UInt;                                                                                   \
        N(T, node)->index = make_index<U>((U)first_id, index_count(N(T, node)->index));                            \
    }                                                                                                              \
    BVH_EXPORT struct bvh_bbox##S bvh_node##S##_get_bbox(const struct bvh_node##S* node) {                         \
        const T* b = NC(T, node)->bounds;                                                                          \
        return bvh_bbox##S { { b[0], b[2], b[4] }, { b[1], b[3], b[5] } };                                         \
    }                                                                                                              \
    BVH_EXPORT void bvh_node##S##_set_bbox(struct bvh_node##S* node, const struct bvh_bbox##S* bbox) {             \
        T* b = N(T, node)->bounds;                                                                                 \
        b[0] = bbox->min.x; b[1] = bbox->max.x; b[2] = bbox->min.y; b[3] = bbox->max.y; b[4] = bbox->min.z; b[5] = bbox->max.z; \
    }                                                                                                              \
    BVH_EXPORT void bvh##S##_append_node(struct bvh##S* bvh) {                                                     \
        auto h = H(T, bvh);                                                                                        \
        if (download_mirror(*h)) return;                                                                           \
        h->nodes.emplace_back(); h->maybe_edited = true; h->synced_hash = 0;                                       \
    }                                                                                                              \
    BVH_EXPORT void bvh##S##_remove_last_node(struct bvh##S* bvh) {                                                \
        auto h = H(T, bvh);                                                                                        \
        if (download_mirror(*h) || h->nodes.empty()) return;                                                       \
        h->nodes.pop_back(); h->maybe_edited = true; h->synced_hash = 0;                                           \
    }                                                                                                              \
    BVH_EXPORT void bvh##S##_refit(struct bvh##S* bvh) {                                                           \
        auto h = H(T, bvh);                                                                                        \
        if (download_mirror(*h)) return;                                                                           \
        refit_mirror(*h); h->maybe_edited = true; h->synced_hash = 0;                                              \
    }                                                                                                              \
    BVH_EXPORT void bvh##S##_optimize(struct bvh_thread_pool* pool, struct bvh##S* bvh) {                          \
        auto h = H(T, bvh);                                                                                        \
        if (!h || download_mirror(*h)) return;                                                                     \
        if (optimize_nodes<T, 3>(h->nodes, 0.05, 3, pool_threads(pool))) { h->maybe_edited = true; h->synced_hash = 0; } \
    }                                                                                                              \
    BVH_EXPORT void bvh##S##_intersect_ray_any(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        auto h = HC(T, bvh); if (!download_mirror(*h)) intersect_mirror<T, true, false>(*h, reinterpret_cast<const T*>(ray), cb); } \
    BVH_EXPORT void bvh##S##_intersect_ray_any_robust(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        auto h = HC(T, bvh); if (!download_mirror(*h)) intersect_mirror<T, true, true>(*h, reinterpret_cast<const T*>(ray), cb); } \
    BVH_EXPORT void bvh##S##_intersect_ray(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        auto h = HC(T, bvh); if (!download_mirror(*h)) intersect_mirror<T, false, false>(*h, reinterpret_cast<const T*>(ray), cb); } \
    BVH_EXPORT void bvh##S##_intersect_ray_robust(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        auto h = HC(T, bvh); if (!download_mirror(*h)) intersect_mirror<T, false, true>(*h, reinterpret_cast<const T*>(ray), cb); } \
    BVH_EXPORT int bvh##S##_set_triangles(struct bvh##S* bvh, const T* vertices, size_t prim_count, unsigned flags) { \
        auto h = H(T, bvh);                                                                                        \
        if (!h) { set_error("null handle"); return -1; }                                                           \
        BVH_ON_DEVICE(h->device);                                                                    \
        if (ensure_device(*h)) return -1;                                                                          \
        if (prim_count != h->dev.prim_count) { set_error("set_triangles: prim_count mismatch"); return -1; }       \
        DeviceInput<T> dv(h->stream);                                                                              \
        if (dv.set(vertices, 9 * prim_count, (flags & BVH_DEVICE_POINTERS) != 0)) return -1;                       \
        if (attach_triangles<T>(h->dev, dv.ptr, h->stream)) return -1;                                             \
        BVH_CUDA_TRY(cudaStreamSynchronize(h->stream));                                                            \
        return 0;                                                                                                  \
    }                                                                                                              \
    BVH_EXPORT int bvh##S##_refit_triangles(struct bvh##S* bvh, const T* vertices, size_t prim_count, unsigned flags) { \
        auto h = H(T, bvh);                                                                                        \
        if (!h) { set_error("null handle"); return -1; }                                                           \
        BVH_ON_DEVICE(h->device);                                                                    \
        if (ensure_device(*h)) return -1;                                                                          \
        if (prim_count != h->dev.prim_count) { set_error("refit_triangles: prim_count mismatch"); return -1; }     \
        DeviceInput<T> dv(h->stream);                                                                              \
        if (dv.set(vertices, 9 * prim_count, (flags & BVH_DEVICE_POINTERS) != 0)) return -1;                       \
        if (refit_triangles<T>(h->dev, dv.ptr, h->stream)) return -1;                                              \
        h->host_valid = false;                   /* the mirror (if any) is stale: re-download on demand */        \
        h->nodes.clear(); h->prim_ids.clear();                                                                     \
        BVH_CUDA_TRY(cudaStreamSynchronize(h->stream));                                                            \
        return 0;                                                                                                  \
    }                                                                                                              \
    BVH_EXPORT int bvh##S##_intersect_rays(struct bvh##S* bvh, const struct bvh_ray##S* rays, size_t ray_count,    \
            struct bvh_hit##S* hits, unsigned flags) {                                                             \
        return intersect_batch<T>(H(T, bvh), rays, ray_count, hits, nullptr, flags);                               \
    }                                                                                                              \
    BVH_EXPORT int bvh##S##_intersect_rays_gather(struct bvh##S* bvh, const struct bvh_ray##S* rays, size_t ray_count, \
            struct bvh_hit##S* hits, void* const* gathered_hits, int world_size, size_t shard_offset,              \
            void* multicast_hits, unsigned flags) {                                                                \
        auto h = H(T, bvh);                                                                                        \
        if (!h) { set_error("null handle"); return -1; }                                                           \
        if (!gathered_hits || world_size < 1 || world_size > 8) { set_error("gather: need 1..8 gathered arrays"); return -1; } \
        std::lock_guard<std::mutex> lock(h->batch_mutex);                                                          \
        BVH_ON_DEVICE(h->device);                                                                    \
        if (ensure_device(*h)) return -1;                                                                          \
        GatherTargets g;                                                                                           \
        for (int r = 0; r < 8; ++r) g.peer[r] = r < world_size ? gathered_hits[r] : nullptr;                      \
        g.count = world_size; g.multicast = multicast_hits; g.offset = shard_offset;                               \
        return trace_rays<T>(h->dev, reinterpret_cast<const DevRay<T>*>(rays), reinterpret_cast<DevHit<T>*>(hits), \
                             ray_count, translate_flags(flags), nullptr, h->stream, &g);                           \
    }                                                                                                              \
    BVH_EXPORT int bvh##S##_intersect_rays_stats(struct bvh##S* bvh, const struct bvh_ray##S* rays, size_t ray_count, \
            struct bvh_hit##S* hits, struct bvh_ray_stats* stats, unsigned flags) {                                \
        if (!stats) { set_error("stats pointer is null"); return -1; }                                             \
        return intersect_batch<T>(H(T, bvh), rays, ray_count, hits, stats, flags);                                 \
    }                                                                                                              \
    BVH_EXPORT int bvh##S##_sync(struct bvh##S* bvh) {                                                             \
        auto h = H(T, bvh);                                                                                        \
        if (!h) { set_error("null handle"); return -1; }                                                           \
        BVH_ON_DEVICE(h->device);                                                                    \
        return check_trace_status(h->dev, h->stream);                                                              \
    }                                                                                                              \
    BVH_EXPORT size_t bvh##S##_get_depth(struct bvh##S* bvh) {                                                     \
        auto h = H(T, bvh);                                                                                        \
        if (!h || ensure_device(*h)) return 0;                                                                     \
        return h->dev.depth;                                                                                       \
    }                                                                                                              \
    BVH_EXPORT const size_t* bvh##S##_get_prim_ids(struct bvh##S* bvh) {                                           \
        auto h = H(T, bvh);                                                                                        \
        if (!h || download_mirror(*h)) return nullptr;                                                             \
        return h->prim_ids.data();                                                                                 \
    }                                                                                                              \
    BVH_EXPORT size_t bvh##S##_get_property(struct bvh##S* bvh, int property) {                                    \
        auto h = H(T, bvh);                                                                                        \
        if (!h || ensure_device(*h)) return (size_t)-1;                                                            \
        switch (property) {                                                                                        \
            case BVH_PROP_DEPTH: return h->dev.depth;                                                              \
            case BVH_PROP_NODE_SLOTS: return h->dev.node_slots;                                                    \
            case BVH_PROP_MORTON_BITS: return (size_t)h->dev.morton_bits;                                          \
            case BVH_PROP_QUALITY: return (size_t)h->dev.quality;                                                  \
            case BVH_PROP_TREELETS: return h->dev.treelets;                                                        \
            case BVH_PROP_WIDE_NODES: return h->dev.wide ? h->dev.wide_count : 0;                                  \
            case BVH_PROP_LAST_KERNEL: return (size_t)h->dev.last_kernel;                                          \
            case BVH_PROP_STREAM: return (size_t)reinterpret_cast<uintptr_t>(h->stream);                           \
            default: return (size_t)-1;                                                                            \
        }                                                                                                          \
    }                                                                                                              \
    BVH_EXPORT int bvh##S##_get_device_view(struct bvh##S* bvh, struct bvh_device_view##S* view) {                 \
        auto h = H(T, bvh);                                                                                        \
        if (!h) { set_error("get_device_view: null handle"); return -1; }                                          \
        if (!view) { set_error("get_device_view: null view"); return -1; }                                         \
        std::lock_guard<std::mutex> lock(h->batch_mutex);                                                          \
        BVH_ON_DEVICE(h->device);                                                                                  \
        if (ensure_device(*h)) return -1;                                                                          \
        if (!h->dev.nodes || h->dev.node_slots < 2) { set_error("get_device_view: handle holds no BVH"); return -1; } \
        view->device = h->device;                                                                                  \
        view->stream = h->stream;                                                                                  \
        view->nodes = h->dev.nodes;                                                                                \
        view->prim_ids = h->dev.prim_ids;                                                                          \
        view->tris = h->dev.tris;                                                                                  \
        view->node_count = h->dev.node_slots - 1;                                                                  \
        view->prim_count = h->dev.prim_count;                                                                      \
        view->depth = h->dev.depth;                                                                                \
        return 0;                                                                                                  \
    }

BVH_IMPL_3D(float, 3f, bvh_intersect_callbackf)
BVH_IMPL_3D(double, 3d, bvh_intersect_callbackd)

#define H2(T, bvh) (reinterpret_cast<Handle2<T>*>(bvh))
#define HC2(T, bvh) (reinterpret_cast<const Handle2<T>*>(bvh))
#define N2(T, node) (reinterpret_cast<HostNode2<T>*>(node))
#define NC2(T, node) (reinterpret_cast<const HostNode2<T>*>(node))

#define BVH_IMPL_2D(T, S, CALLBACK)                                                                                \
    BVH_EXPORT struct bvh##S* bvh##S##_build(struct bvh_thread_pool*, const struct bvh_bbox##S* bboxes,            \
            const struct bvh_vec##S* centers, size_t prim_count, const struct bvh_build_config* config) {          \
        return reinterpret_cast<bvh##S*>(build_handle2<T>(reinterpret_cast<const T*>(bboxes),                      \
            reinterpret_cast<const T*>(centers), prim_count, config));                                             \
    }                                                                                                              \
    BVH_EXPORT void bvh##S##_destroy(struct bvh##S* bvh) { delete H2(T, bvh); }                                    \
    BVH_EXPORT void bvh##S##_save(const struct bvh##S* bvh, FILE* file) { save_nodes2(*HC2(T, bvh), file); }       \
    BVH_EXPORT struct bvh##S* bvh##S##_load(FILE* file) { return reinterpret_cast<bvh##S*>(load_nodes2<T>(file)); } \
    BVH_EXPORT struct bvh_node##S* bvh##S##_get_node(struct bvh##S* bvh, size_t node_id) {                         \
        auto h = H2(T, bvh);                                                                                       \
        return node_id < h->nodes.size() ? reinterpret_cast<bvh_node##S*>(&h->nodes[node_id]) : nullptr;           \
    }                                                                                                              \
    BVH_EXPORT size_t bvh##S##_get_prim_id(const struct bvh##S* bvh, size_t i) {                                   \
        auto h = HC2(T, bvh);                                                                                      \
        return i < h->prim_ids.size() ? h->prim_ids[i] : BVH_INVALID_PRIM_ID;                                      \
    }                                                                                                              \
    BVH_EXPORT size_t bvh##S##_get_prim_count(const struct bvh##S* bvh) { return HC2(T, bvh)->prim_ids.size(); }   \
    BVH_EXPORT size_t bvh##S##_get_node_count(const struct bvh##S* bvh) { return HC2(T, bvh)->nodes.size(); }      \
    BVH_EXPORT bool bvh_node##S##_is_leaf(const struct bvh_node##S* node) { return index_count(NC2(T, node)->index) != 0; } \
    BVH_EXPORT size_t bvh_node##S##_get_prim_count(const struct bvh_node##S* node) { return index_count(NC2(T, node)->index); } \
    BVH_EXPORT void bvh_node##S##_set_prim_count(struct bvh_node##S* node, size_t count) {                         \
        using U = Real<T>::UInt;                                                                                   \
        N2(T, node)->index = make_index<U>(index_first(N2(T, node)->index), (uint32_t)(count & kMaxLeafPrims));    \
    }                                                                                                              \
    BVH_EXPORT size_t bvh_node##S##_get_first_id(const struct bvh_node##S* node) { return (size_t)index_first(NC2(T, node)->index); } \
    BVH_EXPORT void bvh_node##S##_set_first_id(struct bvh_node##S* node, size_t first_id) {                        \
        using U = Real<T>::UInt;                                                                                   \
        N2(T, node)->index = make_index<U>((U)first_id, index_count(N2(T, node)->index));                          \
    }                                                                                                              \
    BVH_EXPORT struct bvh_bbox##S bvh_node##S##_get_bbox(const struct bvh_node##S* node) {                         \
        const T* b = NC2(T, node)->bounds;                                                                         \
        return bvh_bbox##S { { b[0], b[2] }, { b[1], b[3] } };                                                     \
    }                                                                                                              \
    BVH_EXPORT void bvh_node##S##_set_bbox(struct bvh_node##S* node, const struct bvh_bbox##S* bbox) {             \
        T* b = N2(T, node)->bounds;                                                                                \
        b[0] = bbox->min.x; b[1] = bbox->max.x; b[2] = bbox->min.y; b[3] = bbox->max.y;                            \
    }                                                                                                              \
    BVH_EXPORT void bvh##S##_append_node(struct bvh##S* bvh) { H2(T, bvh)->nodes.emplace_back(); }                 \
    BVH_EXPORT void bvh##S##_remove_last_node(struct bvh##S* bvh) { if (!H2(T, bvh)->nodes.empty()) H2(T, bvh)->nodes.pop_back(); } \
    BVH_EXPORT void bvh##S##_refit(struct bvh##S* bvh) { refit_nodes<T, 2>(H2(T, bvh)->nodes); }                   \
    BVH_EXPORT void bvh##S##_optimize(struct bvh_thread_pool* pool, struct bvh##S* bvh) {                          \
        if (bvh) optimize_nodes<T, 2>(H2(T, bvh)->nodes, 0.05, 3, pool_threads(pool));                             \
    }                                                                                                              \
    BVH_EXPORT void bvh##S##_intersect_ray_any(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        intersect_nodes<T, true, false, 2>(HC2(T, bvh)->nodes, reinterpret_cast<const T*>(ray), cb); }            \
    BVH_EXPORT void bvh##S##_intersect_ray_any_robust(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        intersect_nodes<T, true, true, 2>(HC2(T, bvh)->nodes, reinterpret_cast<const T*>(ray), cb); }             \
    BVH_EXPORT void bvh##S##_intersect_ray(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        intersect_nodes<T, false, false, 2>(HC2(T, bvh)->nodes, reinterpret_cast<const T*>(ray), cb); }           \
    BVH_EXPORT void bvh##S##_intersect_ray_robust(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        intersect_nodes<T, false, true, 2>(HC2(T, bvh)->nodes, reinterpret_cast<const T*>(ray), cb); }

BVH_IMPL_2D(float, 2f, bvh_intersect_callbackf)
BVH_IMPL_2D(double, 2d, bvh_intersect_callbackd)

} // extern "C"
