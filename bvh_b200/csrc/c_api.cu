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
#include <cctype>
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

// The switches of bvh_set_option.  Each setter clamps its value and stores it, or returns false for a value it rejects.
// Defaults are the initialisers in Tunables (engine.h).
struct OptionSetter {
    const char* name;
    bool (*set)(Tunables&, long);
};
static const OptionSetter kOptions[] = {
    { "morton_bits", [] (Tunables& t, long v) { t.morton_bits = (int)v; return true; } },
    { "sah_treelets", [] (Tunables& t, long v) { t.sah_treelets = (int)v; return true; } },
    { "hierarchy", [] (Tunables& t, long v) { t.hierarchy = (int)v; return true; } },
    { "e2e_chunks", [] (Tunables& t, long v) { t.e2e_chunks = (int)v; return true; } },
    { "variant", [] (Tunables& t, long v) { if (v != 0 && v != 1) return false; t.variant = (int)v; return true; } },
    { "use_wide", [] (Tunables& t, long v) { t.use_wide = (int)v; return true; } },
    { "chunk_rays", [] (Tunables& t, long v) { t.chunk_rays = v < 32 ? 32u : (uint32_t)v; return true; } },
    { "stack_round", [] (Tunables& t, long v) { t.stack_round = v < 1 ? 1 : (int)v; return true; } },
    { "smem_carveout", [] (Tunables& t, long v) { t.smem_carveout = (int)v; return true; } },
    { "refill_min", [] (Tunables& t, long v) { t.refill_min = v < 1 ? 0u : v > 32 ? 32u : (uint32_t)v; return true; } },   // 0: auto
    { "inner_budget", [] (Tunables& t, long v) { t.inner_budget = v <= 0 ? 0xFFFFFFFFu : (uint32_t)v; return true; } },
    { "wide_budget", [] (Tunables& t, long v) { t.wide_budget = v <= 0 ? 0xFFFFFFFFu : (uint32_t)v; return true; } },
    { "watchdog", [] (Tunables& t, long v) { t.watchdog = (uint32_t)v; return true; } },
    { "gather_staging", [] (Tunables& t, long v) { t.gather_staging = (int)v; return true; } },
    { "sort_onesweep", [] (Tunables& t, long v) { t.sort_onesweep = (int)v; return true; } },
    { "treelet_blocks", [] (Tunables& t, long v) { t.treelet_blocks = (int)v; return true; } },
};

// Initial values: BVH_B200_<NAME> through the same setters (a rejected value keeps the default; unset keeps the default,
// which for inner_budget is auto).  hierarchy is spelt global / thread64 / thread256 there, anything else is 128.
Tunables& tunables() {
    static Tunables t;
    static std::once_flag once;
    std::call_once(once, [] {
        for (const OptionSetter& o : kOptions) {
            std::string var = "BVH_B200_";
            for (const char* c = o.name; *c; ++c) var += (char)toupper((unsigned char)*c);
            const char* e = getenv(var.c_str());
            if (!e) continue;
            const std::string v = e;
            const long value = std::string(o.name) != "hierarchy" ? atol(e)
                             : v == "global" ? 0 : v == "thread64" ? 64 : v == "thread256" ? 256 : 128;
            o.set(t, value);
        }
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

// ---- host trees -------------------------------------------------------------------------------
// The reference's Node<T, kDim> (bounds as min0 max0 min1 max1 ..., then the packed index; node.h:31-37) and the
// node and primitive-id vectors of its Bvh (bvh.h:17-23).  A 2-D handle is a HostTree; a 3-D handle holds one as
// its mirror.
template <typename T, int kDim> struct HostNode { T bounds[2 * kDim]; typename Real<T>::UInt index; };
static_assert(sizeof(HostNode<float, 2>) == 20 && sizeof(HostNode<double, 2>) == 40, "reference Node<T,2> layout");
static_assert(sizeof(HostNode<float, 3>) == 28 && sizeof(HostNode<double, 3>) == 56, "reference Node<T,3> layout");

template <typename T, int kDim> struct HostTree {
    std::vector<HostNode<T, kDim>> nodes;
    std::vector<size_t> prim_ids;
};

template <typename T> struct Handle {
    using U = typename Real<T>::UInt;
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    DeviceBvh<T> dev;
    bool device_valid = false;

    HostTree<T, 3> mirror;
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
    return hash_bytes(h.mirror.prim_ids.data(), h.mirror.prim_ids.size() * sizeof(size_t), h.mirror.prim_ids.size());
}

template <typename T> uint64_t mirror_hash(const Handle<T>& h) {
    uint64_t a = hash_bytes(h.mirror.nodes.data(), h.mirror.nodes.size() * sizeof(HostNode<T, 3>), h.mirror.nodes.size());
    return hash_bytes(h.mirror.prim_ids.data(), h.mirror.prim_ids.size() * sizeof(size_t), a);
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
    if (device_alloc(&d_nodes, node_count * sizeof(HostNode<T, 3>), h.stream)) return -1;
    if (device_alloc(&d_ids, prim_count * sizeof(unsigned long long), h.stream)) { device_free(d_nodes, h.stream); return -1; }
    int rc = export_reference_arrays(h.dev, d_nodes, static_cast<unsigned long long*>(d_ids), h.stream);
    if (!rc) {
        try { h.mirror.nodes.resize(node_count); h.mirror.prim_ids.resize(prim_count); }
        catch (const std::exception&) { set_error("download: out of host memory"); rc = -1; }
    }
    cudaError_t err = cudaSuccess;
    if (!rc) err = cudaMemcpyAsync(h.mirror.nodes.data(), d_nodes, node_count * sizeof(HostNode<T, 3>), cudaMemcpyDeviceToHost, h.stream);
    if (!rc && err == cudaSuccess) err = cudaMemcpyAsync(h.mirror.prim_ids.data(), d_ids, prim_count * sizeof(size_t), cudaMemcpyDeviceToHost, h.stream);
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
    const std::vector<HostNode<T, 3>>& nodes = h.mirror.nodes;
    const size_t node_count = nodes.size();
    if (node_count == 0) { set_error("upload: empty BVH"); return -1; }
    std::vector<DevNode<T>> dev_nodes(node_count + 1);
    std::memset(dev_nodes.data(), 0, sizeof(DevNode<T>));
    for (size_t i = 0; i < node_count; ++i) {
        std::memcpy(dev_nodes[i + 1].bounds, nodes[i].bounds, sizeof(nodes[i].bounds));
        dev_nodes[i + 1].index = nodes[i].index;
        dev_nodes[i + 1].pad = 0;
    }
    std::vector<uint32_t> ids(h.mirror.prim_ids.size());
    for (size_t i = 0; i < ids.size(); ++i) {
        if (h.mirror.prim_ids[i] >= ids.size()) { set_error("upload: primitive id out of range"); return -1; }
        ids[i] = (uint32_t)h.mirror.prim_ids[i];
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
            if (const uint32_t leaf_count = index_count(nodes[i].index)) {
                // the kernels index tris[first .. first + count) and prim_ids[slot] without further checks
                if ((size_t)index_first(nodes[i].index) + leaf_count > ids.size()) { set_error("upload: leaf range exceeds the primitive count"); return -1; }
                continue;
            }
            const size_t first = (size_t)index_first(nodes[i].index);
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

// A legacy call changed the mirror: the next batched call uploads it.
template <typename T> void mark_mirror_edited(Handle<T>& h) { h.maybe_edited = true; h.synced_hash = 0; }
// A batched call changed the device tree: the mirror is stale and is downloaded again when a legacy call needs it.
template <typename T> void drop_mirror(Handle<T>& h) { h.host_valid = false; h.mirror.nodes.clear(); h.mirror.prim_ids.clear(); }

// The prologue of every entry point that may upload the mirror or enqueue work on the handle's stream: such calls
// on one handle are serialised (Handle::batch_mutex), run on the handle's device and see a current device tree.
// `check` returns the error of a call it rejects, before the mirror is uploaded: a rejected call changes nothing.
// A null handle sets `null_error`, where one is given.
template <typename T, typename Check, typename Body>
int on_device_tree(Handle<T>* h, const char* null_error, Check check, Body body) {
    if (!h) { if (null_error) set_error(null_error); return -1; }
    std::lock_guard<std::mutex> lock(h->batch_mutex);
    if (const char* error = check()) { set_error(error); return -1; }
    BVH_ON_DEVICE(h->device);
    if (ensure_device(*h)) return -1;
    return body();
}
template <typename T, typename Body> int on_device_tree(Handle<T>* h, const char* null_error, Body body) {
    return on_device_tree(h, null_error, [] () -> const char* { return nullptr; }, body);
}

// ---- reference semantics on the mirror ---------------------------------------------------------
// Bvh::refit with no leaf function (reference bvh.h:184-218; c_api/bvh_impl.h:218-221).
template <typename T, int kDim> void refit_nodes(std::vector<HostNode<T, kDim>>& nodes) {
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

// Bvh::intersect for one ray with a host callback (reference bvh.h:124-182, c_api/bvh_impl.h:235-250).
// `ray` = org[kDim] dir[kDim] tmin tmax.
template <bool kAny, bool kRobust, typename T, int kDim, typename Callback>
void intersect_nodes(const std::vector<HostNode<T, kDim>>& nodes, const T* ray, const Callback* cb) {
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

// bvhNN_intersect_rays / _stats after the prologue: the handle's device tree is current.
template <typename T, typename RayPod, typename HitPod>
int trace_batch(Handle<T>* h, const RayPod* rays, size_t n, HitPod* hits, bvh_ray_stats* stats, unsigned flags) {
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

template <typename T, typename RayPod, typename HitPod>
int intersect_batch(Handle<T>* h, const RayPod* rays, size_t n, HitPod* hits, bvh_ray_stats* stats, unsigned flags) {
    static_assert(sizeof(RayPod) == sizeof(DevRay<T>) && sizeof(HitPod) == sizeof(DevHit<T>), "POD layouts");
    if (h && n == 0) return 0;
    return on_device_tree(h, "null handle", [&] { return trace_batch(h, rays, n, hits, stats, flags); });
}
template <typename T, typename RayPod, typename HitPod>
int intersect_batch_stats(Handle<T>* h, const RayPod* rays, size_t n, HitPod* hits, bvh_ray_stats* stats, unsigned flags) {
    if (!stats) { set_error("stats pointer is null"); return -1; }
    return intersect_batch(h, rays, n, hits, stats, flags);
}
template <typename T>
int intersect_gather(Handle<T>* h, const DevRay<T>* rays, size_t n, DevHit<T>* hits, void* const* gathered_hits, int world_size,
                     size_t shard_offset, void* multicast_hits, unsigned flags) {
    return on_device_tree(h, "null handle", [&] {
        return !gathered_hits || world_size < 1 || world_size > 8 ? "gather: need 1..8 gathered arrays" : nullptr;
    }, [&] {
        GatherTargets g;
        for (int r = 0; r < 8; ++r) g.peer[r] = r < world_size ? gathered_hits[r] : nullptr;
        g.count = world_size; g.multicast = multicast_hits; g.offset = shard_offset;
        return trace_rays<T>(h->dev, rays, hits, n, translate_flags(flags), nullptr, h->stream, &g);
    });
}

// ---- the other 3-D entry points that build or use the device tree ---------------------------------------------
template <typename T, typename BBox, typename Vec>
Handle<T>* build_boxes(const BBox* bboxes, const Vec* centers, size_t n, const bvh_build_config* config, unsigned flags) {
    static_assert(sizeof(BBox) == 6 * sizeof(T) && sizeof(Vec) == 3 * sizeof(T), "box / centre layout");
    if (!bboxes) { set_error("build_boxes: null boxes"); return nullptr; }
    if (!centers) { set_error("build_boxes: null centres"); return nullptr; }
    return build_handle<T>(nullptr, reinterpret_cast<const T*>(bboxes), reinterpret_cast<const T*>(centers), n, config,
                           (flags & BVH_DEVICE_POINTERS) != 0);
}
template <typename T> int set_handle_triangles(Handle<T>* h, const T* vertices, size_t n, unsigned flags) {
    return on_device_tree(h, "null handle", [&] {
        if (n != h->dev.prim_count) { set_error("set_triangles: prim_count mismatch"); return -1; }
        DeviceInput<T> dv(h->stream);
        if (dv.set(vertices, 9 * n, (flags & BVH_DEVICE_POINTERS) != 0)) return -1;
        if (attach_triangles<T>(h->dev, dv.ptr, h->stream)) return -1;
        BVH_CUDA_TRY(cudaStreamSynchronize(h->stream));
        return 0;
    });
}
template <typename T> int refit_handle_triangles(Handle<T>* h, const T* vertices, size_t n, unsigned flags) {
    return on_device_tree(h, "null handle", [&] {
        if (n != h->dev.prim_count) { set_error("refit_triangles: prim_count mismatch"); return -1; }
        DeviceInput<T> dv(h->stream);
        if (dv.set(vertices, 9 * n, (flags & BVH_DEVICE_POINTERS) != 0)) return -1;
        if (refit_triangles<T>(h->dev, dv.ptr, h->stream)) return -1;
        drop_mirror(*h);
        BVH_CUDA_TRY(cudaStreamSynchronize(h->stream));
        return 0;
    });
}
template <typename T, typename BBox> int refit_handle_boxes(Handle<T>* h, const BBox* bboxes, size_t n, unsigned flags) {
    static_assert(sizeof(BBox) == 6 * sizeof(T), "bbox layout: min3, max3");
    const bool device_ptrs = (flags & BVH_DEVICE_POINTERS) != 0;
    return on_device_tree(h, "refit_boxes: null handle", [&] () -> const char* {
        if (!bboxes) return "refit_boxes: null boxes";
        if (h->host_valid ? h->mirror.nodes.empty() : !h->device_valid) return "refit_boxes: handle holds no BVH";
        if (n != (h->host_valid ? h->mirror.prim_ids.size() : (size_t)h->dev.prim_count)) return "refit_boxes: prim_count mismatch";
        return nullptr;
    }, [&] {
        DeviceInput<T> db(h->stream);
        if (db.set(reinterpret_cast<const T*>(bboxes), 6 * n, device_ptrs)) return -1;
        if (refit_boxes<T>(h->dev, db.ptr, h->stream)) return -1;
        drop_mirror(*h);
        if (!device_ptrs) BVH_CUDA_TRY(cudaStreamSynchronize(h->stream));
        return 0;
    });
}
template <typename T> int sync_handle(Handle<T>* h) {
    if (!h) { set_error("null handle"); return -1; }
    BVH_ON_DEVICE(h->device);
    return check_trace_status(h->dev, h->stream);
}
template <typename T> size_t get_property(Handle<T>* h, int property) {
    size_t value = (size_t)-1;
    on_device_tree(h, nullptr, [&] {
        switch (property) {
            case BVH_PROP_DEPTH: value = h->dev.depth; break;
            case BVH_PROP_NODE_SLOTS: value = h->dev.node_slots; break;
            case BVH_PROP_MORTON_BITS: value = (size_t)h->dev.morton_bits; break;
            case BVH_PROP_QUALITY: value = (size_t)h->dev.quality; break;
            case BVH_PROP_TREELETS: value = h->dev.treelets; break;
            case BVH_PROP_WIDE_NODES: value = h->dev.wide ? h->dev.wide_count : 0; break;
            case BVH_PROP_LAST_KERNEL: value = (size_t)h->dev.last_kernel; break;
            case BVH_PROP_STREAM: value = (size_t)reinterpret_cast<uintptr_t>(h->stream); break;
        }
        return 0;
    });
    return value;
}
template <typename T> size_t get_depth(Handle<T>* h) {
    size_t depth = 0;
    on_device_tree(h, nullptr, [&] { depth = h->dev.depth; return 0; });
    return depth;
}
template <typename T, typename View> int get_device_view(Handle<T>* h, View* view) {
    return on_device_tree(h, "get_device_view: null handle", [&] { return view ? nullptr : "get_device_view: null view"; }, [&] {
        if (!h->dev.nodes || h->dev.node_slots < 2) { set_error("get_device_view: handle holds no BVH"); return -1; }
        view->device = h->device;
        view->stream = h->stream;
        view->nodes = h->dev.nodes;
        view->prim_ids = h->dev.prim_ids;
        view->tris = h->dev.tris;
        view->node_count = h->dev.node_slots - 1;
        view->prim_count = h->dev.prim_count;
        view->depth = h->dev.depth;
        return 0;
    });
}

// ---- save / load (reference bvh.h:220-242, node.h:90-102, stream.h) ---------------------------------------------
// [node_count][prim_count] then per node its 2 * kDim bounds and index, then the primitive ids, all as T / UInt.
template <typename T, int kDim> void write_tree(const HostTree<T, kDim>& t, FILE* file) {
    using U = typename Real<T>::UInt;
    U v = (U)t.nodes.size(); fwrite(&v, sizeof v, 1, file);
    v = (U)t.prim_ids.size(); fwrite(&v, sizeof v, 1, file);
    for (const auto& n : t.nodes) { fwrite(n.bounds, sizeof(T), 2 * kDim, file); fwrite(&n.index, sizeof(U), 1, file); }
    for (size_t id : t.prim_ids) { v = (U)id; fwrite(&v, sizeof v, 1, file); }
}

template <typename T, int kDim> int read_tree(HostTree<T, kDim>& t, FILE* file) {
    using U = typename Real<T>::UInt;
    constexpr size_t kBounds = 2 * kDim;
    U node_count = 0, prim_count = 0;                       // short reads give defaults (stream.h:13-18)
    if (fread(&node_count, sizeof(U), 1, file) != 1) node_count = 0;
    if (fread(&prim_count, sizeof(U), 1, file) != 1) prim_count = 0;
    // A corrupt header must not turn into a multi-gigabyte resize: the counts are bounded by what the file
    // still holds (seekable streams) and allocation failures never cross the C boundary.
    const long here = ftell(file);
    if (here >= 0 && fseek(file, 0, SEEK_END) == 0) {
        const long end = ftell(file);
        fseek(file, here, SEEK_SET);
        const double need = (double)node_count * (kBounds * sizeof(T) + sizeof(U)) + (double)prim_count * sizeof(U);
        if (end >= here && need > (double)(end - here)) { set_error("load: the header announces more nodes / primitives than the file holds"); return -1; }
    }
    try { t.nodes.resize((size_t)node_count); t.prim_ids.resize((size_t)prim_count); }
    catch (const std::exception&) { set_error("load: out of memory for the announced node / primitive counts"); return -1; }
    for (auto& n : t.nodes) {
        std::memset(&n, 0, sizeof n);
        if (fread(n.bounds, sizeof(T), kBounds, file) != kBounds) std::memset(n.bounds, 0, sizeof n.bounds);
        if (fread(&n.index, sizeof(U), 1, file) != 1) n.index = 0;
    }
    for (auto& id : t.prim_ids) { U v = 0; if (fread(&v, sizeof(U), 1, file) != 1) v = 0; id = (size_t)v; }
    return 0;
}

template <typename T> void save_handle(Handle<T>& h, FILE* file) { if (!download_mirror(h)) write_tree(h.mirror, file); }
template <typename T> Handle<T>* load_handle(FILE* file) {
    DeviceGuard guard(g_device);
    if (!guard.ok) return nullptr;
    auto h = new Handle<T>();
    if (init_handle(*h)) { delete h; return nullptr; }
    if (read_tree(h->mirror, file)) { destroy_handle(h); return nullptr; }
    h->host_valid = true;
    return h;
}

// ---- the reference's per-tree calls on the 3-D mirror (downloaded on first use) ---------------------------------
template <typename T> HostNode<T, 3>* get_node(Handle<T>& h, size_t node_id) {
    if (download_mirror(h) || node_id >= h.mirror.nodes.size()) return nullptr;
    if (!h.maybe_edited && h.device_valid) h.synced_hash = mirror_hash(h);
    h.maybe_edited = true;
    return &h.mirror.nodes[node_id];
}
template <typename T> size_t get_prim_id(Handle<T>& h, size_t i) {
    return download_mirror(h) || i >= h.mirror.prim_ids.size() ? BVH_INVALID_PRIM_ID : h.mirror.prim_ids[i];
}
template <typename T> size_t get_prim_count(const Handle<T>& h) { return h.host_valid ? h.mirror.prim_ids.size() : h.dev.prim_count; }
template <typename T> size_t get_node_count(Handle<T>& h) { return download_mirror(h) ? 0 : h.mirror.nodes.size(); }
template <typename T> const size_t* get_prim_ids(Handle<T>* h) { return !h || download_mirror(*h) ? nullptr : h->mirror.prim_ids.data(); }
template <typename T> void append_node(Handle<T>& h) { if (!download_mirror(h)) { h.mirror.nodes.emplace_back(); mark_mirror_edited(h); } }
template <typename T> void remove_last_node(Handle<T>& h) {
    if (!download_mirror(h) && !h.mirror.nodes.empty()) { h.mirror.nodes.pop_back(); mark_mirror_edited(h); }
}
template <typename T> void refit(Handle<T>& h) { if (!download_mirror(h)) { refit_nodes(h.mirror.nodes); mark_mirror_edited(h); } }
template <bool kAny, bool kRobust, typename T, typename Callback> void intersect_ray(Handle<T>& h, const T* ray, const Callback* cb) {
    if (!download_mirror(h)) intersect_nodes<kAny, kRobust>(h.mirror.nodes, ray, cb);
}

// ---- 2-D suffixes (reference c_api/bvh.cpp:7-25 instantiates bvh2f / bvh2d next to the 3-D ones) ----------
// The reference has no 2-D primitive type: leaves are intersected by the caller's callback, one ray per call,
// so there is no batched device traversal to offer here.  What the GPU does is the BUILD: the boxes are lifted
// to z = 0, the LBVH pipeline runs as for 3-D (the z bits of the Morton keys are all zero, so the order is the
// 2-D Z-curve), and the result comes back as a host tree of the reference's Node<T, 2> (4 bounds + index,
// 20 / 40 bytes) on which every other entry point works exactly as the reference's does.
template <typename T>
HostTree<T, 2>* build_tree2(const T* bboxes4, const T* centers2, size_t n, const bvh_build_config* config) {
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
    auto t = new HostTree<T, 2>();
    t->nodes.resize(lifted->mirror.nodes.size());
    for (size_t i = 0; i < t->nodes.size(); ++i) {
        std::memcpy(t->nodes[i].bounds, lifted->mirror.nodes[i].bounds, 4 * sizeof(T));
        t->nodes[i].index = lifted->mirror.nodes[i].index;
    }
    t->prim_ids = lifted->mirror.prim_ids;
    destroy_handle(lifted);
    return t;
}

template <typename T> HostTree<T, 2>* load_tree2(FILE* file) {
    auto t = new HostTree<T, 2>();
    if (read_tree(*t, file)) { delete t; return nullptr; }
    return t;
}
template <typename T> HostNode<T, 2>* get_node(HostTree<T, 2>& t, size_t node_id) { return node_id < t.nodes.size() ? &t.nodes[node_id] : nullptr; }
template <typename T> size_t get_prim_id(const HostTree<T, 2>& t, size_t i) { return i < t.prim_ids.size() ? t.prim_ids[i] : BVH_INVALID_PRIM_ID; }
template <typename T> void remove_last_node(HostTree<T, 2>& t) { if (!t.nodes.empty()) t.nodes.pop_back(); }

// ---- the reference's node accessors (c_api/bvh_impl.h) on Node<T, kDim> ------------------------------------------
template <typename T, int kDim> bool node_is_leaf(const HostNode<T, kDim>* n) { return index_count(n->index) != 0; }
template <typename T, int kDim> size_t node_prim_count(const HostNode<T, kDim>* n) { return index_count(n->index); }
template <typename T, int kDim> void set_node_prim_count(HostNode<T, kDim>* n, size_t count) {
    n->index = make_index(index_first(n->index), (uint32_t)(count & kMaxLeafPrims));
}
template <typename T, int kDim> size_t node_first_id(const HostNode<T, kDim>* n) { return (size_t)index_first(n->index); }
template <typename T, int kDim> void set_node_first_id(HostNode<T, kDim>* n, size_t first_id) {
    n->index = make_index((typename Real<T>::UInt)first_id, index_count(n->index));
}
// bvh_bboxNN is {min[kDim], max[kDim]}; a node interleaves them as min0 max0 min1 max1 ...
template <typename BBox, typename T, int kDim> BBox node_bbox(const HostNode<T, kDim>* n) {
    static_assert(sizeof(BBox) == 2 * kDim * sizeof(T), "bbox layout: min[kDim], max[kDim]");
    T v[2 * kDim];
    for (int k = 0; k < kDim; ++k) { v[k] = n->bounds[2 * k]; v[kDim + k] = n->bounds[2 * k + 1]; }
    BBox b;
    std::memcpy(&b, v, sizeof b);
    return b;
}
template <typename T, int kDim, typename BBox> void set_node_bbox(HostNode<T, kDim>* n, const BBox* bbox) {
    static_assert(sizeof(BBox) == 2 * kDim * sizeof(T), "bbox layout: min[kDim], max[kDim]");
    T v[2 * kDim];
    std::memcpy(v, bbox, sizeof v);
    for (int k = 0; k < kDim; ++k) { n->bounds[2 * k] = v[k]; n->bounds[2 * k + 1] = v[kDim + k]; }
}

// bvhNN_optimize (reference c_api/bvh_impl.h:223-233): with a pool the search runs on the pool's thread count
// (0 = hardware concurrency, thread_pool.h:82-86), without one it is serial (SequentialExecutor).
static size_t optimizer_threads(size_t requested) {
    if (requested != 0) return requested;
    const unsigned hw = std::thread::hardware_concurrency();
    return hw ? hw : 1;
}
template <typename T, int kDim>
bool optimize_nodes(std::vector<HostNode<T, kDim>>& nodes, double ratio, size_t iters, size_t threads) {
    try {
        if (!Reinserter<T, kDim, HostNode<T, kDim>>(nodes, threads).run((T)ratio, iters)) {
            set_error("optimize: the node array is not a well-formed tree");
            return false;
        }
    } catch (const std::exception& e) { set_error(std::string("optimize: ") + e.what()); return false; }
    return true;
}
template <typename T> void optimize(Handle<T>* h, size_t threads) {
    if (h && !download_mirror(*h) && optimize_nodes(h->mirror.nodes, 0.05, 3, threads)) mark_mirror_edited(*h);
}
template <typename T> void optimize(HostTree<T, 2>* t, size_t threads) { if (t) optimize_nodes(t->nodes, 0.05, 3, threads); }

// bvh_optimize_nodes: the Reinserter works on a std::vector; the caller's array is copied in and out (host memory,
// O(node_count)).
template <typename T, int kDim> int optimize_array(void* nodes, size_t node_count, double ratio, size_t iters, size_t threads) {
    HostNode<T, kDim>* first = static_cast<HostNode<T, kDim>*>(nodes);
    std::vector<HostNode<T, kDim>> v(first, first + node_count);
    if (!optimize_nodes(v, ratio, iters, optimizer_threads(threads))) return -1;
    std::copy(v.begin(), v.end(), first);
    return 0;
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
    const std::string n = name;
    for (const OptionSetter& o : kOptions) {
        if (n != o.name) continue;
        if (o.set(tunables(), value)) return 0;
        set_error("set_option: " + n + " does not accept " + std::to_string(value));
        return -1;
    }
    set_error("set_option: unknown option " + n);
    return -1;
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
    try {
        if (dim == 3) return is_double ? optimize_array<double, 3>(nodes, node_count, ratio, iters, threads)
                                       : optimize_array<float, 3>(nodes, node_count, ratio, iters, threads);
        return is_double ? optimize_array<double, 2>(nodes, node_count, ratio, iters, threads)
                         : optimize_array<float, 2>(nodes, node_count, ratio, iters, threads);
    } catch (const std::exception& e) { set_error(std::string("optimize: ") + e.what()); return -1; }
}
BVH_EXPORT struct bvh_thread_pool* bvh_thread_pool_create(size_t thread_count) { return new bvh_thread_pool { thread_count }; }
BVH_EXPORT void bvh_thread_pool_destroy(struct bvh_thread_pool* pool) { delete pool; }

// The exported functions below only convert their arguments and call the templates above.
#define H(T, bvh) (reinterpret_cast<Handle<T>*>(bvh))
#define HC(T, bvh) (const_cast<Handle<T>*>(reinterpret_cast<const Handle<T>*>(bvh)))
#define H2(T, bvh) (reinterpret_cast<HostTree<T, 2>*>(bvh))
#define HC2(T, bvh) (reinterpret_cast<const HostTree<T, 2>*>(bvh))
#define N(T, D, node) (reinterpret_cast<HostNode<T, D>*>(node))
#define NC(T, D, node) (reinterpret_cast<const HostNode<T, D>*>(node))

#define BVH_IMPL_NODE(T, D, S)                                                                                     \
    BVH_EXPORT bool bvh_node##S##_is_leaf(const struct bvh_node##S* node) { return node_is_leaf(NC(T, D, node)); } \
    BVH_EXPORT size_t bvh_node##S##_get_prim_count(const struct bvh_node##S* node) { return node_prim_count(NC(T, D, node)); } \
    BVH_EXPORT void bvh_node##S##_set_prim_count(struct bvh_node##S* node, size_t count) { set_node_prim_count(N(T, D, node), count); } \
    BVH_EXPORT size_t bvh_node##S##_get_first_id(const struct bvh_node##S* node) { return node_first_id(NC(T, D, node)); } \
    BVH_EXPORT void bvh_node##S##_set_first_id(struct bvh_node##S* node, size_t first_id) { set_node_first_id(N(T, D, node), first_id); } \
    BVH_EXPORT struct bvh_bbox##S bvh_node##S##_get_bbox(const struct bvh_node##S* node) { return node_bbox<bvh_bbox##S>(NC(T, D, node)); } \
    BVH_EXPORT void bvh_node##S##_set_bbox(struct bvh_node##S* node, const struct bvh_bbox##S* bbox) { set_node_bbox(N(T, D, node), bbox); }

BVH_IMPL_NODE(float, 2, 2f)
BVH_IMPL_NODE(float, 3, 3f)
BVH_IMPL_NODE(double, 2, 2d)
BVH_IMPL_NODE(double, 3, 3d)

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
    BVH_EXPORT struct bvh##S* bvh##S##_build_boxes(const struct bvh_bbox##S* bboxes, const struct bvh_vec##S* centers, \
            size_t prim_count, const struct bvh_build_config* config, unsigned flags) {                            \
        return reinterpret_cast<bvh##S*>(build_boxes<T>(bboxes, centers, prim_count, config, flags)); }            \
    BVH_EXPORT void bvh##S##_destroy(struct bvh##S* bvh) { destroy_handle(H(T, bvh)); }                            \
    BVH_EXPORT void bvh##S##_save(const struct bvh##S* bvh, FILE* file) { save_handle(*HC(T, bvh), file); }        \
    BVH_EXPORT struct bvh##S* bvh##S##_load(FILE* file) { return reinterpret_cast<bvh##S*>(load_handle<T>(file)); } \
    BVH_EXPORT struct bvh_node##S* bvh##S##_get_node(struct bvh##S* bvh, size_t node_id) {                         \
        return reinterpret_cast<bvh_node##S*>(get_node(*H(T, bvh), node_id)); }                                    \
    BVH_EXPORT size_t bvh##S##_get_prim_id(const struct bvh##S* bvh, size_t i) { return get_prim_id(*HC(T, bvh), i); } \
    BVH_EXPORT size_t bvh##S##_get_prim_count(const struct bvh##S* bvh) { return get_prim_count(*HC(T, bvh)); }    \
    BVH_EXPORT size_t bvh##S##_get_node_count(const struct bvh##S* bvh) { return get_node_count(*HC(T, bvh)); }    \
    BVH_EXPORT void bvh##S##_append_node(struct bvh##S* bvh) { append_node(*H(T, bvh)); }                          \
    BVH_EXPORT void bvh##S##_remove_last_node(struct bvh##S* bvh) { remove_last_node(*H(T, bvh)); }                \
    BVH_EXPORT void bvh##S##_refit(struct bvh##S* bvh) { refit(*H(T, bvh)); }                                      \
    BVH_EXPORT void bvh##S##_optimize(struct bvh_thread_pool* pool, struct bvh##S* bvh) { optimize(H(T, bvh), pool_threads(pool)); } \
    BVH_EXPORT void bvh##S##_intersect_ray_any(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        intersect_ray<true, false>(*HC(T, bvh), reinterpret_cast<const T*>(ray), cb); }                           \
    BVH_EXPORT void bvh##S##_intersect_ray_any_robust(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        intersect_ray<true, true>(*HC(T, bvh), reinterpret_cast<const T*>(ray), cb); }                            \
    BVH_EXPORT void bvh##S##_intersect_ray(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        intersect_ray<false, false>(*HC(T, bvh), reinterpret_cast<const T*>(ray), cb); }                          \
    BVH_EXPORT void bvh##S##_intersect_ray_robust(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        intersect_ray<false, true>(*HC(T, bvh), reinterpret_cast<const T*>(ray), cb); }                           \
    BVH_EXPORT int bvh##S##_set_triangles(struct bvh##S* bvh, const T* vertices, size_t prim_count, unsigned flags) { \
        return set_handle_triangles(H(T, bvh), vertices, prim_count, flags); }                                     \
    BVH_EXPORT int bvh##S##_refit_triangles(struct bvh##S* bvh, const T* vertices, size_t prim_count, unsigned flags) { \
        return refit_handle_triangles(H(T, bvh), vertices, prim_count, flags); }                                   \
    BVH_EXPORT int bvh##S##_refit_boxes(struct bvh##S* bvh, const struct bvh_bbox##S* bboxes, size_t prim_count, unsigned flags) { \
        return refit_handle_boxes(H(T, bvh), bboxes, prim_count, flags); }                                         \
    BVH_EXPORT int bvh##S##_intersect_rays(struct bvh##S* bvh, const struct bvh_ray##S* rays, size_t ray_count,    \
            struct bvh_hit##S* hits, unsigned flags) {                                                             \
        return intersect_batch<T>(H(T, bvh), rays, ray_count, hits, nullptr, flags); }                             \
    BVH_EXPORT int bvh##S##_intersect_rays_gather(struct bvh##S* bvh, const struct bvh_ray##S* rays, size_t ray_count, \
            struct bvh_hit##S* hits, void* const* gathered_hits, int world_size, size_t shard_offset,              \
            void* multicast_hits, unsigned flags) {                                                                \
        return intersect_gather(H(T, bvh), reinterpret_cast<const DevRay<T>*>(rays), ray_count,                    \
            reinterpret_cast<DevHit<T>*>(hits), gathered_hits, world_size, shard_offset, multicast_hits, flags); } \
    BVH_EXPORT int bvh##S##_intersect_rays_stats(struct bvh##S* bvh, const struct bvh_ray##S* rays, size_t ray_count, \
            struct bvh_hit##S* hits, struct bvh_ray_stats* stats, unsigned flags) {                                \
        return intersect_batch_stats<T>(H(T, bvh), rays, ray_count, hits, stats, flags); }                         \
    BVH_EXPORT int bvh##S##_sync(struct bvh##S* bvh) { return sync_handle(H(T, bvh)); }                            \
    BVH_EXPORT size_t bvh##S##_get_depth(struct bvh##S* bvh) { return get_depth(H(T, bvh)); }                      \
    BVH_EXPORT const size_t* bvh##S##_get_prim_ids(struct bvh##S* bvh) { return get_prim_ids(H(T, bvh)); }         \
    BVH_EXPORT size_t bvh##S##_get_property(struct bvh##S* bvh, int property) { return get_property(H(T, bvh), property); } \
    BVH_EXPORT int bvh##S##_get_device_view(struct bvh##S* bvh, struct bvh_device_view##S* view) { return get_device_view(H(T, bvh), view); }

BVH_IMPL_3D(float, 3f, bvh_intersect_callbackf)
BVH_IMPL_3D(double, 3d, bvh_intersect_callbackd)

#define BVH_IMPL_2D(T, S, CALLBACK)                                                                                \
    BVH_EXPORT struct bvh##S* bvh##S##_build(struct bvh_thread_pool*, const struct bvh_bbox##S* bboxes,            \
            const struct bvh_vec##S* centers, size_t prim_count, const struct bvh_build_config* config) {          \
        return reinterpret_cast<bvh##S*>(build_tree2<T>(reinterpret_cast<const T*>(bboxes),                        \
            reinterpret_cast<const T*>(centers), prim_count, config));                                             \
    }                                                                                                              \
    BVH_EXPORT void bvh##S##_destroy(struct bvh##S* bvh) { delete H2(T, bvh); }                                    \
    BVH_EXPORT void bvh##S##_save(const struct bvh##S* bvh, FILE* file) { write_tree(*HC2(T, bvh), file); }        \
    BVH_EXPORT struct bvh##S* bvh##S##_load(FILE* file) { return reinterpret_cast<bvh##S*>(load_tree2<T>(file)); } \
    BVH_EXPORT struct bvh_node##S* bvh##S##_get_node(struct bvh##S* bvh, size_t node_id) {                         \
        return reinterpret_cast<bvh_node##S*>(get_node(*H2(T, bvh), node_id)); }                                   \
    BVH_EXPORT size_t bvh##S##_get_prim_id(const struct bvh##S* bvh, size_t i) { return get_prim_id(*HC2(T, bvh), i); } \
    BVH_EXPORT size_t bvh##S##_get_prim_count(const struct bvh##S* bvh) { return HC2(T, bvh)->prim_ids.size(); }   \
    BVH_EXPORT size_t bvh##S##_get_node_count(const struct bvh##S* bvh) { return HC2(T, bvh)->nodes.size(); }      \
    BVH_EXPORT void bvh##S##_append_node(struct bvh##S* bvh) { H2(T, bvh)->nodes.emplace_back(); }                 \
    BVH_EXPORT void bvh##S##_remove_last_node(struct bvh##S* bvh) { remove_last_node(*H2(T, bvh)); }               \
    BVH_EXPORT void bvh##S##_refit(struct bvh##S* bvh) { refit_nodes(H2(T, bvh)->nodes); }                         \
    BVH_EXPORT void bvh##S##_optimize(struct bvh_thread_pool* pool, struct bvh##S* bvh) { optimize(H2(T, bvh), pool_threads(pool)); } \
    BVH_EXPORT void bvh##S##_intersect_ray_any(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        intersect_nodes<true, false>(HC2(T, bvh)->nodes, reinterpret_cast<const T*>(ray), cb); }                  \
    BVH_EXPORT void bvh##S##_intersect_ray_any_robust(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        intersect_nodes<true, true>(HC2(T, bvh)->nodes, reinterpret_cast<const T*>(ray), cb); }                   \
    BVH_EXPORT void bvh##S##_intersect_ray(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        intersect_nodes<false, false>(HC2(T, bvh)->nodes, reinterpret_cast<const T*>(ray), cb); }                 \
    BVH_EXPORT void bvh##S##_intersect_ray_robust(const struct bvh##S* bvh, const struct bvh_ray##S* ray, const struct CALLBACK* cb) { \
        intersect_nodes<false, true>(HC2(T, bvh)->nodes, reinterpret_cast<const T*>(ray), cb); }

BVH_IMPL_2D(float, 2f, bvh_intersect_callbackf)
BVH_IMPL_2D(double, 2d, bvh_intersect_callbackd)

} // extern "C"
