// include/bvh/v2/cuda/intersect.cuh — traverse a GPU-built BVH from your own CUDA kernels.
//
// The reference library's ray extension point is Bvh::intersect<IsAnyHit, IsRobust>(ray, start, stack, leaf_fn,
// inner_fn) (reference bvh.h:59-73,159-182): the library walks the tree, the caller intersects the primitives of every
// leaf it reaches and shrinks ray.tmax on a hit.  DeviceView::intersect is that call on the device, over the tree a
// handle keeps on its GPU.  It runs the library's own stack machine (bvhb200::traverse_top_down, traverse_core.cuh, the
// one the batched kernels use), so it visits the same leaves in the same order as the reference's Bvh::intersect on the
// same tree.  The general form, Bvh::traverse_top_down with the caller's own node test, is
// DeviceView::traverse_top_down ("Queries other than rays", below).
//
//     bvh3f* bvh = bvh3f_build(nullptr, bboxes, centers, n, nullptr);     // or bvh3f_build_triangles
//     bvh_device_view3f c;
//     bvh3f_get_device_view(bvh, &c);                                       // include/bvh_b200_device.h
//     auto view = bvh::v2::cuda::DeviceView<float>::from(c);               // pass it to the kernel by value
//
//     __global__ void kernel(bvh::v2::cuda::DeviceView<float> view, const MySphere* spheres, bvh_ray3f* rays, ...) {
//         using View = bvh::v2::cuda::DeviceView<float>;
//         bvh_ray3f ray = rays[i];
//         View::SmallStack<64> stack;                                      // capacity >= view.stack_bound()
//         size_t best = SIZE_MAX;
//         view.intersect<false, false>(ray, view.root_index(), stack, [&](size_t begin, size_t end) {
//             for (size_t k = begin; k < end; ++k)                         // BVH-order slots; spheres[view.prim_id(k)]
//                 if (my_test(spheres[view.prim_id(k)], ray)) { ray.tmax = ...; best = k; }
//             return best != SIZE_MAX;
//         });
//     }
//
// Compile with (nvcc 12.x, sm_90a):
//     nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -I <repo>/include -I <repo>/bvh_b200/csrc ...
// The traversal's own arithmetic uses round-to-nearest intrinsics and is exact under any flags.  A leaf function's
// arithmetic is the caller's: to match a host computation bit for bit, compile with --fmad=false (or write it with the
// __fadd_rn / __fmul_rn family), since nvcc otherwise contracts a * b + c into one FMA.  The header also compiles as
// plain host C++ (g++ -std=c++17, same include flags), where the same traversal runs on host-resident copies of the
// arrays.
//
// Rules a leaf function follows (the reference's, bvh.h:124-157):
//   * it receives a BVH-order range [begin, end); view.prim_id(k) is the original primitive id of slot k;
//   * it may shrink (or otherwise change) ray.tmax and ray.tmin: the next box test reads them.  Other ray fields are
//     read once, before the traversal starts;
//   * it returns whether it hit; with IsAnyHit a true return ends the traversal.
// The inner hook, when given, is called once per inner step with the reference index of the left child of the node
// being expanded (the right child is that index + 1), before the step's box tests: the reference's InnerFn, which
// receives those two nodes.
//
// Queries other than rays: view.traverse_top_down<IsAnyHit>(start, stack, leaf_fn, node_fn) is the reference's
// Bvh::traverse_top_down (bvh.h:59-65,124-157), of which intersect is one instance.  It starts at `start`; while the
// current node is an inner node it calls node_fn on its two children and descends to the near one, pushes the far one
// when both are hit, and pops the stack when neither is; at a leaf it calls leaf_fn; it ends when the stack is empty.
//   * node function: called as node_fn(const Node& left, const Node& right) with register copies of the two children
//     (node.bounds[6] as minx, maxx, miny, maxy, minz, maxz, node.index), or as node_fn(left, right, size_t left_index)
//     when it takes a third argument: the reference index of the left child (the right one is left_index + 1), what
//     `&left - bvh.nodes.data()` gives on the host, so that it can read data the caller keeps per node (below, "Data per
//     node").  It returns anything that unpacks with a
//     structured binding into three values convertible to bool, (hit_left, hit_right, should_swap): an aggregate of
//     three bools, cuda::std::tuple on the device or std::tuple on the host (std::tuple is not device code).
//     should_swap (visit the right child first) applies when both children are hit, whatever IsAnyHit is;
//   * leaf function: leaf_fn(size_t begin, size_t end) -> bool with BVH-order slots, as for intersect; with IsAnyHit a
//     true return ends the traversal.  A leaf `start` gets one leaf_fn call and no node_fn call;
//   * shared state: the two functions may share state (a search radius the leaf shrinks, a count); every node_fn call
//     comes after all earlier leaf_fn calls have returned;
//   * stacks: the same as for intersect, with the same bound, stack_bound() = depth + 1.
// Each sibling pair is read as one aligned 64-byte (float) / 128-byte (double) block through the read-only path.  A
// box-overlap query (collision broad phase), counting the primitives whose boxes overlap a query box:
//
//     struct Pick { bool left, right, swap; };
//     __device__ bool overlaps(const float* b, const bvh_bbox3f& q) {        // b: minx, maxx, miny, maxy, minz, maxz
//         return b[0] <= q.max.x && q.min.x <= b[1] && b[2] <= q.max.y && q.min.y <= b[3] &&
//                b[4] <= q.max.z && q.min.z <= b[5];
//     }
//     __global__ void overlap(View view, const bvh_bbox3f* boxes, const bvh_bbox3f* queries, uint32_t* counts, size_t n) {
//         const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
//         if (i >= n) return;
//         const bvh_bbox3f q = queries[i];
//         View::SmallStack<64> stack;
//         uint32_t count = 0;
//         view.traverse_top_down<false>(view.root_index(), stack,
//             [&](size_t begin, size_t end) {
//                 for (size_t k = begin; k < end; ++k) {
//                     const bvh_bbox3f b = boxes[view.prim_id(k)];             // original order
//                     const float f[6] = { b.min.x, b.max.x, b.min.y, b.max.y, b.min.z, b.max.z };
//                     count += overlaps(f, q);
//                 }
//                 return false;
//             },
//             [&](const View::Node& l, const View::Node& r) { return Pick { overlaps(l.bounds, q), overlaps(r.bounds, q), false }; });
//         counts[i] = count;
//     }
//
// Data per node: view.traverse_bottom_up(workspace, workspace_bytes, leaf_fn, inner_fn[, stream]) is the reference's
// Bvh::traverse_bottom_up (bvh.h:184-208), the pass Bvh::refit is built on, for data the caller computes per node: mass
// and centre of mass (Barnes-Hut), summed power and normal cones (light trees), a subtree's largest radius or speed, its
// primitive count.  It runs on the GPU, one thread per leaf climbing towards the root, in two kernels on `stream` (the
// handle's by default) with no host synchronisation: bottom_up_link_kernel, then bottom_up_climb_kernel, over slots
// [1, node_count].
//   * leaf_fn(size_t node, size_t begin, size_t end) is called once per leaf, with its reference index and its BVH-order
//     primitive range [begin, end) (view.prim_id(k) is the original id of slot k, as for intersect);
//   * inner_fn(size_t node, size_t left) is called once per inner node, with its reference index and its left child's
//     (the right one is left + 1);
//   * both are device function objects, copied to the kernel by value: a struct with a __device__ (or
//     __host__ __device__) operator(), or an extended __device__ lambda (nvcc --extended-lambda);
//   * every node of a tree whose nodes are all reachable from the root gets exactly one call; every tree the library
//     builds, and every tree it loads from the reference's format, is such a tree;
//   * an inner node's call comes after both of its children's calls, and their global writes are visible to it (the
//     arrival at a parent is an acquire-release atomic at device scope).  Data the pass writes must not be read through
//     __ldg or a `const __restrict__` pointer inside the pass: the read-only path does not see other threads' writes;
//   * the order is otherwise unspecified, and differs from run to run on the device.  A function that combines only its
//     children's values (and its leaf's primitives) therefore gives a result that does not depend on the order;
//   * workspace: view.bottom_up_workspace_bytes() bytes of device memory, allocated by the caller and not initialised:
//     the pass writes its parent links and clears its arrival flags itself, so the same workspace serves pass after pass
//     on one stream.  Two passes must not share one workspace at the same time.  A smaller workspace throws
//     std::length_error, a failed launch std::runtime_error;
//   * compiled as plain host C++, the pass runs serially on host-resident copies, in the reference's order: leaves in
//     descending index, each climbing while both children of the parent are done, which is the call sequence of
//     Bvh::traverse_bottom_up.
// Subtree mass and centre of mass, then a Barnes-Hut potential that reads them through the three-argument node test
// (compile with --fmad=false to match a host computation bit for bit):
//
//     struct MassCentre {                                                  // one object serves as leaf_fn and inner_fn
//         const uint32_t* prim_ids; const float* pos; const float* mass;  // pos: x, y, z per particle, original order
//         float* node_mass; float* node_centre;                            // node_count and 3 * node_count floats
//         __device__ void operator()(size_t node, size_t begin, size_t end) const {          // leaf
//             float m = 0, c[3] = { 0, 0, 0 };
//             for (size_t k = begin; k < end; ++k) {
//                 const uint32_t id = prim_ids[k];
//                 m += mass[id];
//                 for (int a = 0; a < 3; ++a) c[a] += mass[id] * pos[3 * id + a];
//             }
//             node_mass[node] = m;
//             for (int a = 0; a < 3; ++a) node_centre[3 * node + a] = c[a] / m;
//         }
//         __device__ void operator()(size_t node, size_t left) const {                        // inner: after both children
//             const float ml = node_mass[left], mr = node_mass[left + 1], m = ml + mr;
//             node_mass[node] = m;
//             for (int a = 0; a < 3; ++a)
//                 node_centre[3 * node + a] = (ml * node_centre[3 * left + a] + mr * node_centre[3 * (left + 1) + a]) / m;
//         }
//     };
//     size_t bytes = view.bottom_up_workspace_bytes();                     // on the host
//     void* workspace; cudaMallocAsync(&workspace, bytes, stream);
//     const MassCentre mc { view.prim_ids, d_pos, d_mass, d_node_mass, d_node_centre };
//     view.traverse_bottom_up(workspace, bytes, mc, mc, stream);
//     potential<<<blocks, 128, 0, stream>>>(view, d_node_mass, d_node_centre, d_pos, d_mass, d_points, m, 0.25f, d_phi);
//
//     __global__ void potential(View view, const float* node_mass, const float* node_centre, const float* pos,
//                               const float* mass, const float* points, size_t m, float theta2, float* phi) {
//         const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
//         if (i >= m) return;
//         const float p[3] = { points[3 * i], points[3 * i + 1], points[3 * i + 2] };
//         auto dist2 = [&](const float* c) { float d = 0; for (int a = 0; a < 3; ++a) d += (c[a] - p[a]) * (c[a] - p[a]); return d; };
//         float sum = 0;
//         // far enough (node size < theta * distance): the node's mass at its centre, and no descent
//         auto open = [&](const View::Node& n, size_t k) {
//             const float size = fmaxf(fmaxf(n.bounds[1] - n.bounds[0], n.bounds[3] - n.bounds[2]), n.bounds[5] - n.bounds[4]);
//             const float d2 = dist2(node_centre + 3 * k);
//             if (size * size < theta2 * d2) { sum -= node_mass[k] / sqrtf(d2); return false; }
//             return true;
//         };
//         View::SmallStack<64> stack;
//         view.traverse_top_down<false>(view.root_index(), stack,
//             [&](size_t begin, size_t end) {
//                 for (size_t k = begin; k < end; ++k) {
//                     const uint32_t id = view.prim_id(k);
//                     sum -= mass[id] / sqrtf(dist2(pos + 3 * id));
//                 }
//                 return false;
//             },
//             [&](const View::Node& l, const View::Node& r, size_t left) {
//                 const bool open_left = open(l, left), open_right = open(r, left + 1);
//                 return Pick { open_left, open_right, false };
//             });
//         phi[i] = sum;
//     }
//
// Whole batches: view.trace<IsAnyHit, IsRobust>(n, tracer, workspace, workspace_bytes[, stream]) traces rays 0 .. n-1
// with the library's persistent scheduler, the one bvhNN_intersect_rays uses (persistent_core.cuh): persistent warps,
// runs of consecutive rays claimed with one atomic, idle lanes refilled together once enough of them are idle, a
// bounded inner phase and one leaf per round, a shared-memory stack.  Neighbouring rays start together and share their
// node fetches, which one thread per ray through intersect does not get.  The tracer is a plain struct copied to the
// kernel by value, with a Payload type (per-ray state, kept in registers) and three __device__ (or __host__ __device__)
// functions:
//     Ray  start(size_t i, Payload& p) const;                              // ray i of the batch; sets up p
//     bool leaf(Payload& p, Ray& ray, size_t begin, size_t end) const;    // intersect's leaf_fn
//     void finish(size_t i, const Payload& p, const Ray& ray) const;      // ray i is done
//   * for every i in [0, n), start is called once, then the leaf calls, then finish once.  The leaf calls of a ray are
//     exactly those intersect<IsAnyHit, IsRobust>(ray, root_index(), stack, leaf) makes on the same tree: the same
//     (begin, end) ranges in the same order.  A ray whose interval is a NaN at the start gets no leaf call when the root
//     is an inner node and one when it is a leaf; after a leaf that makes the interval a NaN, the remaining stack
//     entries are drawn without box tests, as traverse_top_down does;
//   * leaf may change ray.tmin and ray.tmax, and the next box test reads them; other ray fields are read once, from
//     what start returned.  With IsAnyHit a true return ends the ray.  finish receives the ray with its final interval;
//   * rays are drawn in index order, in runs per warp, so neighbouring indices share node fetches: number the rays
//     coherently (by pixel tile, by origin) to get coherence.  No ordering holds between different rays;
//   * the three functions run on a subset of a warp's lanes: they must not use __syncthreads or full-mask warp
//     collectives;
//   * there is no watchdog (intersect has none either): a leaf function that never returns hangs the kernel;
//   * the call is stream-ordered on `stream` (the handle's by default), does not synchronise the host, and sets and
//     restores the current device.  n == 0 launches nothing.  Scheduling uses the library's defaults for a
//     closest-hit or any-hit batch (plan_trace, trace_plan.h); there is nothing to set;
//   * workspace: view.trace_workspace_bytes() bytes of device memory (the run cursor), allocated by the caller and not
//     initialised: trace resets it on the stream.  Two calls must not share a workspace at the same time.  A smaller
//     workspace throws std::length_error, and so does a tree whose shared-memory stack would exceed the 200 KB a
//     persistent block may have (float: depth > 398); a failed launch throws std::runtime_error;
//   * compiled as plain host C++, trace runs the rays serially: start, intersect with a host stack of stack_bound()
//     entries, finish.
// The kernel is bvh::v2::cuda::device_view_trace_kernel<T, IsAnyHit, IsRobust, Tracer>, 128 threads per block; its
// registers are limited for 9 resident blocks per SM (float) or 4 (double), as the library's persistent kernel's are, so
// a payload of more than a few words spills.  A sphere tracer (INTEGRATION.md §5 has it whole):
//
//     struct SphereTracer {
//         struct Payload { uint32_t best; };
//         const bvh_ray3f* rays; const float4* spheres; const uint32_t* prim_ids; uint32_t* hit_ids;
//         __device__ bvh_ray3f start(size_t i, Payload& p) const { p.best = UINT32_MAX; return rays[i]; }
//         __device__ bool leaf(Payload& p, bvh_ray3f& ray, size_t begin, size_t end) const {
//             for (size_t k = begin; k < end; ++k)
//                 if (float t; hit_sphere(spheres[prim_ids[k]], ray, t)) { ray.tmax = t; p.best = prim_ids[k]; }
//             return p.best != UINT32_MAX;
//         }
//         __device__ void finish(size_t i, const Payload& p, const bvh_ray3f&) const { hit_ids[i] = p.best; }
//     };
//     view.trace<false, false>(n, SphereTracer { d_rays, d_spheres, view.prim_ids, d_hit_ids }, workspace, bytes, stream);
//
// Whole batches of queries: view.query<IsAnyHit>(n, querier, workspace, workspace_bytes[, stream]) is the batch form of
// traverse_top_down, on the same scheduler as trace: queries 0 .. n-1 with the caller's node test (box overlap, nearest
// neighbour, point location, Barnes-Hut), in runs per warp, idle lanes refilled together, a shared-memory stack sized
// from the tree's depth.  The querier is a plain struct copied to the kernel by value, with a Payload type (per-query
// state, kept in registers) and four __device__ (or __host__ __device__) functions:
//     void start(size_t i, Payload& p) const;                                  // query i of the batch; sets up p
//     auto node(Payload& p, const Node& left, const Node& right) const;         // or (..., size_t left_index)
//     bool leaf(Payload& p, size_t begin, size_t end) const;                   // BVH-order primitive range
//     void finish(size_t i, const Payload& p) const;                           // query i is done
//   * for every i in [0, n), start is called once, then exactly the node and leaf calls that
//     traverse_top_down<IsAnyHit>(root_index(), stack, leaf', node') makes for that query, with the same arguments in
//     the same order (leaf' and node' are leaf and node bound to the query's payload), then finish once.  A root that is
//     a leaf gets one leaf call and no node call;
//   * node returns what traverse_top_down's node function returns: anything that unpacks into (hit_left, hit_right,
//     should_swap).  Node is View::Node.  The three-argument form receives the left child's reference index, so that it
//     can read data written per node by traverse_bottom_up;
//   * with IsAnyHit a true return from leaf ends the query;
//   * queries are drawn in index order, in runs per warp, so neighbouring indices share node fetches.  No ordering holds
//     between different queries.  The functions run on a subset of a warp's lanes: they must not use __syncthreads or
//     full-mask warp collectives.  There is no watchdog;
//   * the call is stream-ordered on `stream` (the handle's by default), does not synchronise the host, and sets and
//     restores the current device.  n == 0 launches nothing.  Scheduling uses plan_query() (trace_plan.h); there is
//     nothing to set;
//   * workspace: view.query_workspace_bytes() bytes of device memory, as for trace.  A smaller workspace, or a tree too
//     deep for the 200 KB shared-memory stack (float: depth > 398), throws std::length_error; a failed launch throws
//     std::runtime_error;
//   * compiled as plain host C++, query runs the queries serially: start, traverse_top_down with a host stack, finish.
// The kernel is bvh::v2::cuda::device_view_query_kernel<T, IsAnyHit, Querier>, with trace's launch bounds, block size,
// stack and run length.  Counting the primitive boxes that overlap each query box (Pick and overlaps as above):
//
//     struct OverlapCounter {
//         struct Payload { bvh_bbox3f q; uint32_t count; };
//         const bvh_bbox3f* queries; const bvh_bbox3f* boxes; const uint32_t* prim_ids; uint32_t* counts;
//         __device__ void start(size_t i, Payload& p) const { p.q = queries[i]; p.count = 0; }
//         __device__ Pick node(Payload& p, const View::Node& l, const View::Node& r) const {
//             return Pick { overlaps(l.bounds, p.q), overlaps(r.bounds, p.q), false };
//         }
//         __device__ bool leaf(Payload& p, size_t begin, size_t end) const {
//             for (size_t k = begin; k < end; ++k) {
//                 const bvh_bbox3f b = boxes[prim_ids[k]];
//                 const float f[6] = { b.min.x, b.max.x, b.min.y, b.max.y, b.min.z, b.max.z };
//                 p.count += overlaps(f, p.q);
//             }
//             return false;
//         }
//         __device__ void finish(size_t i, const Payload& p) const { counts[i] = p.count; }
//     };
//     view.query<false>(n, OverlapCounter { d_queries, d_boxes, view.prim_ids, d_counts }, workspace, bytes, stream);
//
// Whole batches of triangle rays: view.trace_triangles<IsAnyHit, IsRobust, TieLastVisited = false>(n, shader, workspace,
// workspace_bytes[, stream]) runs the library's own triangle traversal (the inner step, leaf and record of
// bvhNN_intersect_rays' persistent kernel) on the scheduler trace uses, with the caller's ray source, hit filter and hit
// sink: what OptiX calls raygen, any-hit and closest-hit programs, reduced to the library's semantics.  The view must have
// triangles (a tree from bvhNN_build_triangles or with bvhNN_set_triangles).  The shader is a plain struct copied to the
// kernel by value, with a Payload type (per-ray state, kept in registers) and three __device__ (or __host__ __device__)
// functions:
//     Ray  start(size_t i, Payload& p) const;                                  // ray i of the batch; sets up p
//     bool accept(Payload& p, size_t prim_id, T t, T u, T v) const;             // a candidate hit; false: ignore it
//     void finish(size_t i, const Payload& p, const Hit& hit) const;           // ray i is done; Hit is bvh_hit3f / 3d
//   * for every i in [0, n), start is called once, then the accept calls, then finish once;
//   * accept is called once per triangle of each leaf reached (in BVH order within the leaf, leaves in the reference's
//     visit order) that passes PrecomputedTri::intersect with its t in [tmin, tmax] and that the tie rule would take as
//     the new closest hit: the lowest original id at equal t, or the last visited with TieLastVisited
//     (BVH_TIE_LAST_VISITED).  prim_id is the original id.  The accept calls of a ray are exactly those a host leaf loop
//     running the same test, tie rule and filter makes in Bvh::intersect<IsAnyHit, IsRobust> on the same tree;
//   * true from accept records the hit and shrinks tmax; with IsAnyHit the ray then ends after that leaf (the leaf's
//     remaining triangles are still tested, as in the library's kernel).  false changes nothing;
//   * finish receives the record bvhNN_intersect_rays writes: the original id, or all ones on a miss; t, or the input
//     tmax on a miss; u and v, or 0 on a miss.  A shader whose accept returns true and whose start and finish read and
//     write arrays reproduces bvhNN_intersect_rays(flags) bit for bit.  A ray whose interval is a NaN gets no accept call
//     and finishes as a miss, as in the library's kernels;
//   * ordering, the warp subset (no __syncthreads, no full-mask collectives), no watchdog, streams, n == 0 and the host
//     build are those of trace.  workspace: view.trace_workspace_bytes() bytes (the run cursor).  A smaller workspace or a
//     tree too deep for the 200 KB shared-memory stack throws std::length_error, a view without triangles
//     std::invalid_argument, a failed launch std::runtime_error.  Compiled as plain host C++, the rays run serially.
// The kernel is bvh::v2::cuda::device_view_triangle_kernel<T, IsAnyHit, IsRobust, TieLastVisited, Shader>, with trace's
// launch bounds, block and stack and the scheduling of bvhNN_intersect_rays' persistent kernel (14 / 4 for closest-hit
// rays).  Under the float bounds (56 registers) an empty payload does not spill; every word of payload competes with the
// traversal's own state, so keep it to a few words.  Shadow rays that leave a surface skip the triangle they start on
// (self-intersection):
//
//     struct ShadowShader {
//         struct Payload { uint32_t origin; };
//         const bvh_ray3f* rays; const uint32_t* origin_ids; uint8_t* lit;   // origin_ids: the triangle each ray leaves
//         __device__ bvh_ray3f start(size_t i, Payload& p) const { p.origin = origin_ids[i]; return rays[i]; }
//         __device__ bool accept(Payload& p, size_t prim_id, float, float, float) const { return prim_id != p.origin; }
//         __device__ void finish(size_t i, const Payload&, const bvh_hit3f& hit) const { lit[i] = hit.prim_id == UINT32_MAX; }
//     };
//     view.trace_triangles<true, false>(n, ShadowShader { d_rays, d_origins, d_lit }, workspace, bytes, stream);
//
// Whole paths: view.trace_paths<IsRobust, TieLastVisited = false>(n, shader, workspace, workspace_bytes[, stream]) traces
// paths 0 .. n-1, each a sequence of triangle-ray segments (bounce and shadow rays of a path tracer, ambient occlusion
// with bounces, acoustics), in one launch: when a segment ends, its lane starts the path's next segment in place, with
// the same payload registers and the same shared-memory stack; only lanes whose path is over are refilled.  What OptiX
// calls tracing from closest-hit, reduced to the library's semantics.  The shader is a plain struct copied to the kernel
// by value, with a Payload type (per-path state, kept in registers) and four __device__ (or __host__ __device__)
// functions:
//     PathStep start(size_t i, Payload& p, Ray& ray) const;                     // first segment of path i, or End
//     bool     accept(Payload& p, size_t prim_id, T t, T u, T v) const;         // exactly as in trace_triangles
//     PathStep next(size_t i, Payload& p, const Hit& hit, Ray& ray) const;      // a segment ended: the next one, or End
//     void     finish(size_t i, const Payload& p) const;                        // path i is done
// PathStep is End, Closest or Occlusion.
//   * for every i in [0, n), start is called once, then zero or more segments, then finish once.  If start returns End,
//     finish follows directly;
//   * each segment is what trace_triangles does for that ray: a Closest segment is trace_triangles<false, IsRobust,
//     TieLastVisited>, an Occlusion segment trace_triangles<true, IsRobust, TieLastVisited>.  It gets the same accept
//     calls, with the same ids and the same bits of t, u and v, in the same order, and then next with the record
//     trace_triangles would hand to finish.  A segment whose interval is a NaN gets no accept call and a miss record;
//   * on entry to next, `ray` is the segment's ray as start or the previous next returned it, not shrunk by the
//     traversal.  On a return other than End, `ray` is the next segment;
//   * the payload lives across segments.  Different paths may be in different segment kinds in the same warp;
//   * the other rules are those of trace_triangles: no __syncthreads and no full-mask collectives in shader code; no
//     watchdog (a shader that never returns End never ends); stream-ordered, setting and restoring the current device;
//     n == 0 launches nothing; workspace: view.trace_workspace_bytes() bytes.  A smaller workspace or a tree too deep for
//     the 200 KB shared-memory stack throws std::length_error, a view without triangles std::invalid_argument, a failed
//     launch std::runtime_error;
//   * scheduling uses plan_trace's closest-hit settings for the whole batch, with grid and run length from n;
//   * compiled as plain host C++, the paths run serially, each segment through the host code of one trace_triangles ray.
// The kernel is bvh::v2::cuda::device_view_path_kernel<T, IsRobust, TieLastVisited, Shader>, with trace_triangles'
// launch bounds, block, stack and phases; a lane's segment kind picks the any-hit or closest-hit inner step.  The payload
// competes with the traversal for the float kernel's 56 registers: keep it to a few words.  A grey diffuse path tracer
// with a point light and next-event estimation (INTEGRATION.md §5 has it whole):
//
//     struct PathTracer {
//         struct Payload { float throughput, radiance, pending; uint32_t prim, bounce; };   // pending: the shadow ray's share
//         ...                                                                 // camera, light, normals, radiance out
//         __device__ PathStep start(size_t i, Payload& p, bvh_ray3f& ray) const {
//             ray = camera_ray(i); p = { 1.0f, 0.0f, 0.0f, UINT32_MAX, 0 };
//             return PathStep::Closest;
//         }
//         __device__ bool accept(Payload& p, size_t prim_id, float, float, float) const { return prim_id != p.prim; }
//         __device__ PathStep next(size_t i, Payload& p, const bvh_hit3f& hit, bvh_ray3f& ray) const {
//             if (p.pending != 0.0f) {                                       // a shadow segment ended
//                 if (hit.prim_id == UINT32_MAX) p.radiance += p.pending;
//                 p.pending = 0.0f;
//                 return bounce(i, p, ray);                                  // ray.org is the surface point
//             }
//             if (hit.prim_id == UINT32_MAX) { p.radiance += p.throughput * sky; return PathStep::End; }
//             p.prim = hit.prim_id;
//             ray.org = ray.org + hit.t * ray.dir;                           // the surface point
//             p.pending = light_share(p, ray.org);                           // 0 when the light is behind the surface
//             if (p.pending == 0.0f) return bounce(i, p, ray);
//             ray.dir = light - ray.org; ray.tmin = 0.0f; ray.tmax = 1.0f;
//             return PathStep::Occlusion;
//         }
//         __device__ void finish(size_t i, const Payload& p) const { image[i] = p.radiance; }
//     };
//     view.trace_paths<false>(width * height, PathTracer { ... }, workspace, bytes, stream);
//
// Instanced scenes: top.trace_instances<IsAnyHit, IsRobust, TieLastVisited = false>(n, instances, shader, workspace,
// workspace_bytes[, stream]) traces triangle rays through a two-level scene: each distinct mesh keeps its own tree (built
// once with bvhNN_build_triangles), and `top` is a tree over the world boxes of its placed copies.  An Instance<T> record
// (make_instance(view, object_to_world)) holds a bottom tree's device arrays, its root and depth, a 3 x 4 row-major
// object_to_world matrix the caller writes and its inverse world_to_object; Instances<T> { records, count, max_depth }
// views count records in device memory, max_depth being the largest bottom depth.  prepare_instances(instances, bboxes,
// centers[, stream]) writes every root index and world_to_object, and the world boxes and centres (bvh_bbox3f / bvh_vec3f, or 3d) that
// bvhNN_build_boxes or bvhNN_refit_boxes take with BVH_DEVICE_POINTERS, in one stream-ordered kernel.  Top primitive k is
// record k: build the top tree from those arrays, then for a rigid move rewrite object_to_world, prepare_instances and
// refit_boxes on the top handle's stream, and trace.  The shader is a plain struct copied to the kernel by value, with a
// Payload type and three __device__ (or __host__ __device__) functions:
//     Ray  start(size_t i, Payload& p) const;                                          // ray i of the batch (world space)
//     bool accept(Payload& p, uint32_t instance, size_t prim_id, T t, T u, T v) const;  // a candidate hit; false: ignore it
//     void finish(size_t i, const Payload& p, const Hit& hit, uint32_t instance) const; // ray i is done; all ones: a miss
//   * for every i in [0, n), start once, then the accept calls, then finish once.  They are exactly the calls of this host
//     loop, which is what the header compiled as plain host C++ runs: Bvh::intersect<IsAnyHit, IsRobust> on the top tree,
//     whose leaf takes the leaf's instances in BVH order and, for each, transforms the world ray by world_to_object
//     (origin as a point, direction as a vector, tmin and tmax unchanged: detail::object_ray), runs the instance's
//     Bvh::intersect<IsAnyHit, IsRobust> with a PrecomputedTri::intersect leaf, the tie rule and accept as the filter, and
//     carries the shrunk tmax back to the top level.  An instance whose world_to_object is NaN (no inverse) is skipped;
//   * t is the world ray's parameter (the object ray is not normalised); u and v are the object-space barycentrics;
//     prim_id is the bottom mesh's original id; `instance` is the record's index;
//   * tie rule: at an exact tie in t the canonical rule keeps the lower instance, then the lower original id; with
//     TieLastVisited the last visited candidate wins.  true from accept records the hit and shrinks tmax; with IsAnyHit
//     the ray ends after the bottom leaf that accepted it.  A ray whose interval is a NaN finishes at once as a miss with
//     no accept call.  finish receives the record of trace_triangles (id, t, u, v; on a miss all ones, the input tmax, 0,
//     0) and the hit's instance;
//   * with one instance whose matrix is the identity (its world box a top tree of one leaf), the accept calls and the
//     record are those of trace_triangles on that mesh, bit for bit: detail::affine_row maps coordinates exactly through
//     an identity, a permutation or a power-of-two scale;
//   * errors, checked on the host before any launch: instances.count other than the top tree's prim_count throws
//     std::invalid_argument; a stack of top depth + max_depth + 9 entries per ray beyond the 200 KB shared-memory stack,
//     or a small workspace, std::length_error; a failed launch std::runtime_error.  That every record's bottom view has
//     triangles, outlives the call and that max_depth is right is the caller's, like the view-lifetime rules;
//   * streams, the workspace (trace_workspace_bytes()), n == 0, the warp subset and the watchdog are those of
//     trace_triangles.  Compiled as plain host C++, the rays run serially through the nested loop above.
// The kernel is bvh::v2::cuda::device_view_instance_kernel<T, IsAnyHit, IsRobust, TieLastVisited, Shader>, with
// trace_triangles' launch bounds, block, scheduling and launch: each lane walks both levels in one stack machine on its
// shared-memory stack (DESIGN.md §8 has the layout).  Two meshes, three copies, one frame (INTEGRATION.md §5 has it whole):
//
//     struct Shade {
//         struct Payload {};
//         const bvh_ray3f* rays; bvh_hit3f* hits; uint32_t* inst;
//         __device__ bvh_ray3f start(size_t i, Payload&) const { return rays[i]; }
//         __device__ bool accept(Payload&, uint32_t, size_t, float, float, float) const { return true; }
//         __device__ void finish(size_t i, const Payload&, const bvh_hit3f& h, uint32_t k) const { hits[i] = h; inst[i] = k; }
//     };
//     Instance<float> recs[3] = { make_instance(rock, m0), make_instance(rock, m1), make_instance(tree, m2) };  // host
//     cudaMemcpyAsync(d_recs, recs, sizeof recs, cudaMemcpyHostToDevice, stream);
//     const Instances<float> instances { d_recs, 3, std::max(rock.depth, tree.depth) };
//     prepare_instances(instances, d_boxes, d_centres, stream);
//     bvh3f* top_bvh = bvh3f_build_boxes(d_boxes, d_centres, 3, nullptr, BVH_DEVICE_POINTERS);   // once; later frames:
//     // bvh3f_refit_boxes(top_bvh, d_boxes, 3, BVH_DEVICE_POINTERS) after prepare_instances on the top handle's stream
//     top.trace_instances<false, false>(n, instances, Shade { d_rays, d_hits, d_inst }, workspace, bytes, stream);
//
// Paths through instanced scenes: top.trace_instance_paths<IsRobust, TieLastVisited = false>(n, instances, shader,
// workspace, workspace_bytes[, stream]) is trace_paths over the two-level scene of trace_instances: `top` and `instances`
// as for trace_instances, and a shader with a Payload type (per-path state, kept in registers) and four __device__ (or
// __host__ __device__) functions:
//     PathStep start(size_t i, Payload& p, Ray& ray) const;                                 // world-space first segment, or End
//     bool     accept(Payload& p, uint32_t instance, size_t prim_id, T t, T u, T v) const;  // as in trace_instances
//     PathStep next(size_t i, Payload& p, const Hit& hit, uint32_t instance, Ray& ray) const;
//     void     finish(size_t i, const Payload& p) const;
//   * for every i in [0, n), start is called once, then zero or more segments, then finish once.  If start returns End,
//     finish follows directly;
//   * a Closest segment is exactly trace_instances<false, IsRobust, TieLastVisited> for that world ray, an Occlusion
//     segment trace_instances<true, IsRobust, TieLastVisited>: the same accept calls (instance, original id, bits of t, u
//     and v) in the same order, then next with the record and instance trace_instances' finish would get (kNoInstance,
//     all ones, on a miss).  A segment whose interval is a NaN gets no accept call and a miss record;
//   * on entry to next, `ray` is the segment's world ray as start or the previous next returned it, bit for bit: not
//     shrunk and not in object space.  On a return other than End, `ray` is the next segment;
//   * the payload lives across segments; lanes of one warp may be in different segment kinds and at different levels;
//   * one identity instance under a top tree of one leaf gives trace_paths on that mesh bit for bit, instance 0 for every
//     hit;
//   * errors, checked on the host before any launch, as for trace_instances: instances.count other than the top tree's
//     prim_count throws std::invalid_argument; a stack of top depth + max_depth + 9 entries beyond the 200 KB
//     shared-memory stack, or a small workspace, std::length_error; a failed launch std::runtime_error.  The workspace
//     (trace_workspace_bytes()), n == 0, streams, the current device, the warp subset and the watchdog are those of
//     trace_paths.  Compiled as plain host C++, the paths run serially, each segment through the nested loop of one
//     trace_instances ray.
// The kernel is bvh::v2::cuda::device_view_instance_path_kernel<T, IsRobust, TieLastVisited, Shader>, with
// trace_instances' launch bounds, block, stack and launch and plan_trace's closest-hit settings.  A lane's segment kind
// picks the any-hit or closest-hit inner step at either level.  An occlusion segment can end inside an instance: the
// world origin and direction are then popped back from under the marker on the lane's stack before next runs.  The
// payload competes with the traversal for the float kernel's 56 registers.  A shadow-ray shader that skips the
// (instance, triangle) its path stands on (INTEGRATION.md §5 has a path tracer whole):
//
//     struct Paths {
//         struct Payload { uint32_t inst, prim; float radiance; };
//         ...                                                                 // camera, light, records, radiance out
//         __device__ PathStep start(size_t i, Payload& p, bvh_ray3f& ray) const {
//             ray = camera_ray(i); p = { kNoInstance, UINT32_MAX, 0.0f };
//             return PathStep::Closest;
//         }
//         __device__ bool accept(Payload& p, uint32_t k, size_t id, float, float, float) const { return !(k == p.inst && id == p.prim); }
//         __device__ PathStep next(size_t i, Payload& p, const bvh_hit3f& hit, uint32_t k, bvh_ray3f& ray) const {
//             if (p.inst != kNoInstance || hit.prim_id == UINT32_MAX) {   // the shadow segment ended, or a primary miss
//                 p.radiance = p.inst != kNoInstance && hit.prim_id == UINT32_MAX ? 1.0f : 0.0f;
//                 return PathStep::End;
//             }
//             p.inst = k; p.prim = hit.prim_id;
//             ray.org = ray.org + hit.t * ray.dir; ray.dir = light - ray.org; ray.tmin = 0.0f; ray.tmax = 1.0f;
//             return PathStep::Occlusion;
//         }
//         __device__ void finish(size_t i, const Payload& p) const { image[i] = p.radiance; }
//     };
//     top.trace_instance_paths<false>(width * height, instances, Paths { ... }, workspace, bytes, stream);
//
// Motion blur: placements that move over the shutter.  A MotionInstance<T> record (make_motion_instance(view, key0,
// key1)) holds a bottom tree as Instance<T> does and two 3 x 4 keys, object_to_world[0] at time 0 and
// object_to_world[1] at time 1, and no inverse; MotionInstances<T> { records, count, max_depth } views them.  A ray at
// time tau sees record k as instance_at(records[k], tau): each coefficient blended linearly, (1 - tau) key0 + tau key1
// rounded step by step with no FMA, tau clamped to [0, 1] (a NaN time as 0), exact at 0 and 1 and wherever the keys
// agree; its world_to_object is prepare_instance's inverse of that (detail::blend_keys, detail::invert_affine).
// prepare_motion_instances(instances, bboxes, centers[, stream]) writes every root index and a world box that holds the
// record's bottom root box at every time of the shutter (the union of the boxes at the two keys, widened for the
// rounding of the blend), for bvhNN_build_boxes / bvhNN_refit_boxes, in one stream-ordered kernel.  A key with a
// non-finite entry gives the empty box; a key without an inverse does not (an object may scale from 0): a ray at a time
// where the placement has no inverse skips the record.  On the top view:
//     top.trace_instances<IsAnyHit, IsRobust, TieLastVisited = false>(n, motion_instances, shader, workspace, bytes[, stream]);
//     top.trace_instance_paths<IsRobust, TieLastVisited = false>(n, motion_instances, shader, workspace, bytes[, stream]);
// take the shaders of the static calls, except that start also gives the ray's (path's) time:
//     Ray      start(size_t i, Payload& p, T& time) const;                     // trace_instances
//     PathStep start(size_t i, Payload& p, Ray& ray, T& time) const;           // trace_instance_paths: for every segment
//   * per ray (segment), the calls are exactly those of the static call on the same top tree with record k replaced by
//     instance_at(records[k], time): the same accept calls (instance, original id, bits of t, u, v), record, instance
//     and, for paths, world ray to next.  With equal keys the motion call is the static call bit for bit at any time;
//   * errors, workspace, streams, n == 0 and the host build are those of the static calls, the errors naming
//     "trace_instances (motion)" or "trace_instance_paths (motion)".  Compiled as plain host C++, each ray runs the
//     nested loop over instance_at;
//   * the time is kept beside the payload in the lane's registers; each instance entry builds the placement (about 60
//     multiplies and adds and 9 divisions).  Linear blending of matrices shrinks an object that turns far within one
//     shutter (a half turn passes through a singular matrix): split such a shutter, or keep the turn small.
// One frame of a renderer (the keys of frame f are the placements at its shutter's open and close):
//
//     struct Shade {
//         struct Payload {};
//         const bvh_ray3f* rays; const float* times; bvh_hit3f* hits; uint32_t* inst;
//         __device__ bvh_ray3f start(size_t i, Payload&, float& time) const { time = times[i]; return rays[i]; }
//         __device__ bool accept(Payload&, uint32_t, size_t, float, float, float) const { return true; }
//         __device__ void finish(size_t i, const Payload&, const bvh_hit3f& h, uint32_t k) const { hits[i] = h; inst[i] = k; }
//     };
//     write_keys<<<...>>>(d_recs, open, close);                       // yours: records[k].object_to_world[0] and [1]
//     const MotionInstances<float> instances { d_recs, count, max_depth };
//     prepare_motion_instances(instances, d_boxes, d_centres, stream);
//     bvh3f_refit_boxes(top_bvh, d_boxes, count, BVH_DEVICE_POINTERS);    // on the top handle's stream
//     top.trace_instances<false, false>(n, instances, Shade { d_rays, d_times, d_hits, d_inst }, workspace, bytes, stream);
//
// Deforming meshes: vertices that move over the shutter (skinning, cloth, a fluid surface).  MotionTriangles<T>
// { vertices[2], count } views two vertex keys in device memory, vertices[0] at time 0 and vertices[1] at time 1, each
// count x 9 values (p0 p1 p2) in original primitive order, the layout bvhNN_build_triangles, bvhNN_set_triangles and
// bvhNN_refit_triangles take; the same pointer twice is a static mesh.  A ray at time tau sees triangle id as
// triangle_at(tris, id, tau, v): each coordinate blended as a motion record's coefficients are (detail::blend_key: tau
// clamped to [0, 1], a NaN time as 0; the key at 0 and 1 and where the keys agree, else (1 - tau) k0 + tau k1 by sub,
// mul, mul, add, never an FMA).  prepare_motion_triangles(tris, bboxes, centers[, stream]) writes, per original id, a box
// that holds triangle_at at every time of the shutter (the union of the key boxes, widened per moving axis for the
// rounding of the blend; exactly tri_bounds_center's box when the keys are equal) and the centre of the triangle at 0.5,
// for bvhNN_build_boxes / bvhNN_refit_boxes, in one stream-ordered kernel.  A key with a non-finite entry gives the empty
// box.  On a view of a tree over those boxes (it needs no attached triangles):
//     view.trace_triangles<IsAnyHit, IsRobust, TieLastVisited = false>(n, motion_tris, shader, workspace, bytes[, stream]);
//     view.trace_paths<IsRobust, TieLastVisited = false>(n, motion_tris, shader, workspace, bytes[, stream]);
// take the shaders of the static calls, except that start also gives the ray's (path's) time:
//     Ray      start(size_t i, Payload& p, T& time) const;                     // trace_triangles
//     PathStep start(size_t i, Payload& p, Ray& ray, T& time) const;           // trace_paths: for every segment
//   * per ray (segment), the calls are exactly those of the static call on the same tree with its triangles replaced by
//     precompute_tri(triangle_at(motion_tris, id, time)): the same accept calls (original id, bits of t, u, v) in the
//     same order, the same record and, for paths, the same next calls.  With equal keys the motion call is the static
//     call bit for bit at any time;
//   * errors, checked on the host before any launch: motion_tris.count other than the tree's prim_count, or a null key
//     pointer, throws std::invalid_argument; a small workspace or a stack beyond 200 KB std::length_error; a failed launch
//     std::runtime_error; the messages name "trace_triangles (motion)" or "trace_paths (motion)".  Streams, the
//     workspace, n == 0, the warp subset and the host build are those of the static calls;
//   * the kernels are the static ones (device_view_triangle_kernel, device_view_path_kernel) under detail::MotionShader,
//     which keeps the time beside the payload; the leaf loads each slot's original id and both keys (72 bytes in float),
//     blends them and runs the library's tri_test on precompute_tri of the result, one triangle at a time.
// One frame of a renderer (INTEGRATION.md §5 has it whole):
//
//     struct Shade {
//         struct Payload {};
//         const bvh_ray3f* rays; const float* times; bvh_hit3f* hits;
//         __device__ bvh_ray3f start(size_t i, Payload&, float& time) const { time = times[i]; return rays[i]; }
//         __device__ bool accept(Payload&, size_t, float, float, float) const { return true; }
//         __device__ void finish(size_t i, const Payload&, const bvh_hit3f& h) const { hits[i] = h; }
//     };
//     skin<<<...>>>(d_key0, d_key1);                                  // yours: the vertices at the shutter's open and close
//     const MotionTriangles<float> mesh { { d_key0, d_key1 }, count };
//     prepare_motion_triangles(mesh, d_boxes, d_centres, stream);
//     bvh3f_refit_boxes(bvh, d_boxes, count, BVH_DEVICE_POINTERS);   // on the handle's stream (first frame: build_boxes)
//     view.trace_triangles<false, false>(n, mesh, Shade { d_rays, d_times, d_hits }, workspace, bytes, stream);
//
// Motion nodes: the shutter boxes above hold each triangle over its whole sweep, so a mesh that moves a few triangle sizes
// per shutter makes every ray test several times as many triangles.  Motion nodes keep the view's topology and give
// each node its box at both keys: MotionNode<T> (per slot of the view's numbering, slot 0 unused: the bounds at key 0
// and key 1 and the view's packed index; 64 bytes in float, 128 in double, so a sibling pair is one aligned 128 / 256-byte
// block) and MotionNodes<T> { nodes, node_count } viewing view.node_count + 1 records in device memory.
// node_at(motion_nodes, slot, time, bounds) is the one definition of a node's box at a time: each bound blended by
// triangle_at's rule (detail::blend_key at detail::shutter_time(time)), so a bound that does not move is the key's own
// bit for bit.  prepare_motion_nodes(view, motion_tris, out, workspace, bytes[, stream]) writes every record in one
// view.traverse_bottom_up pass (workspace: view.bottom_up_workspace_bytes()): a leaf's key k is the union of
// tri_bounds_center's boxes of its finite triangles at key k (refit_from_leaf's fold), widened on an axis on which
// something moves by 4 eps M + the smallest normal number for the rounding of the two blends (triangle_at's and
// node_at's; detail::MotionNodeBuilder states the bound); an inner node's keys are the unions of its children's, and a
// side of it whose keys differ over a child whose keys on that side are equal (a static part beside a moving one) is
// widened by the same rule.  So node_at's box of every node holds triangle_at of every finite triangle of its subtree at
// every time.  With equal keys nothing is widened and both keys are the view's bounds after bvhNN_refit_boxes over
// prepare_motion_triangles' boxes, bit for bit.
// On that view:
//     view.trace_triangles<IsAnyHit, IsRobust, TieLastVisited = false>(n, motion_tris, motion_nodes, shader, workspace, bytes[, stream]);
//     view.trace_paths<IsRobust, TieLastVisited = false>(n, motion_tris, motion_nodes, shader, workspace, bytes[, stream]);
// take the shaders of the motion forms (start also gives the time):
//   * per ray (segment), the calls are exactly those of the motion form on a tree of the same topology whose node boxes
//     are node_at(motion_nodes, slot, time): the same accept calls in the same order, the same record and, for paths,
//     the same next calls.  With equal keys (one pointer twice) the call is the motion form on the shutter-box tree bit
//     for bit, accept sequence included.  With moving keys whose entries are all finite, robust traversal and the
//     canonical tie rule, closest-hit records equal the motion form's on every ray: both trees hold the closest
//     triangle, only the visits differ.  (A triangle with a non-finite key is in neither tree's boxes, but a ray that
//     reaches its leaf for a neighbour tests it, and the two trees reach different leaves.);
//   * the view's node bounds are not read: its indices, prim_ids and depth are (the root index and the stack bound
//     come from the motion nodes and view.depth);
//   * errors, checked on the host before any launch: motion_nodes.node_count other than the view's, a null motion-node
//     pointer, or the motion form's errors throw std::invalid_argument; a small workspace or a stack beyond 200 KB
//     std::length_error; a failed launch std::runtime_error; the messages name "trace_triangles (motion nodes)" or
//     "trace_paths (motion nodes)".  Streams, the workspace, n == 0, the warp subset and the host build are the motion
//     form's; compiled as plain host C++, each ray runs traverse_top_down's loop with the same inner step;
//   * the kernels are the motion forms' (device_view_triangle_kernel, device_view_path_kernel) with the shader wrapped
//     as detail::MotionShader<T, detail::WithMotionNodes<T, Shader>>; the one step that differs is the inner step
//     (detail::motion_inner_step): per child node_at's blend at the lane's time, then node_test's slab arithmetic and
//     descend, unchanged, with float closest-hit rays splitting the fetch as inner_step does (x / y of both keys first,
//     z and the index only for a child its x / y slabs do not reject).
// One frame (the topology built once from the first frame's prepare_motion_triangles boxes):
//
//     skin<<<...>>>(d_key0, d_key1);
//     prepare_motion_nodes(view, mesh, d_motion_nodes, bottom_up, view.bottom_up_workspace_bytes(), stream);
//     view.trace_triangles<false, false>(n, mesh, MotionNodes<float> { d_motion_nodes, view.node_count }, Shade { ... },
//                                        workspace, bytes, stream);
//
// Deforming instances: a scene that mixes static placed meshes with deforming ones (a skinned character among instanced
// set pieces), in one launch.  A DeformingInstance<T> record holds MotionInstance<T>'s fields and a bottom's vertex keys
// and motion nodes; DeformingInstances<T> { records, count, max_depth } views them.  Each record picks its bottom kind
// at run time: vertices[0] == nullptr is a static bottom (the view's tris and node bounds); vertex keys alone are a
// deforming bottom on the view's tree refitted over prepare_motion_triangles' boxes; vertex keys and motion nodes are a
// deforming bottom whose inner steps are motion_inner_step at the ray's time.  make_deforming_instance(view, key0, key1
// [, motion_tris[, motion_nodes]]) fills one on the host (std::invalid_argument for a count other than the view's or a
// null pointer).  prepare_deforming_instances(instances, bboxes, centers[, stream]) writes every root index and a world
// box that holds every finite triangle of the bottom at every time under the placement at that time
// (detail::prepare_deforming_instance states the argument), after each deforming bottom's own step of the frame
// (prepare_motion_triangles + bvhNN_refit_boxes, or prepare_motion_nodes).  On the top view:
//     top.trace_instances<IsAnyHit, IsRobust, TieLastVisited = false>(n, deforming_instances, shader, workspace, bytes[, stream]);
//     top.trace_instance_paths<IsRobust, TieLastVisited = false>(n, deforming_instances, shader, workspace, bytes[, stream]);
// take the motion forms' shaders (start also gives the time):
//   * per ray (segment), the calls are exactly those of the motion forms on the same top tree, except inside a record
//     with a deforming bottom, whose bottom traversal is the motion trace_triangles (shutter boxes) or the motion-node
//     trace_triangles at the ray's time on the object-space ray of instance_at(record, time); leaf ties take the
//     canonical rule on (instance, original id) unless TieLastVisited;
//   * so with static bottoms only the call is the motion trace_instances, one identity record with equal placement keys
//     is the motion (motion-node) trace_triangles / trace_paths on its mesh, and with equal vertex keys a deforming
//     bottom is the static bottom on its tree;
//   * errors, workspace, streams, n == 0 and the host build are the motion forms', the messages naming
//     "trace_instances (deforming)" or "trace_instance_paths (deforming)";
//   * the kernels are the instance kernels with the shader wrapped as detail::MotionShader<T,
//     detail::WithDeformingBottoms<T, Shader>>: an if constexpr on detail::IsDeforming picks, per record, the motion
//     inner step or the plain one and the key leaf (detail::deforming_instance_leaf) or instance_leaf.  The float kernels
//     stay at 56 registers and spill (DESIGN.md section 6).
// One frame (INTEGRATION.md §5 has it whole):
//
//     skin<<<...>>>(d_key0, d_key1);                                   // yours: the character's vertex keys
//     prepare_motion_nodes(character, mesh, d_motion_nodes, bottom_up, character.bottom_up_workspace_bytes(), stream);
//     write_keys<<<...>>>(d_recs, open, close);                        // yours: every record's placement keys
//     prepare_deforming_instances(DeformingInstances<float> { d_recs, count, max_depth }, d_boxes, d_centres, stream);
//     bvh3f_refit_boxes(top_bvh, d_boxes, count, BVH_DEVICE_POINTERS);
//     top.trace_instances<false, false>(n, DeformingInstances<float> { d_recs, count, max_depth }, Shade { ... }, workspace, bytes, stream);
//
// Stacks: anything with push(Index) and try_pop(Index&) (false when empty), empty at the start.  A traversal holds at
// most view.stack_bound() = depth + 1 entries, and no stack checks its capacity on the device: check it on the host
// (DeviceView<T>::from(c, capacity) and bvh::v2::cuda::Accel<T>::device_view(capacity) throw when it is too small).
//   DeviceView<T>::SmallStack<N>   N entries per thread in registers / local memory (the reference's SmallStack);
//   DeviceView<T>::SharedStack     the batched kernels' shared-memory stack: depth + 2 entries per thread, laid out
//                                  [entry][thread] (no bank conflicts); make it with shared_stack(smem, blockDim.x)
//                                  from a dynamic shared array of shared_stack_bytes(blockDim.x) bytes.
#pragma once

#include <bvh_b200_device.h>
#include <cstddef>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "persistent_core.cuh"
#include "refit_core.cuh"
#include "trace_plan.h"
#include "traverse_core.cuh"

namespace bvh::v2::cuda {

// What a path shader of DeviceView::trace_paths asks for next: the path's end, a closest-hit segment or an occlusion
// (any-hit) segment.
enum class PathStep { End, Closest, Occlusion };

// One placed copy of a triangle mesh for DeviceView::trace_instances: the bottom tree's device arrays (from a DeviceView
// with triangles), its root and depth, and the placement.  Fill it with make_instance(view, object_to_world) and keep the
// records in device memory of the caller's.  object_to_world is the caller's; root_index and world_to_object are written
// by prepare_instances (all NaN for a matrix that has no inverse, which trace_instances then skips).
template <typename T> struct alignas(16) Instance {
    const bvhb200::DevNode<T>* nodes;   // the bottom view's nodes, prim_ids (BVH order) and tris (BVH order)
    const uint32_t* prim_ids;
    const bvhb200::DevTri<T>* tris;
    typename bvhb200::Real<T>::UInt root_index;     // the bottom root's index, written by prepare_instances
    uint32_t depth;                     // the bottom tree's depth
    T object_to_world[12];              // 3 x 4 row-major affine: world = A * object + b, row i = A[i][0..2], b[i]
    T world_to_object[12];              // its inverse, same layout
};

// A plain view of `count` instance records in device memory.  max_depth is the largest bottom depth among them: the
// host sizes the shared-memory stack of trace_instances from it.
template <typename T> struct Instances {
    Instance<T>* records = nullptr;
    size_t count = 0;
    size_t max_depth = 0;
};

// One placed copy of a triangle mesh that moves over the shutter, for the motion forms of trace_instances and
// trace_instance_paths: the bottom tree as in Instance<T>, and two placements (keys), object_to_world[0] at time 0 and
// object_to_world[1] at time 1, each 3 x 4 row-major as in Instance<T>.  A ray at time tau sees the record as
// instance_at(record, tau).  Fill it with make_motion_instance(view, key0, key1); root_index is written by
// prepare_motion_instances.  It stores no inverse: the placement at the ray's time is built on every entry.
template <typename T> struct alignas(16) MotionInstance {
    const bvhb200::DevNode<T>* nodes;   // the bottom view's nodes, prim_ids (BVH order) and tris (BVH order)
    const uint32_t* prim_ids;
    const bvhb200::DevTri<T>* tris;
    typename bvhb200::Real<T>::UInt root_index;     // the bottom root's index, written by prepare_motion_instances
    uint32_t depth;                     // the bottom tree's depth
    T object_to_world[2][12];           // the keys at time 0 and time 1, each row i = A[i][0..2], b[i]
};

// A plain view of `count` motion records in device memory; max_depth as in Instances<T>.
template <typename T> struct MotionInstances {
    MotionInstance<T>* records = nullptr;
    size_t count = 0;
    size_t max_depth = 0;
};

// A triangle mesh whose vertices move over the shutter, for the motion forms of trace_triangles and trace_paths: the
// vertices at time 0 (vertices[0]) and at time 1 (vertices[1]), each count x 9 values (p0, p1, p2 of each triangle) in
// original primitive order, as bvhNN_build_triangles, bvhNN_set_triangles and bvhNN_refit_triangles take them, in
// device memory of the caller's.  A ray at time tau sees triangle id as triangle_at(tris, id, tau).  The same pointer
// twice is a static mesh.  The keys are read on the device through the read-only (non-coherent) cache: write them in an
// earlier kernel or copy on the stream, never in the kernel that traces or reads them.
template <typename T> struct MotionTriangles {
    const T* vertices[2] = { nullptr, nullptr };
    size_t count = 0;
};

// The node of a deforming mesh's tree at the two keys, for the motion-node forms of trace_triangles and trace_paths: per
// slot of a DeviceView's numbering (slot = reference index + 1, slot 0 unused) the node's bounds at time 0 and at time
// 1 and its packed index, copied from the view, so that a traversal reads this array alone.  Key k's bounds are
// minx, maxx, miny, maxy = xy[k][0..3] and minz, maxz = z[k][0..1].  64 bytes in float, 128 in double, so that a sibling
// pair (slots 2j, 2j + 1) is one aligned 128 / 256-byte block of an array from cudaMalloc; in float the first 32 bytes
// hold x and y of both keys and the second z of both keys and the index, the halves of the closest-hit step's split load.
// prepare_motion_nodes writes them; node_at gives the box a ray of a given time tests.
template <typename T> struct alignas(16 * sizeof(T)) MotionNode {
    T xy[2][4];                         // key k: minx, maxx, miny, maxy
    T z[2][2];                          // key k: minz, maxz
    typename bvhb200::Real<T>::UInt index;          // the view's packed index of this slot
    typename bvhb200::Real<T>::UInt pad[3];
};
static_assert(sizeof(MotionNode<float>) == 64 && sizeof(MotionNode<double>) == 128, "motion node size");

// A plain view of the node_count + 1 motion nodes of a tree (slot 0 unused) in device memory.
template <typename T> struct MotionNodes {
    const MotionNode<T>* nodes = nullptr;
    size_t node_count = 0;
};

// One placed copy of a mesh in a scene that mixes bottom kinds, for the deforming forms of trace_instances and
// trace_instance_paths: MotionInstance<T>'s fields (the bottom view's arrays, root, depth and the two placement keys,
// in the same layout), then the bottom's vertex keys and motion nodes.  Each record picks its bottom kind:
//   * vertices[0] == nullptr: a static bottom, the view's tris and node bounds, as in MotionInstance<T>;
//   * vertices set, motion_nodes == nullptr: a deforming bottom on shutter boxes, triangle_at(vertices, id, time) under
//     the view's tree (refitted over prepare_motion_triangles' boxes);
//   * both set: a deforming bottom with motion nodes, whose inner steps are motion_inner_step at the ray's time (the
//     view's node bounds are not read).
// vertices[k] is the MotionTriangles<T> layout (count x 9 values in original order).  Fill it with
// make_deforming_instance; root_index is written by prepare_deforming_instances.  160 bytes in float, 256 in double.
template <typename T> struct alignas(16) DeformingInstance {
    const bvhb200::DevNode<T>* nodes;   // the bottom view's nodes, prim_ids (BVH order) and tris (BVH order; static bottoms)
    const uint32_t* prim_ids;
    const bvhb200::DevTri<T>* tris;
    typename bvhb200::Real<T>::UInt root_index;     // the bottom root's index, written by prepare_deforming_instances
    uint32_t depth;                     // the bottom tree's depth
    T object_to_world[2][12];           // the placement keys at time 0 and time 1, as in MotionInstance<T>
    const T* vertices[2];               // the bottom's vertex keys at time 0 and time 1, or nullptr (a static bottom)
    const MotionNode<T>* motion_nodes;  // the bottom's motion nodes (view.node_count + 1 records), or nullptr
};
static_assert(sizeof(DeformingInstance<float>) == 160 && sizeof(DeformingInstance<double>) == 256, "deforming instance size");

// A plain view of `count` deforming-scene records in device memory; max_depth as in Instances<T>.
template <typename T> struct DeformingInstances {
    DeformingInstance<T>* records = nullptr;
    size_t count = 0;
    size_t max_depth = 0;
};

namespace detail {
template <typename T> struct ViewTypes;
template <> struct ViewTypes<float>  {
    using CView = bvh_device_view3f; using Ray = bvh_ray3f; using Hit = bvh_hit3f; using BBox = bvh_bbox3f; using Vec = bvh_vec3f;
};
template <> struct ViewTypes<double> {
    using CView = bvh_device_view3d; using Ray = bvh_ray3d; using Hit = bvh_hit3d; using BBox = bvh_bbox3d; using Vec = bvh_vec3d;
};
struct NoInnerFn { template <typename I> BVH_HD void operator()(I) const {} };
template <typename T, typename Ray> BVH_HD void load_ray(const Ray& ray, bvhb200::RayCtx<T>& r) {
    r.org[0] = ray.org.x; r.org[1] = ray.org.y; r.org[2] = ray.org.z;
    r.dir[0] = ray.dir.x; r.dir[1] = ray.dir.y; r.dir[2] = ray.dir.z;
    r.tmin = ray.tmin; r.tmax = ray.tmax;
}
template <typename Ray, typename T> BVH_HD Ray make_ray(const bvhb200::RayCtx<T>& r) {
    Ray ray;
    ray.org.x = r.org[0]; ray.org.y = r.org[1]; ray.org.z = r.org[2];
    ray.dir.x = r.dir[0]; ray.dir.y = r.dir[1]; ray.dir.z = r.dir[2];
    ray.tmin = r.tmin; ray.tmax = r.tmax;
    return ray;
}
// DeviceView::trace's stack when the header is compiled as host C++
template <typename U> struct VectorStack {
    std::vector<U> elems;
    void push(U v) { elems.push_back(v); }
    bool try_pop(U& out) {
        if (elems.empty()) return false;
        out = elems.back();
        elems.pop_back();
        return true;
    }
};
// A querier's node function bound to one query's payload, as traverse_nodes calls a node test: the three-argument form
// when the querier has node(payload, left, right, left_index), the two-argument one otherwise.
template <typename Querier, typename Payload, typename Node, typename = void> struct TakesLeftIndex : std::false_type {};
template <typename Querier, typename Payload, typename Node>
struct TakesLeftIndex<Querier, Payload, Node, std::void_t<decltype(std::declval<const Querier&>().node(
    std::declval<Payload&>(), std::declval<const Node&>(), std::declval<const Node&>(), size_t(0)))>> : std::true_type {};
template <typename Querier, typename Payload, typename Node, bool = TakesLeftIndex<Querier, Payload, Node>::value>
struct BoundNode {
    const Querier& q;
    Payload& p;
    BVH_HD decltype(auto) operator()(const Node& l, const Node& r) const { return q.node(p, l, r); }
};
template <typename Querier, typename Payload, typename Node> struct BoundNode<Querier, Payload, Node, true> {
    const Querier& q;
    Payload& p;
    BVH_HD decltype(auto) operator()(const Node& l, const Node& r, size_t left) const { return q.node(p, l, r, left); }
};
// The library's hit record as the C ABI reports it
template <typename T> BVH_HD typename ViewTypes<T>::Hit make_hit(const bvhb200::DevHit<T>& rec) {
    typename ViewTypes<T>::Hit hit;
    hit.prim_id = rec.prim_id; hit.t = rec.t; hit.u = rec.u; hit.v = rec.v;
    return hit;
}
// The shader the motion forms of trace_triangles, trace_paths, trace_instances and trace_instance_paths run: the
// caller's, with the ray's time kept beside its payload (so in the lane's registers) from start on; defined below.
template <typename T, typename Shader> struct MotionShader;
// The triangle source of a shader: the tree's BVH-order triangles, or the keys of MotionTriangles<T> under a MotionShader.
template <typename T, typename Shader> struct TrianglesOf { using type = const bvhb200::DevTri<T>*; };
template <typename T, typename Shader> struct TrianglesOf<T, MotionShader<T, Shader>> { using type = MotionTriangles<T>; };

// What the kernel of DeviceView::trace_triangles reads besides the nodes: the caller's shader and the triangles.
template <typename T, typename Shader> struct TriangleShader {
    Shader shader;
    typename TrianglesOf<T, Shader>::type tris;     // BVH order; for motion, the keys in original order
    const uint32_t* prim_ids;
};
// The triangle leaf of DeviceView::trace_triangles (both builds): the library's leaf_range over [first, first + count)
// with the shader's accept as tri_test's filter, which receives the original id.
template <typename T, bool TieLastVisited, typename Shader, typename Payload>
BVH_HD void shader_leaf(const TriangleShader<T, Shader>& ts, Payload& payload, uint32_t first, uint32_t count,
                        bvhb200::RayCtx<T>& r, bvhb200::HitState<T>& hit) {
    bvhb200::leaf_range<T>(ts.tris, ts.prim_ids, !TieLastVisited, first, count, r, hit, nullptr,
                           [&](uint32_t slot, T t, T u, T v) {
                               return static_cast<bool>(ts.shader.accept(payload, static_cast<size_t>(ts.prim_ids[slot]), t, u, v));
                           });
}
// The caller's shader of the deforming forms of trace_instances and trace_instance_paths; defined below.
template <typename T, typename Shader> struct WithDeformingBottoms;
// The record kind of a shader: Instance<T>, MotionInstance<T> under a MotionShader, or DeformingInstance<T> under a
// MotionShader of WithDeformingBottoms.
template <typename T, typename Shader> struct RecordOf { using type = Instance<T>; };
template <typename T, typename Shader> struct RecordOf<T, MotionShader<T, Shader>> { using type = MotionInstance<T>; };
template <typename T, typename Shader> struct RecordOf<T, MotionShader<T, WithDeformingBottoms<T, Shader>>> {
    using type = DeformingInstance<T>;
};

// What the kernel of DeviceView::trace_instances reads besides the top tree's nodes: the caller's shader, the instance
// records and the top tree's prim_ids (BVH-order slot -> record).
template <typename T, typename Shader> struct InstanceShader {
    Shader shader;
    const typename RecordOf<T, Shader>::type* records;
    const uint32_t* prim_ids;
};
// The instance trace_instances reports for a miss
constexpr uint32_t kNoInstance = 0xFFFFFFFFu;
// The stack entry below an instance's bottom traversal: a leaf of 14 primitives at the last representable position,
// which no tree has (kTraversalDone is the one of 15), so the inner loops stop on it as on a leaf.
template <typename U> constexpr U kInstanceMarker = bvhb200::kTraversalDone<U> - 1;
// Stack entries an instance visit adds to the two trees' own: the rest of the top leaf, the world ray's origin and
// direction (6), the marker, and the bottom traversal's one entry beyond its depth.
constexpr size_t kInstanceStackExtra = 9;

// Row `row` of a 3 x 4 affine map (row[3] the translation) applied to a point (with the translation) or a vector
// (without).  The sum starts from -0, the identity of IEEE addition, and skips terms whose coefficient is 0, so a
// coordinate mapped by an identity, permutation or power-of-two-scale row keeps its exact bits (signed zeros included).
template <typename T> BVH_HD T affine_row(const T* row, const T p[3], bool point) {
    using R = bvhb200::Real<T>;
    T acc = R::neg(T(0));
    for (int j = 0; j < 3; ++j)
        if (row[j] != T(0)) acc = R::add(acc, R::mul(row[j], p[j]));
    if (point && row[3] != T(0)) acc = R::add(acc, row[3]);
    return acc;
}
// The object-space ray of an instance (both builds): the world origin as a point and the direction as a vector through
// world_to_object, tmin and tmax unchanged, so t keeps its meaning.  `obj` may be `world`.
template <typename T> BVH_HD void object_ray(const T* world_to_object, const bvhb200::RayCtx<T>& world, bvhb200::RayCtx<T>& obj) {
    T org[3], dir[3];
    for (int i = 0; i < 3; ++i) {
        org[i] = affine_row(world_to_object + 4 * i, world.org, true);
        dir[i] = affine_row(world_to_object + 4 * i, world.dir, false);
    }
    for (int i = 0; i < 3; ++i) { obj.org[i] = org[i]; obj.dir[i] = dir[i]; }
    obj.tmin = world.tmin; obj.tmax = world.tmax;
}
// An instance trace_instances skips: prepare_instances found no inverse (its world_to_object is NaN)
template <typename T> BVH_HD bool instance_is_singular(const T* world_to_object) { return world_to_object[0] != world_to_object[0]; }

// The inverse of the 3 x 4 affine map m (both builds) into inv: the adjugate of A over its determinant, then
// -(A^-1 b); all NaN, and false, when an entry of m is not finite, the determinant is 0 or not finite, or an entry of
// the inverse is not finite.  prepare_instance's world_to_object, and the placement of a motion record at a time.
template <typename T> BVH_HD bool invert_affine(const T* m, T* out) {
    using R = bvhb200::Real<T>;
    using UI = typename R::UInt;
    const T nan = R::from_bits(~(UI)0 >> 1);
    bool ok = true;
    for (int k = 0; k < 12; ++k) ok = ok && R::is_finite(m[k]);
    const T a[3][3] = { { m[0], m[1], m[2] }, { m[4], m[5], m[6] }, { m[8], m[9], m[10] } };
    T c[3][3];                          // cofactors
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
            c[i][j] = R::sub(R::mul(a[i1][j1], a[i2][j2]), R::mul(a[i1][j2], a[i2][j1]));
        }
    const T det = bvhb200::dot3(a[0], c[0]);
    ok = ok && det != T(0) && R::is_finite(det);
    T inv[12];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) inv[4 * i + j] = R::div(c[j][i], det);
    const T b[3] = { m[3], m[7], m[11] };
    for (int i = 0; i < 3; ++i) inv[4 * i + 3] = R::neg(affine_row(inv + 4 * i, b, false));
    for (int k = 0; k < 12; ++k) ok = ok && R::is_finite(inv[k]);
    for (int k = 0; k < 12; ++k) out[k] = ok ? inv[k] : nan;
    return ok;
}

// Axis i of the world box of the root box rb (minx, maxx, miny, maxy, minz, maxz) under the 3 x 4 map m (both builds):
// b_i plus the sums of min / max(a_ij lo_j, a_ij hi_j), which in exact arithmetic is the box of the eight transformed
// corners.  Its rounding error is below 2.5 eps S_i, S_i = |b_i| + sum_j |a_ij| max(|lo_j|, |hi_j|) (returned in s), so
// each side is moved out by 4 eps S_i + the smallest normal number (for underflow): [lo, hi] contains the exact image of
// the root box.  An overflow to NaN gives the whole axis on that side.
template <typename T> BVH_HD void world_box_axis(const T* m, const T* rb, int i, T& lo, T& hi, T& s) {
    using R = bvhb200::Real<T>;
    using UI = typename R::UInt;
    const T inf = R::from_bits(sizeof(T) == 4 ? (UI)0x7F800000u : (UI)0x7FF0000000000000ull);
    const T pad = R::mul(R::eps(), T(4)), tiny = sizeof(T) == 4 ? (T)FLT_MIN : (T)DBL_MIN;
    T l = m[4 * i + 3], h = m[4 * i + 3];
    s = R::abs(m[4 * i + 3]);
    for (int j = 0; j < 3; ++j) {
        const T p = R::mul(m[4 * i + j], rb[2 * j]), q = R::mul(m[4 * i + j], rb[2 * j + 1]);
        l = R::add(l, p < q ? p : q);
        h = R::add(h, p < q ? q : p);
        const T e = R::abs(rb[2 * j]) < R::abs(rb[2 * j + 1]) ? R::abs(rb[2 * j + 1]) : R::abs(rb[2 * j]);
        s = R::add(s, R::mul(R::abs(m[4 * i + j]), e));
    }
    const T d = R::add(R::mul(s, pad), tiny);
    lo = R::sub(l, d);
    hi = R::add(h, d);
    if (lo != lo) lo = R::neg(inf);     // (an overflow: the whole axis)
    if (hi != hi) hi = inf;
}

// prepare_instances for one record (both builds).  root_index: the bottom root's.  world_to_object: invert_affine of
// object_to_world.  The box: world_box_axis of the bottom root box, which contains the exact image of the root box; an
// empty box (min = +inf, max = -inf) and a zero centre for a matrix without an inverse.
template <typename T>
BVH_HD void prepare_instance(Instance<T>& rec, typename ViewTypes<T>::BBox& box, typename ViewTypes<T>::Vec& centre) {
    using R = bvhb200::Real<T>;
    using UI = typename R::UInt;
    const T inf = R::from_bits(sizeof(T) == 4 ? (UI)0x7F800000u : (UI)0x7FF0000000000000ull);
    const T* m = rec.object_to_world;
    const bool ok = invert_affine(m, rec.world_to_object);
    rec.root_index = rec.nodes[1].index;
    const T* rb = rec.nodes[1].bounds;  // the bottom root box: minx, maxx, miny, maxy, minz, maxz
    T lo[3], hi[3], mid[3];
    for (int i = 0; i < 3; ++i) {
        T s;
        world_box_axis(m, rb, i, lo[i], hi[i], s);
        mid[i] = R::mul(R::add(lo[i], hi[i]), T(0.5));
        if (!R::is_finite(mid[i])) mid[i] = T(0);
        if (!ok) { lo[i] = inf; hi[i] = R::neg(inf); mid[i] = T(0); }
    }
    box.min.x = lo[0]; box.min.y = lo[1]; box.min.z = lo[2];
    box.max.x = hi[0]; box.max.y = hi[1]; box.max.z = hi[2];
    centre.x = mid[0]; centre.y = mid[1]; centre.z = mid[2];
}

// The linear blend of two keys, the one rule of every motion form (blend_keys, triangle_at).  shutter_time is the time
// clamped to [0, 1], a NaN time counting as 0; blend_key of one value, with tau = shutter_time(time) and rest = 1 - tau,
// is k0 at tau == 0, k1 at tau == 1, k0 where the keys agree, and otherwise (1 - tau) k0 + tau k1 rounded step by step
// (sub, mul, mul, add; never an FMA).  The endpoints and every value that does not move are exact.
template <typename T> BVH_HD T shutter_time(T time) { return time > T(0) ? (time < T(1) ? time : T(1)) : T(0); }  // (NaN: 0)
template <typename T> BVH_HD T blend_key(T k0, T k1, T tau, T rest) {
    using R = bvhb200::Real<T>;
    return tau == T(0) ? k0 : tau == T(1) ? k1 : k0 == k1 ? k0 : R::add(R::mul(rest, k0), R::mul(tau, k1));
}
// The placement of a motion record at `time` (both builds; instance_at is its public form): blend_key of each coefficient.
template <typename T> BVH_HD void blend_keys(const T (&keys)[2][12], T time, T* m) {
    using R = bvhb200::Real<T>;
    const T tau = shutter_time(time);
    const T rest = R::sub(T(1), tau);
    for (int k = 0; k < 12; ++k) m[k] = blend_key(keys[0][k], keys[1][k], tau, rest);
}
// A key of a motion triangle, read once per use (on the device through the read-only cache)
template <typename T> BVH_HD T load_key(const T* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}

// The halves of a motion node, read through the read-only cache on the device: x and y of both keys (the first 32 bytes
// in float, two 128-bit loads), and z of both keys with the index (one 128-bit load and one 32-bit load in float).
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ void load_motion_xy(const MotionNode<float>* p, float (&xy)[2][4]) {
    const float4* q = reinterpret_cast<const float4*>(p);
    const float4 a = __ldg(q), b = __ldg(q + 1);
    xy[0][0] = a.x; xy[0][1] = a.y; xy[0][2] = a.z; xy[0][3] = a.w;
    xy[1][0] = b.x; xy[1][1] = b.y; xy[1][2] = b.z; xy[1][3] = b.w;
}
__device__ __forceinline__ void load_motion_z(const MotionNode<float>* p, float (&z)[2][2], uint32_t& index) {
    const float4 c = __ldg(reinterpret_cast<const float4*>(p) + 2);
    z[0][0] = c.x; z[0][1] = c.y; z[1][0] = c.z; z[1][1] = c.w;
    index = __ldg(&p->index);
}
__device__ __forceinline__ void load_motion_xy(const MotionNode<double>* p, double (&xy)[2][4]) {
    const double2* q = reinterpret_cast<const double2*>(p);
    #pragma unroll
    for (int k = 0; k < 4; ++k) {
        const double2 a = __ldg(q + k);
        xy[k / 2][2 * (k % 2)] = a.x; xy[k / 2][2 * (k % 2) + 1] = a.y;
    }
}
__device__ __forceinline__ void load_motion_z(const MotionNode<double>* p, double (&z)[2][2], uint64_t& index) {
    const double2* q = reinterpret_cast<const double2*>(p) + 4;
    const double2 a = __ldg(q), b = __ldg(q + 1);
    z[0][0] = a.x; z[0][1] = a.y; z[1][0] = b.x; z[1][1] = b.y;
    index = (uint64_t)__ldg(reinterpret_cast<const unsigned long long*>(&p->index));
}
#else
template <typename T> inline void load_motion_xy(const MotionNode<T>* p, T (&xy)[2][4]) {
    for (int k = 0; k < 2; ++k)
        for (int q = 0; q < 4; ++q) xy[k][q] = p->xy[k][q];
}
template <typename T> inline void load_motion_z(const MotionNode<T>* p, T (&z)[2][2], typename bvhb200::Real<T>::UInt& index) {
    for (int k = 0; k < 2; ++k) { z[k][0] = p->z[k][0]; z[k][1] = p->z[k][1]; }
    index = p->index;
}
#endif
// The bounds of the motion node at p blended to (tau, rest) by blend_key: x and y into b[0..3], z into b[4..5] (and the
// node's index).  node_at and the inner step of the motion-node forms both blend through these.
template <typename T> BVH_HD void blend_node_xy(const MotionNode<T>* p, T tau, T rest, T* b) {
    T xy[2][4];
    load_motion_xy(p, xy);
    for (int q = 0; q < 4; ++q) b[q] = blend_key(xy[0][q], xy[1][q], tau, rest);
}
template <typename T>
BVH_HD void blend_node_z(const MotionNode<T>* p, T tau, T rest, T* b, typename bvhb200::Real<T>::UInt& index) {
    T z[2][2];
    load_motion_z(p, z, index);
    b[4] = blend_key(z[0][0], z[1][0], tau, rest);
    b[5] = blend_key(z[0][1], z[1][1], tau, rest);
}
}

// Triangle `id` of a deforming mesh at `time` (both builds), its three vertices p0, p1, p2 into v: each coordinate
// blended from the two keys by the rule of the motion forms (detail::blend_key: time clamped to [0, 1], a NaN time as 0;
// exact at 0 and 1 and for coordinates that do not move).  The motion forms of trace_triangles and trace_paths test a
// ray of that time against precompute_tri of exactly these values; a shader may call it too (a normal at the ray's
// time).  On the device it reads the keys through the read-only (non-coherent) cache (__ldg), so the keys must not be
// written by the kernel that calls it: write them in an earlier kernel or copy on the stream.
template <typename T> BVH_HD void triangle_at(const MotionTriangles<T>& tris, size_t id, T time, T v[9]) {
    using R = bvhb200::Real<T>;
    const T tau = detail::shutter_time(time);
    const T rest = R::sub(T(1), tau);
    const T* k0 = tris.vertices[0] + 9 * id;
    const T* k1 = tris.vertices[1] + 9 * id;
    for (int k = 0; k < 9; ++k) v[k] = detail::blend_key(detail::load_key(k0 + k), detail::load_key(k1 + k), tau, rest);
}

// The box of motion node `slot` at `time` (both builds), minx, maxx, miny, maxy, minz, maxz into bounds: each bound
// blended from the node's two keys by triangle_at's rule (detail::blend_key with tau = detail::shutter_time(time): time
// clamped to [0, 1], a NaN time as 0; exact at 0 and 1 and for bounds whose keys agree, so a bound that does not move is
// the key's own bit for bit).  The motion-node forms of trace_triangles and trace_paths test a ray of that time against
// exactly this box with the library's slab test.  On the device it reads the node through the read-only cache.
template <typename T> BVH_HD void node_at(const MotionNodes<T>& motion_nodes, size_t slot, T time, T bounds[6]) {
    using R = bvhb200::Real<T>;
    const T tau = detail::shutter_time(time);
    const T rest = R::sub(T(1), tau);
    typename R::UInt index;
    detail::blend_node_xy(motion_nodes.nodes + slot, tau, rest, bounds);
    detail::blend_node_z(motion_nodes.nodes + slot, tau, rest, bounds, index);
}

namespace detail {
// prepare_motion_triangles for triangle `id` (both builds).  The box holds triangle_at(tris, id, tau) at every tau of
// the shutter:
//   * in exact arithmetic each coordinate (1 - tau) k0 + tau k1 lies between its two keys, so the triangle lies in the
//     union of tri_bounds_center's boxes at the two keys;
//   * blend_key rounds a moving coordinate three times (1 - tau, the two products, the sum: the first is exact for
//     tau >= 1/2), so it is within 1.5 eps max(|k0|, |k1|) (1 + O(eps)) of the exact blend, and within 1.5 eps M_a
//     (1 + O(eps)) on axis a, M_a = max(|lo_a|, |hi_a|) of the union;
//   * so each side of an axis on which some coordinate moves is moved out by 3 eps M_a + the smallest normal number
//     (for underflow): the rounding of that widening takes at most eps/2 (M_a + the widening) back.
// An axis on which no coordinate moves is the keys' own (blend_key gives the shared value), so with equal keys the box
// is tri_bounds_center's bit for bit.  The centre is tri_bounds_center's of triangle_at at 0.5 (with equal keys, the
// static centre).  A key with a non-finite entry gives the empty box and a zero centre: no ray reaches the triangle.
template <typename T>
BVH_HD void prepare_motion_triangle(const MotionTriangles<T>& tris, size_t id, typename ViewTypes<T>::BBox& box,
                                    typename ViewTypes<T>::Vec& centre) {
    using R = bvhb200::Real<T>;
    using UI = typename R::UInt;
    const T inf = R::from_bits(sizeof(T) == 4 ? (UI)0x7F800000u : (UI)0x7FF0000000000000ull);
    const T pad = R::mul(R::eps(), T(3)), tiny = sizeof(T) == 4 ? (T)FLT_MIN : (T)DBL_MIN;
    T v0[9], v1[9], vm[9];
    bool ok = true;
    for (int k = 0; k < 9; ++k) {
        v0[k] = load_key(tris.vertices[0] + 9 * id + k);
        v1[k] = load_key(tris.vertices[1] + 9 * id + k);
        ok = ok && R::is_finite(v0[k]) && R::is_finite(v1[k]);
    }
    const T half = T(0.5), rest = R::sub(T(1), half);                     // triangle_at(tris, id, 0.5), from v0 and v1
    for (int k = 0; k < 9; ++k) vm[k] = blend_key(v0[k], v1[k], half, rest);
    T lo0[3], hi0[3], c0[3], lo1[3], hi1[3], c1[3], lom[3], him[3], lo[3], hi[3], mid[3];
    bvhb200::tri_bounds_center(v0, lo0, hi0, c0);
    bvhb200::tri_bounds_center(v1, lo1, hi1, c1);
    bvhb200::tri_bounds_center(vm, lom, him, mid);
    for (int a = 0; a < 3; ++a) {
        lo[a] = lo1[a] < lo0[a] ? lo1[a] : lo0[a];
        hi[a] = hi0[a] < hi1[a] ? hi1[a] : hi0[a];
        const bool moves = v0[a] != v1[a] || v0[3 + a] != v1[3 + a] || v0[6 + a] != v1[6 + a];
        if (moves) {
            const T m = R::abs(lo[a]) < R::abs(hi[a]) ? R::abs(hi[a]) : R::abs(lo[a]);
            const T d = R::add(R::mul(m, pad), tiny);
            lo[a] = R::sub(lo[a], d);
            hi[a] = R::add(hi[a], d);
        }
        if (!ok) { lo[a] = inf; hi[a] = R::neg(inf); mid[a] = T(0); }
    }
    box.min.x = lo[0]; box.min.y = lo[1]; box.min.z = lo[2];
    box.max.x = hi[0]; box.max.y = hi[1]; box.max.z = hi[2];
    centre.x = mid[0]; centre.y = mid[1]; centre.z = mid[2];
}

// A sibling's motion node was written by another thread (another SM on the device): read it through L2, as
// refit_load_child reads a refitted node.
template <typename T> BVH_HD MotionNode<T> load_motion_child(const MotionNode<T>* p) {
#if defined(__CUDA_ARCH__)
    MotionNode<T> out;
    const uint4* s = reinterpret_cast<const uint4*>(p);
    uint4* d = reinterpret_cast<uint4*>(&out);
    #pragma unroll
    for (int k = 0; k < (int)(sizeof(MotionNode<T>) / 16); ++k) d[k] = __ldcg(s + k);
    return out;
#else
    return *p;
#endif
}

// prepare_motion_nodes' leaf and inner functions for DeviceView::traverse_bottom_up (both builds): motion node `node`
// (a reference index; its record is out[node + 1]) from the two vertex keys.
//   * leaf: per key, the union of tri_bounds_center's boxes of the leaf's triangles at that key, in BVH order, with
//     robust_min / robust_max from +-max (refit_from_leaf's fold, so with equal keys both keys are the refitted bounds
//     of prepare_motion_triangles' boxes bit for bit).  A triangle with a non-finite key adds nothing to either key;
//   * then each side of an axis on which some coordinate of the leaf's triangles moves is moved out, at both keys, by
//     d = 4 eps M + the smallest normal number, M the largest magnitude of the axis' four unwidened bounds;
//   * inner: per key, the union of its children's records (left first, as refit_from_leaf), read through L2; then a side
//     whose two keys differ while a child's two keys on it are equal is moved out at both keys by d, M now the largest
//     magnitude of the node's four bounds on that axis;
//   * the index is the view's; a node that holds nothing keeps +-max at both keys, which node_at returns exactly and
//     the slab test misses at every time.
// Why node_at(node, tau) holds triangle_at of every finite triangle of the subtree (the lower side of an axis; the upper
// is symmetric).  node_at and triangle_at blend with the same weights tau and rest = fl(1 - tau), both >= 0, and each
// blend_key of keys k0, k1 is within eps (rest |k0| + tau |k1|) (1 + O(eps)) of the exact weighted sum rest k0 + tau k1
// (two products and a sum, each within eps/2; the exact branches within eps/2 |k|, as rest + tau is within eps/2 of 1).
// So a node bound P blends to at most G(P) = rest F(P0) + tau F(P1) and a coordinate c to at least
// rest F-(c0) + tau F-(c1), F(x) = x + eps |x| (1 + O(eps)) and F-(x) = x - eps |x| (1 + O(eps)) both increasing: a node
// bound further out only moves its bound on the blend further out.  Each node side keeps one of two invariants:
//   (E) its two keys are equal: node_at returns the key P exactly.  A coordinate that does not move blends to itself,
//       and lies at or inside P.  One that moves lies in a widened leaf, d inside P at both keys, and its blend loses at
//       most eps M (1 + O(eps)) of that;
//   (W) its keys differ, and every coordinate of the subtree lies at least a widening d (of a node at or below this
//       one, whose M is at least the coordinate's magnitude or whose bound is further out by more than the excess) inside
//       the node's bound at both keys.  A leaf whose keys differ has a moving axis, so it was widened.  An inner node
//       keeps (W) from a child that has it (its own bound is the union, further out), and takes it from a child with
//       equal keys by its own widening: without that, rest P + tau (P - e) for a static coordinate P of that child can
//       round to one ulp beyond P when rest + tau > 1.
//   Under (W) the two blends lose at most 2 eps M + eps d and the rounding of the widened bound takes back at most
//   eps/2 (M + d): 2.5 eps M + 1.5 eps d < d.  (The 3 eps M of prepare_motion_triangle covers one rounded blend, not two.)
// With equal keys nothing moves, no side is widened, and every record is the refitted bound bit for bit.  A bound is
// widened once per level at most where static and moving parts of the mesh meet under it, so at most depth x d.
template <typename T> struct MotionNodeBuilder {
    const bvhb200::DevNode<T>* nodes;   // the view's nodes: only their packed indices are read
    const uint32_t* prim_ids;
    MotionTriangles<T> tris;
    MotionNode<T>* out;

    BVH_HD void operator()(size_t node, size_t begin, size_t end) const {
        using R = bvhb200::Real<T>;
        const T pad = R::mul(R::eps(), T(4)), tiny = sizeof(T) == 4 ? (T)FLT_MIN : (T)DBL_MIN;
        T lo[2][3], hi[2][3];
        bool moves[3] = { false, false, false };
        for (int k = 0; k < 2; ++k)
            for (int a = 0; a < 3; ++a) { lo[k][a] = R::max(); hi[k][a] = R::neg(R::max()); }
        for (size_t slot = begin; slot < end; ++slot) {
            const size_t id = prim_ids[slot];
            T v[2][9];
            bool ok = true;
            for (int q = 0; q < 9; ++q) {
                v[0][q] = load_key(tris.vertices[0] + 9 * id + q);
                v[1][q] = load_key(tris.vertices[1] + 9 * id + q);
                ok = ok && R::is_finite(v[0][q]) && R::is_finite(v[1][q]);
            }
            if (!ok) continue;
            for (int k = 0; k < 2; ++k) {
                T bmin[3], bmax[3], c[3];
                bvhb200::tri_bounds_center(v[k], bmin, bmax, c);
                for (int a = 0; a < 3; ++a) {
                    lo[k][a] = bvhb200::robust_min(lo[k][a], bmin[a]);
                    hi[k][a] = bvhb200::robust_max(hi[k][a], bmax[a]);
                }
            }
            for (int a = 0; a < 3; ++a)
                moves[a] = moves[a] || v[0][a] != v[1][a] || v[0][3 + a] != v[1][3 + a] || v[0][6 + a] != v[1][6 + a];
        }
        for (int a = 0; a < 3; ++a) {
            if (!moves[a]) continue;
            T m = T(0);
            for (int k = 0; k < 2; ++k) {
                m = m < R::abs(lo[k][a]) ? R::abs(lo[k][a]) : m;
                m = m < R::abs(hi[k][a]) ? R::abs(hi[k][a]) : m;
            }
            const T d = R::add(R::mul(m, pad), tiny);
            for (int k = 0; k < 2; ++k) { lo[k][a] = R::sub(lo[k][a], d); hi[k][a] = R::add(hi[k][a], d); }
        }
        write(node, lo, hi);
    }

    BVH_HD void operator()(size_t node, size_t left) const {
        const MotionNode<T> l = load_motion_child(out + left + 1), r = load_motion_child(out + left + 2);
        T lo[2][3], hi[2][3];
        for (int k = 0; k < 2; ++k) {
            for (int a = 0; a < 2; ++a) {
                lo[k][a] = bvhb200::robust_min(l.xy[k][2 * a], r.xy[k][2 * a]);
                hi[k][a] = bvhb200::robust_max(l.xy[k][2 * a + 1], r.xy[k][2 * a + 1]);
            }
            lo[k][2] = bvhb200::robust_min(l.z[k][0], r.z[k][0]);
            hi[k][2] = bvhb200::robust_max(l.z[k][1], r.z[k][1]);
        }
        // a side whose keys differ over a child side whose keys are equal (a part that does not move): moved out by d
        using R = bvhb200::Real<T>;
        const T pad = R::mul(R::eps(), T(4)), tiny = sizeof(T) == 4 ? (T)FLT_MIN : (T)DBL_MIN;
        auto side = [](const MotionNode<T>& c, int k, int a, int hi_side) {
            return a < 2 ? c.xy[k][2 * a + hi_side] : c.z[k][hi_side];
        };
        for (int a = 0; a < 3; ++a) {
            bool widen[2];
            for (int h = 0; h < 2; ++h) {
                const T* key = h ? &hi[0][a] : &lo[0][a];           // key k at key[3 k]
                widen[h] = key[0] != key[3] && (side(l, 0, a, h) == side(l, 1, a, h) || side(r, 0, a, h) == side(r, 1, a, h));
            }
            if (!widen[0] && !widen[1]) continue;
            T m = T(0);
            for (int k = 0; k < 2; ++k) {
                m = m < R::abs(lo[k][a]) ? R::abs(lo[k][a]) : m;
                m = m < R::abs(hi[k][a]) ? R::abs(hi[k][a]) : m;
            }
            const T d = R::add(R::mul(m, pad), tiny);
            for (int k = 0; k < 2; ++k) {
                if (widen[0]) lo[k][a] = R::sub(lo[k][a], d);
                if (widen[1]) hi[k][a] = R::add(hi[k][a], d);
            }
        }
        write(node, lo, hi);
    }

    BVH_HD void write(size_t node, const T (&lo)[2][3], const T (&hi)[2][3]) const {
        MotionNode<T> o;
        for (int k = 0; k < 2; ++k) {
            for (int a = 0; a < 2; ++a) { o.xy[k][2 * a] = lo[k][a]; o.xy[k][2 * a + 1] = hi[k][a]; }
            o.z[k][0] = lo[k][2]; o.z[k][1] = hi[k][2];
        }
        o.index = nodes[node + 1].index;
        o.pad[0] = o.pad[1] = o.pad[2] = 0;
        out[node + 1] = o;
    }
};

// prepare_motion_instances for one record (both builds).  root_index: the bottom root's.  The box holds the bottom
// root box at every time of the shutter, under the placement blend_keys computes:
//   * in exact arithmetic, the image of a point p under (1 - tau) M0 + tau M1 is the convex combination
//     (1 - tau) M0 p + tau M1 p of its images under the keys, so it lies in the union of world_box_axis' box at each
//     key (each contains the exact image of the root box, whether or not the key has an inverse);
//   * blend_keys rounds each moving coefficient three times (1 - tau, the two products, the sum: the first is exact
//     for tau >= 1/2), so it is within 1.5 eps max(|k0|, |k1|) (1 + O(eps)) of the exact blend, and the image of a
//     root-box point moves by at most 1.5 eps (S0_i + S1_i) (1 + O(eps)), with S0_i, S1_i world_box_axis' S_i at
//     the keys;
//   * so each side of the union is moved out by a further 3 eps (S0_i + S1_i) + the smallest normal number: the
//     margin beyond 1.5 eps covers the rounding of that widening (at most eps/2 of a bound below S0_i + S1_i).
// A key with a non-finite entry gives the empty box and a zero centre: no ray reaches the record.
// (shutter_keys_finite and shutter_world_box, `ok` its result, are that box; prepare_deforming_instance uses them too.
// The root index is written between them, in the order this function always had.)
template <typename T> BVH_HD bool shutter_keys_finite(const T (&keys)[2][12]);
template <typename T>
BVH_HD void shutter_world_box(const T (&keys)[2][12], const T* rb, bool ok, typename ViewTypes<T>::BBox& box, typename ViewTypes<T>::Vec& centre);
template <typename T>
BVH_HD void prepare_motion_instance(MotionInstance<T>& rec, typename ViewTypes<T>::BBox& box, typename ViewTypes<T>::Vec& centre) {
    const bool ok = shutter_keys_finite(rec.object_to_world);
    rec.root_index = rec.nodes[1].index;
    shutter_world_box(rec.object_to_world, rec.nodes[1].bounds, ok, box, centre);
}
template <typename T> BVH_HD bool shutter_keys_finite(const T (&keys)[2][12]) {
    using R = bvhb200::Real<T>;
    bool ok = true;
    for (int k = 0; k < 12; ++k) ok = ok && R::is_finite(keys[0][k]) && R::is_finite(keys[1][k]);
    return ok;
}
template <typename T>
BVH_HD void shutter_world_box(const T (&keys)[2][12], const T* rb, bool ok, typename ViewTypes<T>::BBox& box, typename ViewTypes<T>::Vec& centre) {
    using R = bvhb200::Real<T>;
    using UI = typename R::UInt;
    const T inf = R::from_bits(sizeof(T) == 4 ? (UI)0x7F800000u : (UI)0x7FF0000000000000ull);
    const T pad = R::mul(R::eps(), T(3)), tiny = sizeof(T) == 4 ? (T)FLT_MIN : (T)DBL_MIN;
    T lo[3], hi[3], mid[3];
    for (int i = 0; i < 3; ++i) {
        T lo0, hi0, s0, lo1, hi1, s1;
        world_box_axis(keys[0], rb, i, lo0, hi0, s0);
        world_box_axis(keys[1], rb, i, lo1, hi1, s1);
        const T d = R::add(R::mul(R::add(s0, s1), pad), tiny);
        lo[i] = R::sub(lo1 < lo0 ? lo1 : lo0, d);
        hi[i] = R::add(hi0 < hi1 ? hi1 : hi0, d);
        if (lo[i] != lo[i]) lo[i] = R::neg(inf);
        if (hi[i] != hi[i]) hi[i] = inf;
        mid[i] = R::mul(R::add(lo[i], hi[i]), T(0.5));
        if (!R::is_finite(mid[i])) mid[i] = T(0);
        if (!ok) { lo[i] = inf; hi[i] = R::neg(inf); mid[i] = T(0); }
    }
    box.min.x = lo[0]; box.min.y = lo[1]; box.min.z = lo[2];
    box.max.x = hi[0]; box.max.y = hi[1]; box.max.z = hi[2];
    centre.x = mid[0]; centre.y = mid[1]; centre.z = mid[2];
}

// prepare_deforming_instances for one record (both builds): prepare_motion_instance's box (shutter_world_box) of a
// bottom box B that holds every finite triangle of the bottom at every time, and the root index.
//   * static and shutter-box bottoms: B is the view's root box.  A static bottom's box holds its triangles; a
//     shutter-box bottom's tree is refitted over prepare_motion_triangles' boxes, each of which holds triangle_at at
//     every time (detail::prepare_motion_triangle);
//   * motion-node bottoms: B is the union of the root motion node's two key boxes, and root_index is the root motion
//     node's index.  Every coordinate of triangle_at(tris, id, tau) lies in it: in exact arithmetic the blend lies
//     between the coordinate's two keys, each inside the unwidened key box of its leaf; blend_key rounds it by at most
//     1.5 eps M (1 + O(eps)), M the largest magnitude of the leaf's bounds on that axis, and a leaf side on an axis on
//     which anything moves is widened by 4 eps M + the smallest normal number (MotionNodeBuilder), of which the
//     rounding of the widening takes back at most eps/2 (M + d).  On an axis on which nothing moves the blend is the key
//     itself.  Inner keys are unions of their children's (and possibly widened further), so the root's keys hold every
//     leaf's.  (node_at at some time is not used: its own blend can round one ulp inside a key, which the union
//     of the keys never does.)
// A triangle with a non-finite key is in no box (prepare_motion_triangles and prepare_motion_nodes leave it out).
template <typename T>
BVH_HD void prepare_deforming_instance(DeformingInstance<T>& rec, typename ViewTypes<T>::BBox& box, typename ViewTypes<T>::Vec& centre) {
    if (rec.vertices[0] && rec.motion_nodes) {
        const MotionNode<T>& root = rec.motion_nodes[1];
        T rb[6];
        for (int a = 0; a < 2; ++a) {
            rb[2 * a] = root.xy[1][2 * a] < root.xy[0][2 * a] ? root.xy[1][2 * a] : root.xy[0][2 * a];
            rb[2 * a + 1] = root.xy[0][2 * a + 1] < root.xy[1][2 * a + 1] ? root.xy[1][2 * a + 1] : root.xy[0][2 * a + 1];
        }
        rb[4] = root.z[1][0] < root.z[0][0] ? root.z[1][0] : root.z[0][0];
        rb[5] = root.z[0][1] < root.z[1][1] ? root.z[1][1] : root.z[0][1];
        rec.root_index = root.index;
        shutter_world_box(rec.object_to_world, rb, shutter_keys_finite(rec.object_to_world), box, centre);
    } else {
        rec.root_index = rec.nodes[1].index;
        shutter_world_box(rec.object_to_world, rec.nodes[1].bounds, shutter_keys_finite(rec.object_to_world), box, centre);
    }
}

// The triangle leaf of trace_instances (both builds): the library's leaf_range over [first, first + count) of instance
// `inst`'s bottom tree, without its own tie rule (a slot of another bottom tree is not comparable through this tree's
// prim_ids).  The filter applies the canonical rule on (instance, original id) instead, then the shader's accept, and
// notes the instance of an accepted hit.
template <typename T, bool TieLastVisited, typename Shader, typename Payload>
BVH_HD void instance_leaf(const Shader& shader, const bvhb200::DevTri<T>* tris, const uint32_t* ids, uint32_t inst, Payload& payload,
                          uint32_t first, uint32_t count, bvhb200::RayCtx<T>& r, bvhb200::HitState<T>& hit, uint32_t& hit_inst) {
    bvhb200::leaf_range<T>(tris, ids, false, first, count, r, hit, nullptr, [&](uint32_t slot, T t, T u, T v) {
        const uint32_t id = ids[slot];
        if (!TieLastVisited && hit.slot != bvhb200::kInvalidId && !(t < hit.t)) {      // an exact tie with the current best
            if (inst != hit_inst ? inst > hit_inst : !(id < ids[hit.slot])) return false;
        }
        if (!static_cast<bool>(shader.accept(payload, inst, static_cast<size_t>(id), t, u, v))) return false;
        hit_inst = inst;
        return true;
    });
}

template <typename T, typename Shader> struct MotionShader {
    using Ray = typename ViewTypes<T>::Ray;
    using Hit = typename ViewTypes<T>::Hit;
    struct Payload {
        typename Shader::Payload user;
        T time;                         // the ray's (path's) time, as start gave it
    };
    Shader shader;
    // trace_triangles and trace_instances
    BVH_HD Ray start(size_t i, Payload& p) const { return shader.start(i, p.user, p.time); }
    BVH_HD void finish(size_t i, const Payload& p, const Hit& hit) const { shader.finish(i, p.user, hit); }
    BVH_HD void finish(size_t i, const Payload& p, const Hit& hit, uint32_t inst) const { shader.finish(i, p.user, hit, inst); }
    // trace_paths and trace_instance_paths
    BVH_HD PathStep start(size_t i, Payload& p, Ray& ray) const { return shader.start(i, p.user, ray, p.time); }
    BVH_HD PathStep next(size_t i, Payload& p, const Hit& hit, Ray& ray) const { return shader.next(i, p.user, hit, ray); }
    BVH_HD PathStep next(size_t i, Payload& p, const Hit& hit, uint32_t inst, Ray& ray) const {
        return shader.next(i, p.user, hit, inst, ray);
    }
    BVH_HD void finish(size_t i, const Payload& p) const { shader.finish(i, p.user); }
    // the triangle calls, and the instance calls
    BVH_HD bool accept(Payload& p, size_t prim_id, T t, T u, T v) const {
        return static_cast<bool>(shader.accept(p.user, prim_id, t, u, v));
    }
    BVH_HD bool accept(Payload& p, uint32_t inst, size_t prim_id, T t, T u, T v) const {
        return static_cast<bool>(shader.accept(p.user, inst, prim_id, t, u, v));
    }
};

// The triangle leaf of the motion forms of trace_triangles and trace_paths (both builds): shader_leaf with the triangles
// built at the payload's time.  Per slot: the original id, both keys, the blend (triangle_at), precompute_tri and the
// library's tri_test with the canonical tie rule on original ids (unless TieLastVisited) and the shader's accept as the
// filter: the static leaf on precompute_tri(triangle_at(tris, id, time)).  Not unrolled, so one triangle's registers are
// live at a time.
template <typename T, bool TieLastVisited, typename Shader, typename Payload>
BVH_HD void shader_leaf(const TriangleShader<T, MotionShader<T, Shader>>& ts, Payload& payload, uint32_t first, uint32_t count,
                        bvhb200::RayCtx<T>& r, bvhb200::HitState<T>& hit) {
#if defined(__CUDA_ARCH__)
    #pragma unroll 1
#endif
    for (uint32_t slot = first; slot < first + count; ++slot) {
        const uint32_t id = ts.prim_ids[slot];
        T v[9];
        triangle_at(ts.tris, id, payload.time, v);
        const bvhb200::DevTri<T> tri = bvhb200::precompute_tri(v);
        bvhb200::tri_test<T>(tri, slot, ts.prim_ids, !TieLastVisited, r, hit, [&](uint32_t, T t, T u, T w) {
            return ts.shader.accept(payload, static_cast<size_t>(id), t, u, w);
        });
    }
}

// The caller's shader of the motion-node forms of trace_triangles and trace_paths with the tree's motion nodes beside
// it.  It runs wrapped in MotionShader, like the shader of the motion forms, so the leaf, the record and the time are
// theirs; the kernels see the motion nodes through HasMotionNodes and take motion_inner_step instead of inner_step.
template <typename T, typename Shader> struct WithMotionNodes {
    using Payload = typename Shader::Payload;
    Shader shader;
    MotionNodes<T> motion_nodes;
    template <typename... A> BVH_HD decltype(auto) start(A&&... a) const { return shader.start(std::forward<A>(a)...); }
    template <typename... A> BVH_HD decltype(auto) accept(A&&... a) const { return shader.accept(std::forward<A>(a)...); }
    template <typename... A> BVH_HD decltype(auto) next(A&&... a) const { return shader.next(std::forward<A>(a)...); }
    template <typename... A> BVH_HD void finish(A&&... a) const { shader.finish(std::forward<A>(a)...); }
};
// Whether a triangle kernel's shader carries motion nodes
template <typename Shader> struct HasMotionNodes : std::false_type {};
template <typename T, typename Shader> struct HasMotionNodes<MotionShader<T, WithMotionNodes<T, Shader>>> : std::true_type {};

// The caller's shader of the deforming forms of trace_instances and trace_instance_paths.  It runs wrapped in
// MotionShader, like the shader of the motion forms (so the time, the placement at that time and the record are
// theirs); the instance kernels see it through IsDeforming, read DeformingInstance<T> records and pick each record's
// bottom kind at run time.
template <typename T, typename Shader> struct WithDeformingBottoms {
    using Payload = typename Shader::Payload;
    Shader shader;
    template <typename... A> BVH_HD decltype(auto) start(A&&... a) const { return shader.start(std::forward<A>(a)...); }
    template <typename... A> BVH_HD decltype(auto) accept(A&&... a) const { return shader.accept(std::forward<A>(a)...); }
    template <typename... A> BVH_HD decltype(auto) next(A&&... a) const { return shader.next(std::forward<A>(a)...); }
    template <typename... A> BVH_HD void finish(A&&... a) const { shader.finish(std::forward<A>(a)...); }
};
// Whether an instance kernel's shader runs DeformingInstance<T> records
template <typename Shader> struct IsDeforming : std::false_type {};
template <typename T, typename Shader> struct IsDeforming<MotionShader<T, WithDeformingBottoms<T, Shader>>> : std::true_type {};

// The triangle leaf of a deforming bottom (both builds): instance_leaf with the triangles built at the payload's time.
// Per slot: the original id, triangle_at from the record's vertex keys, precompute_tri and the library's tri_test
// without its own tie rule; the filter applies instance_leaf's canonical rule on (instance, original id), then the
// shader's accept, and notes the instance of an accepted hit.  Not unrolled, as the motion forms' leaf.
template <typename T, bool TieLastVisited, typename Shader, typename Payload>
BVH_HD void deforming_instance_leaf(const Shader& shader, const DeformingInstance<T>& rec, uint32_t inst, Payload& payload, uint32_t first,
                                    uint32_t count, bvhb200::RayCtx<T>& r, bvhb200::HitState<T>& hit, uint32_t& hit_inst) {
    const MotionTriangles<T> tris { { rec.vertices[0], rec.vertices[1] }, 0 };
    const uint32_t* ids = rec.prim_ids;
#if defined(__CUDA_ARCH__)
    #pragma unroll 1
#endif
    for (uint32_t slot = first; slot < first + count; ++slot) {
        const uint32_t id = ids[slot];
        T v[9];
        triangle_at(tris, id, payload.time, v);
        const bvhb200::DevTri<T> tri = bvhb200::precompute_tri(v);
        bvhb200::tri_test<T>(tri, slot, ids, false, r, hit, [&](uint32_t, T t, T u, T w) {
            if (!TieLastVisited && hit.slot != bvhb200::kInvalidId && !(t < hit.t)) {  // an exact tie with the current best
                if (inst != hit_inst ? inst > hit_inst : !(id < ids[hit.slot])) return false;
            }
            if (!static_cast<bool>(shader.accept(payload, inst, static_cast<size_t>(id), t, u, w))) return false;
            hit_inst = inst;
            return true;
        });
    }
}
// The leaf phase of a deforming-scene record (both builds): deforming_instance_leaf when it has vertex keys, otherwise
// instance_leaf on the view's triangles.
template <typename T, bool TieLastVisited, typename Shader, typename Payload>
BVH_HD void deforming_bottom_leaf(const Shader& shader, const DeformingInstance<T>& rec, uint32_t inst, Payload& payload, uint32_t first,
                                  uint32_t count, bvhb200::RayCtx<T>& r, bvhb200::HitState<T>& hit, uint32_t& hit_inst) {
    if (rec.vertices[0]) deforming_instance_leaf<T, TieLastVisited>(shader, rec, inst, payload, first, count, r, hit, hit_inst);
    else instance_leaf<T, TieLastVisited>(shader, rec.tris, rec.prim_ids, inst, payload, first, count, r, hit, hit_inst);
}

// The inner step of the motion-node forms (both builds): inner_step with each child's box blended to the ray's time.
// Per child, node_at's blend (blend_node_xy, blend_node_z) at tau = shutter_time(time), then node_test's slab arithmetic
// and descend, unchanged.  Float closest-hit rays split the fetch as inner_step does: x and y of both keys of both
// children first (two 32-byte halves), and z and the index of a child only when its x / y interval is not already
// empty, with the same operations in the same order as node_test.  Any-hit and double-precision rays read whole nodes.
template <typename T, bool kAny, bool kRobust, typename Stack>
BVH_HD void motion_inner_step(const MotionNode<T>* __restrict__ nodes, T time, const bvhb200::RayCtx<T>& r,
                              typename bvhb200::Real<T>::UInt& top, Stack& stack) {
    using R = bvhb200::Real<T>;
    using U = typename R::UInt;
    const T tau = shutter_time(time);
    const T rest = R::sub(T(1), tau);
    const MotionNode<T>* p = nodes + 1 + bvhb200::index_first(top);       // the left child's slot
    T lb[6], rb[6];
    U li = 0, ri = 0;
    T l0 = r.tmin, l1 = r.tmax, r0 = r.tmin, r1 = r.tmax;
    if constexpr (sizeof(T) == 4 && !kAny) {
        blend_node_xy(p, tau, rest, lb);
        blend_node_xy(p + 1, tau, rest, rb);
        bvhb200::node_test_axes<T, kRobust, 0, 2>(lb, r, l0, l1);
        bvhb200::node_test_axes<T, kRobust, 0, 2>(rb, r, r0, r1);
        if (l0 <= l1) { blend_node_z(p, tau, rest, lb, li); bvhb200::node_test_axes<T, kRobust, 2, 3>(lb, r, l0, l1); }
        if (r0 <= r1) { blend_node_z(p + 1, tau, rest, rb, ri); bvhb200::node_test_axes<T, kRobust, 2, 3>(rb, r, r0, r1); }
    } else {
        blend_node_xy(p, tau, rest, lb);
        blend_node_z(p, tau, rest, lb, li);
        blend_node_xy(p + 1, tau, rest, rb);
        blend_node_z(p + 1, tau, rest, rb, ri);
        bvhb200::node_test<T, kRobust>(lb, r, l0, l1);
        bvhb200::node_test<T, kRobust>(rb, r, r0, r1);
    }
    // ties go left first, as in inner_step
    bvhb200::descend<U>(l0 <= l1, r0 <= r1, !kAny && l0 > r0, li, ri, top, stack);
}

// The placement a ray meets a record at, as its world_to_object handed to f (both builds): a static record's own; for
// a motion record, the inverse of blend_keys at the payload's time (instance_at's), built here.  All NaN: no inverse.
template <typename T, typename Payload, typename F>
BVH_HD void with_world_to_object(const Instance<T>& rec, const Payload&, F&& f) { f(static_cast<const T*>(rec.world_to_object)); }
// The records whose placement moves over the shutter, both keys in object_to_world[2][12]: MotionInstance<T> and
// DeformingInstance<T>
template <typename Rec> struct MotionRecord : std::false_type {};
template <typename T> struct MotionRecord<MotionInstance<T>> : std::true_type { using Scalar = T; };
template <typename T> struct MotionRecord<DeformingInstance<T>> : std::true_type { using Scalar = T; };
template <typename Rec, typename Payload, typename F, std::enable_if_t<MotionRecord<Rec>::value, int> = 0>
BVH_HD void with_world_to_object(const Rec& rec, const Payload& payload, F&& f) {
    using T = typename MotionRecord<Rec>::Scalar;
    T m[12], inv[12];
    blend_keys(rec.object_to_world, payload.time, m);
    invert_affine(m, inv);
    f(static_cast<const T*>(inv));
}
}

// The placement of motion record `rec` (MotionInstance<T> or DeformingInstance<T>) at `time` (both builds): the
// Instance<T> the motion and deforming forms of trace_instances and trace_instance_paths trace a ray of that time
// through.  Its object_to_world is the blend of the keys (detail::blend_keys: time clamped to [0, 1], a NaN time as 0;
// exact at 0 and 1 and for coefficients that do not move), its world_to_object prepare_instance's inverse of that (all
// NaN when it has none: the ray skips the record), and root_index, depth and the bottom arrays are the record's.  (A
// deforming bottom's triangles at that time are triangle_at of the record's vertex keys, not these arrays' tris.)
template <typename Rec, std::enable_if_t<detail::MotionRecord<Rec>::value, int> = 0>
BVH_HD Instance<typename detail::MotionRecord<Rec>::Scalar> instance_at(const Rec& rec, typename detail::MotionRecord<Rec>::Scalar time) {
    Instance<typename detail::MotionRecord<Rec>::Scalar> out;
    out.nodes = rec.nodes; out.prim_ids = rec.prim_ids; out.tris = rec.tris;
    out.root_index = rec.root_index;
    out.depth = rec.depth;
    detail::blend_keys(rec.object_to_world, time, out.object_to_world);
    detail::invert_affine(out.object_to_world, out.world_to_object);
    return out;
}

#if defined(__CUDACC__)
// The two kernels of DeviceView::traverse_bottom_up, one thread per slot of [1, slots).
template <typename T>
__global__ void bottom_up_link_kernel(const bvhb200::DevNode<T>* __restrict__ nodes, size_t slots, uint32_t* __restrict__ parent,
                                      int* __restrict__ flags) {
    const size_t i = 1 + blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < slots) bvhb200::refit_link(nodes, slots, i, parent, flags);
}
template <typename T, typename LeafFn, typename InnerFn>
__global__ void bottom_up_climb_kernel(const bvhb200::DevNode<T>* nodes, size_t slots, const uint32_t* __restrict__ parent,
                                       int* __restrict__ flags, LeafFn leaf_fn, InnerFn inner_fn) {
    const size_t i = 1 + blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < slots) bvhb200::climb_from_leaf<T>(nodes, i, parent, flags, leaf_fn, inner_fn);
}

namespace detail {
// One draw of the DeviceView batch kernels: the idle lanes take the next indices of the warp's run, claiming a new run of
// `run_rays` from `cursor` when it is used up.  begin(i) starts index i on each lane that is not `busy` and takes one.
// False, with the run exhausted, when the batch has none left.
template <typename Begin>
__device__ __forceinline__ bool draw_run(bvhb200::RunCursor& run, unsigned long long* cursor, unsigned long long n, uint32_t run_rays,
                                         unsigned lane, bool busy, unsigned idle, unsigned rank, Begin&& begin) {
    if (run.pos == run.end) {
        const unsigned long long first = bvhb200::claim_run(cursor, run_rays, lane, 0xFFFFFFFFu);
        if (first >= n) { run.exhausted = true; return false; }
        run.pos = first;
        run.end = first + run_rays < n ? first + run_rays : n;
    }
    const unsigned avail = (unsigned)(run.end - run.pos), want = __popc(idle);
    const unsigned take = want < avail ? want : avail;
    if (!busy && rank < take) begin(run.pos + rank);
    run.pos += take;
    return true;
}

// The steps the path kernels (device_view_path_kernel, device_view_instance_path_kernel) and the instance kernels
// (device_view_instance_kernel, device_view_instance_path_kernel) share.  Each kernel keeps a lambda per step that
// forwards to the helper, and that form compiles the older kernels to the same instructions as when the lambdas held
// the code.  One step stays in the kernels: the root part of arming a segment (prologue, root index, empty stack).
// Every helper form tried for it (the whole arm as one helper, with the nodes by value, by reference or through a
// callable, `inline` or `__forceinline__`, or this part as a helper of its own) reordered device_view_path_kernel's
// instructions.
//
// reset_segment: the first part of arming a lane for its next segment: the ray, its tmax as the shader gave it (r.tmax
// shrinks on hits), a reset hit state and the segment kind.  The kernel then sets `top` to kTraversalDone for a segment
// whose interval is a NaN (no traversal: it ends as a miss in the next leaf phase, with no accept call), and otherwise
// runs the prologue and takes the root, and clears the stack.
template <typename T, typename Ray>
__device__ __forceinline__ void reset_segment(PathStep step, const Ray& ray, bvhb200::RayCtx<T>& r, T& tmax_in, bvhb200::HitState<T>& hit,
                                              bool& occlusion) {
    load_ray<T>(ray, r);
    tmax_in = r.tmax;
    hit.slot = bvhb200::kInvalidId; hit.t = r.tmax; hit.u = T(0); hit.v = T(0);
    occlusion = step == PathStep::Occlusion;
}
// A segment ended: next(ray) receives its ray as the shader gave it (r's origin, direction and tmin, tmax_in) and
// returns the next step; End retires the path, anything else arms the lane with the ray next left.
template <typename Ray, typename T, typename Next, typename Retire, typename Arm>
__device__ __forceinline__ void end_segment(const bvhb200::RayCtx<T>& r, T tmax_in, Next&& next, Retire&& retire, Arm&& arm) {
    Ray ray = make_ray<Ray>(r);
    ray.tmax = tmax_in;
    const PathStep step = next(ray);
    if (step == PathStep::End) retire();
    else arm(step, ray);
}

// The two-level stack machine of DeviceView::trace_instances and trace_instance_paths on a lane's shared-memory stack.
// `inst` is the instance the lane is in (kNoInstance at the top level), `r` the world ray or inside an instance its
// object-space ray.  Entering an instance pushes the rest of the top leaf (when it has more), the world ray's origin and
// direction and the marker, then makes `r` the object-space ray with the current tmax.
//
// pop_world_ray: the world ray's origin and direction, from the six entries on top of the stack, into `r`.
template <typename T, typename U> __device__ __forceinline__ void pop_world_ray(bvhb200::SmemStack<U>& stack, bvhb200::RayCtx<T>& r) {
    using R = bvhb200::Real<T>;
    for (int k = 2; k >= 0; --k) r.dir[k] = R::from_bits(stack.pop());
    for (int k = 2; k >= 0; --k) r.org[k] = R::from_bits(stack.pop());
}
// leave_instance: the marker was popped: the world ray back, with the current tmax, and the next entry of the top level
template <typename T, bool IsRobust, typename U>
__device__ __forceinline__ void leave_instance(bvhb200::SmemStack<U>& stack, bvhb200::RayCtx<T>& r, uint32_t& inst, U& top) {
    pop_world_ray<T>(stack, r);
    bvhb200::ray_prologue<T, IsRobust>(r);
    inst = kNoInstance;
    top = bvhb200::pop_or_done<U>(stack);
}
// enter_instance: `top` is a leaf of the top tree: enter its first instance, or go past it when it is singular
template <typename T, bool IsRobust, typename U, typename Shader>
__device__ __forceinline__ void enter_instance(const InstanceShader<T, Shader>& is, bvhb200::SmemStack<U>& stack, bvhb200::RayCtx<T>& r,
                                               uint32_t& inst, U& top) {
    using R = bvhb200::Real<T>;
    const U first = bvhb200::index_first(top);
    const uint32_t count = bvhb200::index_count(top);
    const uint32_t id = is.prim_ids[first];
    const Instance<T>* rec = is.records + id;
    const U rest = bvhb200::make_index<U>(first + 1, count - 1);
    if (instance_is_singular(rec->world_to_object)) {
        top = count > 1 ? rest : bvhb200::pop_or_done<U>(stack);
        return;
    }
    if (count > 1) stack.push(rest);
    for (int k = 0; k < 3; ++k) stack.push(R::bits(r.org[k]));
    for (int k = 0; k < 3; ++k) stack.push(R::bits(r.dir[k]));
    stack.push(kInstanceMarker<U>);
    object_ray(rec->world_to_object, r, r);
    bvhb200::ray_prologue<T, IsRobust>(r);
    inst = id;
    top = rec->root_index;
}
// enter_motion_instance: enter_instance for motion records (MotionInstance<T> or DeformingInstance<T>): the placement
// at the time in the lane's payload is built first (with_world_to_object), and the instance is skipped when it has no
// inverse at that time.  A separate function rather than a form of enter_instance: every shared form tried changed the
// register assignment of device_view_instance_kernel for static records (DESIGN.md section 8).
template <typename T, bool IsRobust, typename U, typename Shader, typename Payload>
__device__ __forceinline__ void enter_motion_instance(const InstanceShader<T, Shader>& is, const Payload& payload,
                                                      bvhb200::SmemStack<U>& stack, bvhb200::RayCtx<T>& r, uint32_t& inst, U& top) {
    using R = bvhb200::Real<T>;
    const U first = bvhb200::index_first(top);
    const uint32_t count = bvhb200::index_count(top);
    const uint32_t id = is.prim_ids[first];
    const auto* rec = is.records + id;
    const U rest = bvhb200::make_index<U>(first + 1, count - 1);
    with_world_to_object(*rec, payload, [&](const T* world_to_object) {
        if (instance_is_singular(world_to_object)) {
            top = count > 1 ? rest : bvhb200::pop_or_done<U>(stack);
            return;
        }
        if (count > 1) stack.push(rest);
        for (int k = 0; k < 3; ++k) stack.push(R::bits(r.org[k]));
        for (int k = 0; k < 3; ++k) stack.push(R::bits(r.dir[k]));
        stack.push(kInstanceMarker<U>);
        object_ray(world_to_object, r, r);
        bvhb200::ray_prologue<T, IsRobust>(r);
        inst = id;
        top = rec->root_index;
    });
}
// Whether a shader runs motion records
template <typename Shader> struct IsMotion : std::false_type {};
template <typename T, typename Shader> struct IsMotion<MotionShader<T, Shader>> : std::true_type {};
// walk_levels: the level changes the entry in `top` asks for, until the lane holds a node of some tree (or
// kTraversalDone: the top level's stack is empty): leave() (leave_instance) on the marker, enter() (enter_instance) on a
// leaf of the top tree
template <typename U, typename Leave, typename Enter>
__device__ __forceinline__ void walk_levels(const U& top, const uint32_t& inst, Leave&& leave, Enter&& enter) {
    for (;;) {
        if (top == kInstanceMarker<U>) leave();
        else if (inst == kNoInstance && bvhb200::index_count(top) != 0 && top != bvhb200::kTraversalDone<U>) enter();
        else break;
    }
}
}

// The kernel of DeviceView::trace: the library's persistent scheduler (persistent_core.cuh) over the caller's tracer.
// Each warp claims runs of `run_rays` consecutive ray indices from `cursor`; a lane draws ray i through
// tracer.start, descends with the library's inner step (a lane whose interval is a NaN pops its stack instead, as
// bvhb200::traverse_top_down does), hands its leaf to tracer.leaf and retires the ray through tracer.finish.
template <typename T, bool IsAnyHit, bool IsRobust, typename Tracer>
__global__ void __launch_bounds__(bvhb200::kTraceBlock, sizeof(T) == 4 ? BVH_TRACE_BLOCKS : 4)
device_view_trace_kernel(const bvhb200::DevNode<T>* __restrict__ nodes, unsigned long long n, unsigned long long* cursor,
                         uint32_t run_rays, uint32_t refill_min, uint32_t inner_budget, Tracer tracer) {
    using U = typename bvhb200::Real<T>::UInt;
    using Ray = typename detail::ViewTypes<T>::Ray;
    extern __shared__ __align__(128) unsigned char device_view_trace_smem[];
    constexpr unsigned kFull = 0xFFFFFFFFu;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned lt_mask = (1u << lane) - 1u;
    bvhb200::SmemStack<U> stack { reinterpret_cast<U*>(device_view_trace_smem) + threadIdx.x, bvhb200::kTraceBlock, 0 };
    const U root_index = nodes[1].index;

    bvhb200::RunCursor run;
    bool has_ray = false;
    unsigned long long index = 0;
    bvhb200::RayCtx<T> r;
    typename Tracer::Payload payload;
    U top = 0;
    auto retire = [&] {
        tracer.finish(static_cast<size_t>(index), static_cast<const typename Tracer::Payload&>(payload), detail::make_ray<Ray>(r));
        has_ray = false;
    };

    // one draw: the idle lanes take the next rays of the warp's run
    auto draw = [&] (unsigned idle, unsigned rank) {
        return detail::draw_run(run, cursor, n, run_rays, lane, has_ray, idle, rank, [&] (unsigned long long i) {
            index = i;
            detail::load_ray<T>(tracer.start(static_cast<size_t>(index), payload), r);
            bvhb200::ray_prologue<T, IsRobust>(r);
            top = root_index;
            stack.clear();
            has_ray = true;
        });
    };

    // inner phase: descend until this lane holds a leaf, its ray is finished, or the step budget of this round is spent
    auto inner = [&] {
        if (has_ray) {
            uint32_t budget = inner_budget;
            const bool nan = bvhb200::ray_interval_is_nan(r);
            while (bvhb200::index_count(top) == 0 && budget != 0) {     // (kTraversalDone ends it too)
                --budget;
                if (nan) top = bvhb200::pop_or_done<U>(stack);           // both children missed, no box test
                else bvhb200::inner_step<T, IsAnyHit, IsRobust>(nodes, r, top, stack);
            }
            if (top == bvhb200::kTraversalDone<U>) retire();
        }
    };

    // leaf phase: the caller's leaf, whose interval the next box test reads; the ray ends on an any-hit hit or an empty stack
    auto leaf = [&] {
        if (has_ray && bvhb200::index_count(top) != 0) {
            const U first = bvhb200::index_first(top);
            Ray ray = detail::make_ray<Ray>(r);
            const bool hit = static_cast<bool>(tracer.leaf(payload, ray, static_cast<size_t>(first),
                                                           static_cast<size_t>(first + (U)bvhb200::index_count(top))));
            r.tmin = ray.tmin;
            r.tmax = ray.tmax;
            if ((IsAnyHit && hit) || !stack.try_pop(top)) retire();
        }
    };
    bvhb200::run_rounds<false>(run, has_ray, kFull, 0u, 0u, nullptr, kFull, refill_min, lt_mask, lane, draw, [] {}, inner, leaf,
                               [] {});
}

// The kernel of DeviceView::query: the same scheduler, launch settings and stack as device_view_trace_kernel, over the
// caller's querier.  A lane draws query i through querier.start, descends with traverse_nodes' step (node_step) and the
// querier's node test, hands its leaf to querier.leaf and retires the query through querier.finish.
template <typename T, bool IsAnyHit, typename Querier>
__global__ void __launch_bounds__(bvhb200::kTraceBlock, sizeof(T) == 4 ? BVH_TRACE_BLOCKS : 4)
device_view_query_kernel(const bvhb200::DevNode<T>* __restrict__ nodes, unsigned long long n, unsigned long long* cursor,
                         uint32_t run_rays, uint32_t refill_min, uint32_t inner_budget, Querier querier) {
    using U = typename bvhb200::Real<T>::UInt;
    using Payload = typename Querier::Payload;
    extern __shared__ __align__(128) unsigned char device_view_query_smem[];
    constexpr unsigned kFull = 0xFFFFFFFFu;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned lt_mask = (1u << lane) - 1u;
    bvhb200::SmemStack<U> stack { reinterpret_cast<U*>(device_view_query_smem) + threadIdx.x, bvhb200::kTraceBlock, 0 };
    const U root_index = nodes[1].index;

    bvhb200::RunCursor run;
    bool has_query = false;
    unsigned long long index = 0;
    Payload payload;
    detail::BoundNode<Querier, Payload, bvhb200::DevNode<T>> node_fn { querier, payload };
    U top = 0;
    auto retire = [&] {
        querier.finish(static_cast<size_t>(index), static_cast<const Payload&>(payload));
        has_query = false;
    };

    // one draw: the idle lanes take the next queries of the warp's run
    auto draw = [&] (unsigned idle, unsigned rank) {
        return detail::draw_run(run, cursor, n, run_rays, lane, has_query, idle, rank, [&] (unsigned long long i) {
            index = i;
            querier.start(static_cast<size_t>(index), payload);
            top = root_index;
            stack.clear();
            has_query = true;
        });
    };

    // inner phase: node steps until this lane holds a leaf, its query is finished, or the step budget of this round is spent
    auto inner = [&] {
        if (has_query) {
            uint32_t budget = inner_budget;
            while (bvhb200::index_count(top) == 0 && budget != 0) {     // (kTraversalDone ends it too)
                --budget;
                bvhb200::node_step<T>(nodes, top, stack, node_fn);
            }
            if (top == bvhb200::kTraversalDone<U>) retire();
        }
    };

    // leaf phase: the caller's leaf; the query ends on an any-hit hit or an empty stack
    auto leaf = [&] {
        if (has_query && bvhb200::index_count(top) != 0) {
            const U first = bvhb200::index_first(top);
            const bool hit = static_cast<bool>(querier.leaf(payload, static_cast<size_t>(first),
                                                            static_cast<size_t>(first + (U)bvhb200::index_count(top))));
            if ((IsAnyHit && hit) || !stack.try_pop(top)) retire();
        }
    };
    bvhb200::run_rounds<false>(run, has_query, kFull, 0u, 0u, nullptr, kFull, refill_min, lt_mask, lane, draw, [] {}, inner, leaf,
                               [] {});
}

// The kernel of DeviceView::trace_triangles: the same scheduler, launch settings and stack as device_view_trace_kernel, with
// the library's own triangle traversal.  A lane draws ray i through shader.start (a ray whose interval is a NaN retires at
// once as a miss), descends with the library's inner step, tests its leaf's triangles against its RayCtx in registers
// with the shader's accept as the filter, and retires the ray with the library's record through shader.finish.
template <typename T, bool IsAnyHit, bool IsRobust, bool TieLastVisited, typename Shader>
__global__ void __launch_bounds__(bvhb200::kTraceBlock, sizeof(T) == 4 ? BVH_TRACE_BLOCKS : 4)
device_view_triangle_kernel(const bvhb200::DevNode<T>* __restrict__ nodes, unsigned long long n, unsigned long long* cursor,
                            uint32_t run_rays, uint32_t refill_min, uint32_t inner_budget, detail::TriangleShader<T, Shader> ts) {
    using U = typename bvhb200::Real<T>::UInt;
    using Payload = typename Shader::Payload;
    extern __shared__ __align__(128) unsigned char device_view_triangle_smem[];
    constexpr unsigned kFull = 0xFFFFFFFFu;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned lt_mask = (1u << lane) - 1u;
    bvhb200::SmemStack<U> stack { reinterpret_cast<U*>(device_view_triangle_smem) + threadIdx.x, bvhb200::kTraceBlock, 0 };

    bvhb200::RunCursor run;
    bool has_ray = false;
    unsigned long long index = 0;
    bvhb200::RayCtx<T> r;
    bvhb200::HitState<T> hit;           // (hit.t is the ray's input tmax until a hit is recorded: a miss's record t)
    Payload payload;
    U top = 0;
    auto retire = [&] {
        ts.shader.finish(static_cast<size_t>(index), static_cast<const Payload&>(payload),
                         detail::make_hit<T>(bvhb200::make_record(hit, hit.t, ts.prim_ids)));
        has_ray = false;
    };

    // one draw: the idle lanes take the next rays of the warp's run; a ray whose interval is a NaN retires at once as a
    // miss.  The root's index is read per ray (one L1 hit) rather than held for the whole kernel: that register is what
    // lets the float kernel fit its 56 without spills.
    auto draw = [&] (unsigned idle, unsigned rank) {
        return detail::draw_run(run, cursor, n, run_rays, lane, has_ray, idle, rank, [&] (unsigned long long i) {
            index = i;
            detail::load_ray<T>(ts.shader.start(static_cast<size_t>(index), payload), r);
            hit.slot = bvhb200::kInvalidId; hit.t = r.tmax; hit.u = T(0); hit.v = T(0);
            if (bvhb200::ray_interval_is_nan(r)) { retire(); return; }
            bvhb200::ray_prologue<T, IsRobust>(r);
            if constexpr (detail::HasMotionNodes<Shader>::value) top = ts.shader.shader.motion_nodes.nodes[1].index;
            else top = nodes[1].index;
            stack.clear();
            has_ray = true;
        });
    };

    // inner phase: descend until this lane holds a leaf, its ray is finished, or the step budget of this round is spent
    // (with motion nodes, each child's box at the ray's time)
    auto inner = [&] {
        if (has_ray) {
            uint32_t budget = inner_budget;
            while (bvhb200::index_count(top) == 0 && budget != 0) {     // (kTraversalDone ends it too)
                --budget;
                if constexpr (detail::HasMotionNodes<Shader>::value)
                    detail::motion_inner_step<T, IsAnyHit, IsRobust>(ts.shader.shader.motion_nodes.nodes, payload.time, r, top, stack);
                else bvhb200::inner_step<T, IsAnyHit, IsRobust>(nodes, r, top, stack);
            }
            if (top == bvhb200::kTraversalDone<U>) retire();
        }
    };

    // leaf phase: the leaf's triangles through the shader's filter; the ray ends on an any-hit hit or an empty stack
    auto leaf = [&] {
        if (has_ray && bvhb200::index_count(top) != 0) {
            detail::shader_leaf<T, TieLastVisited>(ts, payload, (uint32_t)bvhb200::index_first(top), bvhb200::index_count(top), r, hit);
            if ((IsAnyHit && hit.slot != bvhb200::kInvalidId) || !stack.try_pop(top)) retire();
        }
    };
    bvhb200::run_rounds<false>(run, has_ray, kFull, 0u, 0u, nullptr, kFull, refill_min, lt_mask, lane, draw, [] {}, inner, leaf,
                               [] {});
}

// The kernel of DeviceView::trace_paths: device_view_triangle_kernel's scheduler, launch settings, stack and phases, with
// a path per lane instead of a ray.  A lane draws path i through shader.start; each segment runs the any-hit or the
// closest-hit inner step by the lane's segment kind; when a segment ends (leaf phase) the lane hands its record to
// shader.next and either re-arms in place for the next segment, keeping its payload, or retires the path through
// shader.finish.  Only lanes whose path is over become idle and are refilled.
template <typename T, bool IsRobust, bool TieLastVisited, typename Shader>
__global__ void __launch_bounds__(bvhb200::kTraceBlock, sizeof(T) == 4 ? BVH_TRACE_BLOCKS : 4)
device_view_path_kernel(const bvhb200::DevNode<T>* __restrict__ nodes, unsigned long long n, unsigned long long* cursor,
                        uint32_t run_rays, uint32_t refill_min, uint32_t inner_budget, detail::TriangleShader<T, Shader> ts) {
    using U = typename bvhb200::Real<T>::UInt;
    using Payload = typename Shader::Payload;
    using Ray = typename detail::ViewTypes<T>::Ray;
    extern __shared__ __align__(128) unsigned char device_view_path_smem[];
    constexpr unsigned kFull = 0xFFFFFFFFu;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned lt_mask = (1u << lane) - 1u;
    bvhb200::SmemStack<U> stack { reinterpret_cast<U*>(device_view_path_smem) + threadIdx.x, bvhb200::kTraceBlock, 0 };

    bvhb200::RunCursor run;
    bool has_path = false;
    unsigned long long index = 0;
    bvhb200::RayCtx<T> r;
    bvhb200::HitState<T> hit;
    T tmax_in = T(0);                   // the segment's tmax as the shader gave it (r.tmax shrinks on hits)
    bool occlusion = false;             // the segment's kind: any-hit inner step, ends on its first accepted hit
    Payload payload;
    U top = 0;
    auto retire = [&] {
        ts.shader.finish(static_cast<size_t>(index), static_cast<const Payload&>(payload));
        has_path = false;
    };

    // the lane's next segment: hit state reset, prologue, root, empty stack.  A segment whose interval is a NaN gets no
    // traversal: it starts at kTraversalDone and ends as a miss in the next leaf phase, with no accept call.
    auto arm = [&](PathStep step, const Ray& ray) {
        detail::reset_segment<T>(step, ray, r, tmax_in, hit, occlusion);
        top = bvhb200::kTraversalDone<U>;
        if (!bvhb200::ray_interval_is_nan(r)) {
            bvhb200::ray_prologue<T, IsRobust>(r);
            // (read per segment, as device_view_triangle_kernel reads it per ray)
            if constexpr (detail::HasMotionNodes<Shader>::value) top = ts.shader.shader.motion_nodes.nodes[1].index;
            else top = nodes[1].index;
        }
        stack.clear();
        has_path = true;
    };

    // a segment ended: its record and its ray as the shader gave it to next, then the next segment or the path's end
    auto end_segment = [&] {
        detail::end_segment<Ray>(r, tmax_in, [&](Ray& ray) {
            return ts.shader.next(static_cast<size_t>(index), payload,
                                  detail::make_hit<T>(bvhb200::make_record(hit, tmax_in, ts.prim_ids)), ray);
        }, retire, arm);
    };

    // one draw: the idle lanes take the next paths of the warp's run
    auto draw = [&] (unsigned idle, unsigned rank) {
        return detail::draw_run(run, cursor, n, run_rays, lane, has_path, idle, rank, [&] (unsigned long long i) {
            index = i;
            Ray ray;
            const PathStep step = ts.shader.start(static_cast<size_t>(index), payload, ray);
            if (step == PathStep::End) retire();
            else arm(step, ray);
        });
    };

    // inner phase: descend until this lane holds a leaf, its segment is finished, or the step budget of this round is spent
    auto inner = [&] {
        if (has_path) {
            uint32_t budget = inner_budget;
            while (bvhb200::index_count(top) == 0 && budget != 0) {     // (kTraversalDone ends it too)
                --budget;
                if constexpr (detail::HasMotionNodes<Shader>::value) {
                    const MotionNode<T>* motion_nodes = ts.shader.shader.motion_nodes.nodes;
                    if (occlusion) detail::motion_inner_step<T, true, IsRobust>(motion_nodes, payload.time, r, top, stack);
                    else detail::motion_inner_step<T, false, IsRobust>(motion_nodes, payload.time, r, top, stack);
                } else {
                    if (occlusion) bvhb200::inner_step<T, true, IsRobust>(nodes, r, top, stack);
                    else bvhb200::inner_step<T, false, IsRobust>(nodes, r, top, stack);
                }
            }
        }
    };

    // leaf phase: the leaf's triangles through the shader's filter; the segment ends on an occlusion hit, an empty stack,
    // or when the inner phase found nothing left (kTraversalDone)
    auto leaf = [&] {
        if (!has_path) return;
        bool ended = top == bvhb200::kTraversalDone<U>;
        if (!ended && bvhb200::index_count(top) != 0) {
            detail::shader_leaf<T, TieLastVisited>(ts, payload, (uint32_t)bvhb200::index_first(top), bvhb200::index_count(top), r, hit);
            ended = (occlusion && hit.slot != bvhb200::kInvalidId) || !stack.try_pop(top);
        }
        if (ended) end_segment();
    };
    bvhb200::run_rounds<false>(run, has_path, kFull, 0u, 0u, nullptr, kFull, refill_min, lt_mask, lane, draw, [] {}, inner, leaf,
                               [] {});
}

// The kernel of DeviceView::trace_instances: device_view_triangle_kernel's scheduler, launch settings and phases, with
// both levels in one stack machine on the lane's shared-memory stack.  `inst` is the instance the lane is in
// (kNoInstance at the top level); the inner phase steps through the top tree's nodes or that instance's.  In the leaf
// phase a top-level leaf enters its first instance: the rest of the leaf (a top-level leaf index), the world ray's
// origin and direction and the marker are pushed, and the lane's RayCtx becomes the object-space ray with the current
// tmax.  The bottom traversal then runs in the ordinary inner and leaf phases until it pops the marker (its stack is
// empty); the leaf phase then pops the world ray back, keeping the shrunk tmax, and goes on with the next entry.
template <typename T, bool IsAnyHit, bool IsRobust, bool TieLastVisited, typename Shader>
__global__ void __launch_bounds__(bvhb200::kTraceBlock, sizeof(T) == 4 ? BVH_TRACE_BLOCKS : 4)
device_view_instance_kernel(const bvhb200::DevNode<T>* __restrict__ nodes, unsigned long long n, unsigned long long* cursor,
                            uint32_t run_rays, uint32_t refill_min, uint32_t inner_budget, detail::InstanceShader<T, Shader> is) {
    using U = typename bvhb200::Real<T>::UInt;
    using Payload = typename Shader::Payload;
    extern __shared__ __align__(128) unsigned char device_view_instance_smem[];
    constexpr unsigned kFull = 0xFFFFFFFFu;
    constexpr U kMarker = detail::kInstanceMarker<U>;
    constexpr U kDone = bvhb200::kTraversalDone<U>;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned lt_mask = (1u << lane) - 1u;
    bvhb200::SmemStack<U> stack { reinterpret_cast<U*>(device_view_instance_smem) + threadIdx.x, bvhb200::kTraceBlock, 0 };

    bvhb200::RunCursor run;
    bool has_ray = false;
    unsigned long long index = 0;
    bvhb200::RayCtx<T> r;               // the world ray, or inside an instance its object-space ray
    bvhb200::HitState<T> hit;           // hit.slot is a slot of instance hit_inst's bottom tree
    uint32_t hit_inst = detail::kNoInstance;
    uint32_t inst = detail::kNoInstance;
    Payload payload;
    U top = 0;
    auto retire = [&] {
        const uint32_t* ids = hit_inst != detail::kNoInstance ? is.records[hit_inst].prim_ids : is.prim_ids;
        is.shader.finish(static_cast<size_t>(index), static_cast<const Payload&>(payload),
                         detail::make_hit<T>(bvhb200::make_record(hit, hit.t, ids)), hit_inst);
        has_ray = false;
    };

    // one draw: the idle lanes take the next rays of the warp's run; a ray whose interval is a NaN retires at once as a miss
    auto draw = [&] (unsigned idle, unsigned rank) {
        return detail::draw_run(run, cursor, n, run_rays, lane, has_ray, idle, rank, [&] (unsigned long long i) {
            index = i;
            detail::load_ray<T>(is.shader.start(static_cast<size_t>(index), payload), r);
            hit.slot = bvhb200::kInvalidId; hit.t = r.tmax; hit.u = T(0); hit.v = T(0);
            hit_inst = detail::kNoInstance;
            if (bvhb200::ray_interval_is_nan(r)) { retire(); return; }
            bvhb200::ray_prologue<T, IsRobust>(r);
            inst = detail::kNoInstance;
            top = nodes[1].index;
            stack.clear();
            has_ray = true;
        });
    };

    // inner phase: descend the current level until this lane holds a leaf or the marker, its ray is finished, or the step
    // budget of this round is spent (in a deforming scene, a bottom with motion nodes takes their boxes at the ray's time)
    auto inner = [&] {
        if (has_ray) {
            const bvhb200::DevNode<T>* level = inst == detail::kNoInstance ? nodes : is.records[inst].nodes;
            uint32_t budget = inner_budget;
            if constexpr (detail::IsDeforming<Shader>::value) {
                const MotionNode<T>* motion_nodes = inst == detail::kNoInstance ? nullptr : is.records[inst].motion_nodes;
                while (bvhb200::index_count(top) == 0 && budget != 0) {
                    --budget;
                    if (motion_nodes) detail::motion_inner_step<T, IsAnyHit, IsRobust>(motion_nodes, payload.time, r, top, stack);
                    else bvhb200::inner_step<T, IsAnyHit, IsRobust>(level, r, top, stack);
                }
            } else {
                while (bvhb200::index_count(top) == 0 && budget != 0) {     // (kTraversalDone and the marker end it too)
                    --budget;
                    bvhb200::inner_step<T, IsAnyHit, IsRobust>(level, r, top, stack);
                }
            }
            if (top == kDone) retire();
        }
    };

    // the marker was popped: the world ray back, with the current tmax, and the next entry of the top level
    auto leave = [&] { detail::leave_instance<T, IsRobust>(stack, r, inst, top); };
    // `top` is a leaf of the top tree: enter its first instance, or go past it when it is singular
    auto enter = [&] {
        if constexpr (detail::IsMotion<Shader>::value) detail::enter_motion_instance<T, IsRobust>(is, payload, stack, r, inst, top);
        else detail::enter_instance<T, IsRobust>(is, stack, r, inst, top);
    };

    // leaf phase: a bottom leaf's triangles through the filter (the ray ends on an any-hit hit), then the level changes
    // the next entry asks for, until the lane holds a node of some tree; the ray ends when the top level's stack is empty
    auto leaf = [&] {
        if (!has_ray || bvhb200::index_count(top) == 0) return;
        if (inst != detail::kNoInstance && top != kMarker) {
            const auto* rec = is.records + inst;
            if constexpr (detail::IsDeforming<Shader>::value)
                detail::deforming_bottom_leaf<T, TieLastVisited>(is.shader, *rec, inst, payload, (uint32_t)bvhb200::index_first(top),
                                                                 bvhb200::index_count(top), r, hit, hit_inst);
            else
                detail::instance_leaf<T, TieLastVisited>(is.shader, rec->tris, rec->prim_ids, inst, payload, (uint32_t)bvhb200::index_first(top),
                                                         bvhb200::index_count(top), r, hit, hit_inst);
            if (IsAnyHit && hit.slot != bvhb200::kInvalidId) { retire(); return; }
            top = bvhb200::pop_or_done<U>(stack);                  // (the marker at the latest)
        }
        detail::walk_levels(top, inst, leave, enter);
        if (top == kDone) retire();
    };
    bvhb200::run_rounds<false>(run, has_ray, kFull, 0u, 0u, nullptr, kFull, refill_min, lt_mask, lane, draw, [] {}, inner, leaf,
                               [] {});
}

// The kernel of DeviceView::trace_instance_paths: device_view_instance_kernel's scheduler, launch settings and two-level
// stack machine, with a path per lane as in device_view_path_kernel.  Each segment steps through the current level with
// the any-hit or closest-hit inner step by the lane's segment kind.  A segment ends in the leaf phase, on an accepted
// occlusion hit or when the top level is done; an occlusion hit can end it inside an instance, and then the world ray's
// origin and direction are popped back from under the marker before next sees the ray.  next receives the record and
// the hit's instance, and the lane re-arms at the top level or retires the path.
template <typename T, bool IsRobust, bool TieLastVisited, typename Shader>
__global__ void __launch_bounds__(bvhb200::kTraceBlock, sizeof(T) == 4 ? BVH_TRACE_BLOCKS : 4)
device_view_instance_path_kernel(const bvhb200::DevNode<T>* __restrict__ nodes, unsigned long long n, unsigned long long* cursor,
                                 uint32_t run_rays, uint32_t refill_min, uint32_t inner_budget, detail::InstanceShader<T, Shader> is) {
    using U = typename bvhb200::Real<T>::UInt;
    using Payload = typename Shader::Payload;
    using Ray = typename detail::ViewTypes<T>::Ray;
    extern __shared__ __align__(128) unsigned char device_view_instance_path_smem[];
    constexpr unsigned kFull = 0xFFFFFFFFu;
    constexpr U kMarker = detail::kInstanceMarker<U>;
    constexpr U kDone = bvhb200::kTraversalDone<U>;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned lt_mask = (1u << lane) - 1u;
    bvhb200::SmemStack<U> stack { reinterpret_cast<U*>(device_view_instance_path_smem) + threadIdx.x, bvhb200::kTraceBlock, 0 };

    bvhb200::RunCursor run;
    bool has_path = false;
    unsigned long long index = 0;
    bvhb200::RayCtx<T> r;               // the world ray, or inside an instance its object-space ray
    bvhb200::HitState<T> hit;           // hit.slot is a slot of instance hit_inst's bottom tree
    uint32_t hit_inst = detail::kNoInstance;
    uint32_t inst = detail::kNoInstance;
    T tmax_in = T(0);                   // the segment's tmax as the shader gave it
    bool occlusion = false;             // the segment's kind
    Payload payload;
    U top = 0;
    auto retire = [&] {
        is.shader.finish(static_cast<size_t>(index), static_cast<const Payload&>(payload));
        has_path = false;
    };

    // the lane's next segment, at the top level: device_view_path_kernel's arm, and no instance
    auto arm = [&](PathStep step, const Ray& ray) {
        detail::reset_segment<T>(step, ray, r, tmax_in, hit, occlusion);
        top = bvhb200::kTraversalDone<U>;
        if (!bvhb200::ray_interval_is_nan(r)) {
            bvhb200::ray_prologue<T, IsRobust>(r);
            top = nodes[1].index;
        }
        stack.clear();
        hit_inst = detail::kNoInstance;
        inst = detail::kNoInstance;
        has_path = true;
    };

    // a segment ended: inside an instance (an occlusion hit) the world ray comes back from under the marker; then its
    // record, instance and world ray to next, and the next segment or the path's end
    auto end_segment = [&] {
        if (inst != detail::kNoInstance) {
            while (stack.pop() != kMarker) {}
            detail::pop_world_ray<T>(stack, r);
        }
        detail::end_segment<Ray>(r, tmax_in, [&](Ray& ray) {
            const uint32_t* ids = hit_inst != detail::kNoInstance ? is.records[hit_inst].prim_ids : is.prim_ids;
            return is.shader.next(static_cast<size_t>(index), payload, detail::make_hit<T>(bvhb200::make_record(hit, tmax_in, ids)),
                                  hit_inst, ray);
        }, retire, arm);
    };

    // one draw: the idle lanes take the next paths of the warp's run
    auto draw = [&] (unsigned idle, unsigned rank) {
        return detail::draw_run(run, cursor, n, run_rays, lane, has_path, idle, rank, [&] (unsigned long long i) {
            index = i;
            Ray ray;
            const PathStep step = is.shader.start(static_cast<size_t>(index), payload, ray);
            if (step == PathStep::End) retire();
            else arm(step, ray);
        });
    };

    // inner phase: descend the current level until this lane holds a leaf or the marker, its segment is finished, or the
    // step budget of this round is spent
    auto inner = [&] {
        if (has_path) {
            const bvhb200::DevNode<T>* level = inst == detail::kNoInstance ? nodes : is.records[inst].nodes;
            uint32_t budget = inner_budget;
            if constexpr (detail::IsDeforming<Shader>::value) {       // (device_view_instance_kernel's choice per record)
                const MotionNode<T>* motion_nodes = inst == detail::kNoInstance ? nullptr : is.records[inst].motion_nodes;
                while (bvhb200::index_count(top) == 0 && budget != 0) {
                    --budget;
                    if (motion_nodes) {
                        if (occlusion) detail::motion_inner_step<T, true, IsRobust>(motion_nodes, payload.time, r, top, stack);
                        else detail::motion_inner_step<T, false, IsRobust>(motion_nodes, payload.time, r, top, stack);
                    } else {
                        if (occlusion) bvhb200::inner_step<T, true, IsRobust>(level, r, top, stack);
                        else bvhb200::inner_step<T, false, IsRobust>(level, r, top, stack);
                    }
                }
            } else {
                while (bvhb200::index_count(top) == 0 && budget != 0) {     // (kTraversalDone and the marker end it too)
                    --budget;
                    if (occlusion) bvhb200::inner_step<T, true, IsRobust>(level, r, top, stack);
                    else bvhb200::inner_step<T, false, IsRobust>(level, r, top, stack);
                }
            }
        }
    };

    auto leave = [&] { detail::leave_instance<T, IsRobust>(stack, r, inst, top); };
    auto enter = [&] {
        if constexpr (detail::IsMotion<Shader>::value) detail::enter_motion_instance<T, IsRobust>(is, payload, stack, r, inst, top);
        else detail::enter_instance<T, IsRobust>(is, stack, r, inst, top);
    };

    // leaf phase: a bottom leaf's triangles through the filter, then the level walk of device_view_instance_kernel; the
    // segment ends on an occlusion hit or when the top level is done (kTraversalDone, also a NaN segment's start)
    auto leaf = [&] {
        if (!has_path || bvhb200::index_count(top) == 0) return;
        if (inst != detail::kNoInstance && top != kMarker) {
            const auto* rec = is.records + inst;
            if constexpr (detail::IsDeforming<Shader>::value)
                detail::deforming_bottom_leaf<T, TieLastVisited>(is.shader, *rec, inst, payload, (uint32_t)bvhb200::index_first(top),
                                                                 bvhb200::index_count(top), r, hit, hit_inst);
            else
                detail::instance_leaf<T, TieLastVisited>(is.shader, rec->tris, rec->prim_ids, inst, payload, (uint32_t)bvhb200::index_first(top),
                                                         bvhb200::index_count(top), r, hit, hit_inst);
            if (occlusion && hit.slot != bvhb200::kInvalidId) { end_segment(); return; }
            top = bvhb200::pop_or_done<U>(stack);                  // (the marker at the latest)
        }
        detail::walk_levels(top, inst, leave, enter);
        if (top == kDone) end_segment();
    };
    bvhb200::run_rounds<false>(run, has_path, kFull, 0u, 0u, nullptr, kFull, refill_min, lt_mask, lane, draw, [] {}, inner, leaf,
                               [] {});
}

// The kernel of prepare_instances: one thread per instance record.
template <typename T>
__global__ void prepare_instances_kernel(Instance<T>* records, size_t count, typename detail::ViewTypes<T>::BBox* bboxes,
                                         typename detail::ViewTypes<T>::Vec* centers) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < count) detail::prepare_instance<T>(records[i], bboxes[i], centers[i]);
}

// The kernel of prepare_motion_instances: one thread per motion record.
template <typename T>
__global__ void prepare_motion_instances_kernel(MotionInstance<T>* records, size_t count, typename detail::ViewTypes<T>::BBox* bboxes,
                                                typename detail::ViewTypes<T>::Vec* centers) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < count) detail::prepare_motion_instance<T>(records[i], bboxes[i], centers[i]);
}

// The kernel of prepare_deforming_instances: one thread per record.
template <typename T>
__global__ void prepare_deforming_instances_kernel(DeformingInstance<T>* records, size_t count, typename detail::ViewTypes<T>::BBox* bboxes,
                                                   typename detail::ViewTypes<T>::Vec* centers) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < count) detail::prepare_deforming_instance<T>(records[i], bboxes[i], centers[i]);
}

// The kernel of prepare_motion_triangles: one thread per triangle.
template <typename T>
__global__ void prepare_motion_triangles_kernel(MotionTriangles<T> tris, typename detail::ViewTypes<T>::BBox* bboxes,
                                                typename detail::ViewTypes<T>::Vec* centers) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < tris.count) detail::prepare_motion_triangle<T>(tris, i, bboxes[i], centers[i]);
}
#endif

// A plain-data view of one device tree (what bvhNN_get_device_view reports), passed to kernels by value.
template <typename T> struct DeviceView {
    using Scalar = T;
    using Index = typename bvhb200::Real<T>::UInt;      // a node's packed index: first id << 4 | primitive count
    using Ray = typename detail::ViewTypes<T>::Ray;     // bvh_ray3f / bvh_ray3d
    using Hit = typename detail::ViewTypes<T>::Hit;     // bvh_hit3f / bvh_hit3d: { prim_id; t, u, v }
    using Node = bvhb200::DevNode<T>;                   // { T bounds[6] (minx, maxx, miny, maxy, minz, maxz); Index index; pad }
    using Tri = bvhb200::DevTri<T>;                     // PrecomputedTri: p0, e1 = p0 - p1, e2 = p2 - p0, n = cross(e1, e2)
    template <unsigned Capacity> using SmallStack = bvhb200::ArrayStack<Index, Capacity>;
#if defined(__CUDACC__)
    using SharedStack = bvhb200::SmemStack<Index>;
#endif

    const Node* nodes = nullptr;        // node_count + 1 slots: reference node i at slot i + 1 (slot 0 is padding)
    const uint32_t* prim_ids = nullptr; // prim_ids[k]: original id of BVH-order primitive k
    const Tri* tris = nullptr;          // BVH-order triangles, or nullptr when none are attached
    size_t node_count = 0, prim_count = 0;
    size_t depth = 0;                   // longest chain of inner nodes below the root
    int device = 0;
    void* stream = nullptr;             // the handle's cudaStream_t

    static DeviceView from(const typename detail::ViewTypes<T>::CView& c) {
        DeviceView v;
        v.nodes = static_cast<const Node*>(c.nodes);
        v.prim_ids = c.prim_ids;
        v.tris = static_cast<const Tri*>(c.tris);
        v.node_count = c.node_count; v.prim_count = c.prim_count; v.depth = c.depth;
        v.device = c.device; v.stream = c.stream;
        return v;
    }
    // Same, for kernels whose per-thread stack holds `stack_capacity` entries: throws std::length_error when the tree
    // needs more.
    static DeviceView from(const typename detail::ViewTypes<T>::CView& c, size_t stack_capacity) {
        if (stack_capacity < c.depth + 1)
            throw std::length_error("bvh::v2::cuda::DeviceView: a stack of " + std::to_string(stack_capacity) +
                                    " entries is too small for a tree of depth " + std::to_string(c.depth));
        return from(c);
    }

    // get_root().index (reference bvh.h:54)
    BVH_HD Index root_index() const { return nodes[1].index; }
    // reference node i
    BVH_HD const Node& node(size_t i) const { return nodes[i + 1]; }
    BVH_HD size_t prim_id(size_t i) const { return prim_ids[i]; }
    // entries a traversal's stack can hold at once
    BVH_HD size_t stack_bound() const { return depth + 1; }
    // dynamic shared memory of a block of `threads` threads that each use a SharedStack
    BVH_HD size_t shared_stack_bytes(unsigned threads) const { return (depth + 2) * (size_t)threads * sizeof(Index); }
#if defined(__CUDACC__)
    // this thread's stack in a dynamic shared array of shared_stack_bytes(threads) bytes
    __device__ __forceinline__ static SharedStack shared_stack(void* smem, unsigned threads) {
        return SharedStack(static_cast<Index*>(smem) + threadIdx.x, threads, 0);
    }
#endif

    // Bvh::intersect<IsAnyHit, IsRobust> (reference bvh.h:159-182): see the rules at the top of this file.  `ray` is
    // read again after every leaf call, so the leaf function updates the same object (through its own reference).
    template <bool IsAnyHit, bool IsRobust, typename Stack, typename LeafFn, typename InnerFn = detail::NoInnerFn>
    BVH_HD void intersect(const Ray& ray, Index start, Stack& stack, LeafFn&& leaf_fn, InnerFn&& inner_fn = {}) const {
        bvhb200::RayCtx<T> r;
        load(ray, r);
        bvhb200::ray_prologue<T, IsRobust>(r);
        bvhb200::traverse_top_down<T, IsAnyHit, IsRobust>(
            nodes, r, start, stack,
            [&](Index begin, Index end) {
                const bool hit = static_cast<bool>(leaf_fn(static_cast<size_t>(begin), static_cast<size_t>(end)));
                r.tmin = ray.tmin;
                r.tmax = ray.tmax;
                return hit;
            },
            [&](Index first_child) { inner_fn(static_cast<size_t>(first_child)); });
    }

    // Bvh::traverse_top_down<IsAnyHit> (reference bvh.h:59-65,124-157) with the caller's node test: see "Queries other
    // than rays" at the top of this file.
    template <bool IsAnyHit, typename Stack, typename LeafFn, typename NodeFn>
    BVH_HD void traverse_top_down(Index start, Stack& stack, LeafFn&& leaf_fn, NodeFn&& node_fn) const {
        bvhb200::traverse_nodes<T, IsAnyHit>(
            nodes, start, stack,
            [&](Index begin, Index end) { return static_cast<bool>(leaf_fn(static_cast<size_t>(begin), static_cast<size_t>(end))); },
            node_fn);
    }

    // Bvh::traverse_bottom_up (reference bvh.h:184-208) with the caller's leaf and inner functions: see "Data per node"
    // at the top of this file.  The workspace is the parent links and the arrival flags, one of each per slot.
    BVH_HD size_t bottom_up_workspace_bytes() const { return 2 * (node_count + 1) * sizeof(uint32_t); }

    template <typename LeafFn, typename InnerFn>
    void traverse_bottom_up(void* workspace, size_t workspace_bytes, LeafFn leaf_fn, InnerFn inner_fn) const {
        traverse_bottom_up(workspace, workspace_bytes, leaf_fn, inner_fn, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <typename LeafFn, typename InnerFn>
    void traverse_bottom_up(void* workspace, size_t workspace_bytes, LeafFn leaf_fn, InnerFn inner_fn, void* on_stream) const {
        const size_t need = bottom_up_workspace_bytes();
        if (workspace_bytes < need || (need && !workspace))
            throw std::length_error("bvh::v2::cuda::DeviceView::traverse_bottom_up: a workspace of " +
                                    std::to_string(workspace ? workspace_bytes : 0) + " bytes is too small for " +
                                    std::to_string(node_count) + " nodes (" + std::to_string(need) + " bytes)");
        if (node_count == 0) return;
        const size_t slots = node_count + 1;
        uint32_t* parent = static_cast<uint32_t*>(workspace);
        int* flags = reinterpret_cast<int*>(parent + slots);
#if defined(__CUDACC__)
        cudaStream_t s = static_cast<cudaStream_t>(on_stream);
        int previous = 0;
        check(cudaGetDevice(&previous), "cudaGetDevice");
        if (previous != device) check(cudaSetDevice(device), "cudaSetDevice");
        // a slot no inner node points to (possible only in a tree with unreachable nodes) stops the climb
        cudaError_t e = cudaMemsetAsync(parent, 0, slots * sizeof(uint32_t), s);
        const unsigned block = 256, grid = (unsigned)((node_count + block - 1) / block);
        if (e == cudaSuccess) {
            bottom_up_link_kernel<T><<<grid, block, 0, s>>>(nodes, slots, parent, flags);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) {
            bottom_up_climb_kernel<T><<<grid, block, 0, s>>>(nodes, slots, parent, flags, leaf_fn, inner_fn);
            e = cudaGetLastError();
        }
        if (previous != device) cudaSetDevice(previous);
        check(e, "launch");
#else
        (void)on_stream;
        for (size_t i = 0; i < slots; ++i) parent[i] = 0;
        for (size_t i = 1; i < slots; ++i) bvhb200::refit_link(nodes, slots, i, parent, flags);
        for (size_t i = slots; i-- > 1;) bvhb200::climb_from_leaf<T>(nodes, i, parent, flags, leaf_fn, inner_fn);
#endif
    }

    // A whole batch of rays on the library's persistent scheduler, with the caller's per-ray functions: see "Whole
    // batches" at the top of this file.  The workspace is the warps' run cursor.
    BVH_HD size_t trace_workspace_bytes() const { return sizeof(unsigned long long); }

    template <bool IsAnyHit, bool IsRobust, typename Tracer>
    void trace(size_t n, const Tracer& tracer, void* workspace, size_t workspace_bytes) const {
        trace<IsAnyHit, IsRobust>(n, tracer, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsAnyHit, bool IsRobust, typename Tracer>
    void trace(size_t n, const Tracer& tracer, void* workspace, size_t workspace_bytes, void* on_stream) const {
        const bvhb200::TracePlan plan = batch_plan<IsAnyHit, IsRobust>(n, 0u);
#if defined(__CUDACC__)
        run_batch("trace", device_view_trace_kernel<T, IsAnyHit, IsRobust, Tracer>, tracer, n, plan.refill_min, plan.inner_budget,
                  workspace, workspace_bytes, on_stream);
#else
        (void)on_stream; (void)plan;
        batch_stack_bytes("trace", workspace, workspace_bytes);
        using Payload = typename Tracer::Payload;
        for (size_t i = 0; i < n; ++i) {
            Payload payload;
            const Ray start = tracer.start(i, payload);
            Ray ray = start;
            detail::VectorStack<Index> stack;
            stack.elems.reserve(stack_bound());
            intersect<IsAnyHit, IsRobust>(ray, root_index(), stack, [&](size_t begin, size_t end) {
                Ray leaf_ray = start;                        // (other fields are read once, as on the device)
                leaf_ray.tmin = ray.tmin; leaf_ray.tmax = ray.tmax;
                const bool hit = static_cast<bool>(tracer.leaf(payload, leaf_ray, begin, end));
                ray.tmin = leaf_ray.tmin; ray.tmax = leaf_ray.tmax;
                return hit;
            });
            Ray out = start;
            out.tmin = ray.tmin; out.tmax = ray.tmax;
            tracer.finish(i, static_cast<const Payload&>(payload), out);
        }
#endif
    }

    // A whole batch of node-test queries on the same scheduler, with the caller's querier: see "Whole batches of
    // queries" at the top of this file.  The workspace is the warps' run cursor, as trace's.
    BVH_HD size_t query_workspace_bytes() const { return sizeof(unsigned long long); }

    template <bool IsAnyHit, typename Querier>
    void query(size_t n, const Querier& querier, void* workspace, size_t workspace_bytes) const {
        query<IsAnyHit>(n, querier, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsAnyHit, typename Querier>
    void query(size_t n, const Querier& querier, void* workspace, size_t workspace_bytes, void* on_stream) const {
        const bvhb200::QueryPlan plan = bvhb200::plan_query();
#if defined(__CUDACC__)
        run_batch("query", device_view_query_kernel<T, IsAnyHit, Querier>, querier, n, plan.refill_min, plan.inner_budget,
                  workspace, workspace_bytes, on_stream);
#else
        (void)on_stream; (void)plan;
        batch_stack_bytes("query", workspace, workspace_bytes);
        using Payload = typename Querier::Payload;
        for (size_t i = 0; i < n; ++i) {
            Payload payload;
            querier.start(i, payload);
            detail::VectorStack<Index> stack;
            stack.elems.reserve(stack_bound());
            traverse_top_down<IsAnyHit>(root_index(), stack,
                                        [&](size_t begin, size_t end) { return static_cast<bool>(querier.leaf(payload, begin, end)); },
                                        detail::BoundNode<Querier, Payload, Node> { querier, payload });
            querier.finish(i, static_cast<const Payload&>(payload));
        }
#endif
    }

    // A whole batch of rays through the library's triangle traversal, with the caller's ray source, hit filter and hit
    // sink: see "Whole batches of triangle rays" at the top of this file.  The workspace is the warps' run cursor,
    // trace_workspace_bytes() bytes.
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_triangles(size_t n, const Shader& shader, void* workspace, size_t workspace_bytes) const {
        trace_triangles<IsAnyHit, IsRobust, TieLastVisited>(n, shader, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_triangles(size_t n, const Shader& shader, void* workspace, size_t workspace_bytes, void* on_stream) const {
        if (!tris)
            throw std::invalid_argument("bvh::v2::cuda::DeviceView::trace_triangles: the tree has no triangles (built from boxes)");
        triangle_batch<IsAnyHit, IsRobust, TieLastVisited>("trace_triangles", n, detail::TriangleShader<T, Shader> { shader, tris, prim_ids },
                                                           workspace, workspace_bytes, on_stream);
    }
    // The same through a mesh whose vertices move over the shutter, each ray at its own time: see "Deforming meshes" at
    // the top of this file.  The view needs no triangles (a tree from bvhNN_build_boxes over prepare_motion_triangles'
    // boxes is the usual one); the shader's start also gives the ray's time.
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_triangles(size_t n, const MotionTriangles<T>& motion, const Shader& shader, void* workspace, size_t workspace_bytes) const {
        trace_triangles<IsAnyHit, IsRobust, TieLastVisited>(n, motion, shader, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_triangles(size_t n, const MotionTriangles<T>& motion, const Shader& shader, void* workspace, size_t workspace_bytes,
                         void* on_stream) const {
        using MS = detail::MotionShader<T, Shader>;
        check_motion_triangles("trace_triangles (motion)", motion);
        triangle_batch<IsAnyHit, IsRobust, TieLastVisited>("trace_triangles (motion)", n,
                                                           detail::TriangleShader<T, MS> { MS { shader }, motion, prim_ids },
                                                           workspace, workspace_bytes, on_stream);
    }
    // The same with the tree's motion nodes (prepare_motion_nodes): each inner step tests the children's boxes at the
    // ray's time (node_at) instead of this view's boxes over the whole shutter.  See "Deforming meshes" at the top of
    // this file.  The view's node bounds are not read.
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_triangles(size_t n, const MotionTriangles<T>& motion, const MotionNodes<T>& motion_nodes, const Shader& shader,
                         void* workspace, size_t workspace_bytes) const {
        trace_triangles<IsAnyHit, IsRobust, TieLastVisited>(n, motion, motion_nodes, shader, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_triangles(size_t n, const MotionTriangles<T>& motion, const MotionNodes<T>& motion_nodes, const Shader& shader,
                         void* workspace, size_t workspace_bytes, void* on_stream) const {
        using MS = detail::MotionShader<T, detail::WithMotionNodes<T, Shader>>;
        check_motion_triangles("trace_triangles (motion nodes)", motion);
        check_motion_nodes("trace_triangles (motion nodes)", motion_nodes);
        triangle_batch<IsAnyHit, IsRobust, TieLastVisited>(
            "trace_triangles (motion nodes)", n,
            detail::TriangleShader<T, MS> { MS { detail::WithMotionNodes<T, Shader> { shader, motion_nodes } }, motion, prim_ids },
            workspace, workspace_bytes, on_stream);
    }

    // Whole paths of triangle-ray segments, each continued in place from the last: see "Whole paths" at the top of this
    // file.  The workspace is the warps' run cursor, trace_workspace_bytes() bytes.
    template <bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_paths(size_t n, const Shader& shader, void* workspace, size_t workspace_bytes) const {
        trace_paths<IsRobust, TieLastVisited>(n, shader, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_paths(size_t n, const Shader& shader, void* workspace, size_t workspace_bytes, void* on_stream) const {
        if (!tris)
            throw std::invalid_argument("bvh::v2::cuda::DeviceView::trace_paths: the tree has no triangles (built from boxes)");
        path_batch<IsRobust, TieLastVisited>("trace_paths", n, detail::TriangleShader<T, Shader> { shader, tris, prim_ids }, workspace,
                                             workspace_bytes, on_stream);
    }
    // The same through a mesh whose vertices move over the shutter, each path at its own time: see "Deforming meshes" at
    // the top of this file.  The shader's start also gives the path's time, which holds for all its segments.
    template <bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_paths(size_t n, const MotionTriangles<T>& motion, const Shader& shader, void* workspace, size_t workspace_bytes) const {
        trace_paths<IsRobust, TieLastVisited>(n, motion, shader, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_paths(size_t n, const MotionTriangles<T>& motion, const Shader& shader, void* workspace, size_t workspace_bytes,
                     void* on_stream) const {
        using MS = detail::MotionShader<T, Shader>;
        check_motion_triangles("trace_paths (motion)", motion);
        path_batch<IsRobust, TieLastVisited>("trace_paths (motion)", n, detail::TriangleShader<T, MS> { MS { shader }, motion, prim_ids },
                                             workspace, workspace_bytes, on_stream);
    }
    // The same with the tree's motion nodes (prepare_motion_nodes), as for trace_triangles.
    template <bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_paths(size_t n, const MotionTriangles<T>& motion, const MotionNodes<T>& motion_nodes, const Shader& shader, void* workspace,
                     size_t workspace_bytes) const {
        trace_paths<IsRobust, TieLastVisited>(n, motion, motion_nodes, shader, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_paths(size_t n, const MotionTriangles<T>& motion, const MotionNodes<T>& motion_nodes, const Shader& shader, void* workspace,
                     size_t workspace_bytes, void* on_stream) const {
        using MS = detail::MotionShader<T, detail::WithMotionNodes<T, Shader>>;
        check_motion_triangles("trace_paths (motion nodes)", motion);
        check_motion_nodes("trace_paths (motion nodes)", motion_nodes);
        path_batch<IsRobust, TieLastVisited>(
            "trace_paths (motion nodes)", n,
            detail::TriangleShader<T, MS> { MS { detail::WithMotionNodes<T, Shader> { shader, motion_nodes } }, motion, prim_ids },
            workspace, workspace_bytes, on_stream);
    }

    // A whole batch of triangle rays through a top-level tree of placed meshes: see "Instanced scenes" at the top of this
    // file.  This view is the top tree; its primitive k is instances.records[prim_ids[k]].  The workspace is the warps'
    // run cursor, trace_workspace_bytes() bytes.
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_instances(size_t n, const Instances<T>& instances, const Shader& shader, void* workspace, size_t workspace_bytes) const {
        trace_instances<IsAnyHit, IsRobust, TieLastVisited>(n, instances, shader, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_instances(size_t n, const Instances<T>& instances, const Shader& shader, void* workspace, size_t workspace_bytes,
                         void* on_stream) const {
        instance_batch<IsAnyHit, IsRobust, TieLastVisited>("trace_instances", n, instances,
                                                           detail::InstanceShader<T, Shader> { shader, instances.records, prim_ids },
                                                           workspace, workspace_bytes, on_stream);
    }
    // The same through a top-level tree of moving placements, each ray at its own time: see "Motion blur" at the top of
    // this file.  The shader's start also gives the ray's time.
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_instances(size_t n, const MotionInstances<T>& instances, const Shader& shader, void* workspace, size_t workspace_bytes) const {
        trace_instances<IsAnyHit, IsRobust, TieLastVisited>(n, instances, shader, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_instances(size_t n, const MotionInstances<T>& instances, const Shader& shader, void* workspace, size_t workspace_bytes,
                         void* on_stream) const {
        using MS = detail::MotionShader<T, Shader>;
        instance_batch<IsAnyHit, IsRobust, TieLastVisited>("trace_instances (motion)", n, instances,
                                                           detail::InstanceShader<T, MS> { MS { shader }, instances.records, prim_ids },
                                                           workspace, workspace_bytes, on_stream);
    }

    // Whole paths through a top-level tree of placed meshes, each segment continued in place from the last: see "Paths
    // through instanced scenes" at the top of this file.  This view is the top tree, as for trace_instances.  The
    // workspace is the warps' run cursor, trace_workspace_bytes() bytes.
    template <bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_instance_paths(size_t n, const Instances<T>& instances, const Shader& shader, void* workspace, size_t workspace_bytes) const {
        trace_instance_paths<IsRobust, TieLastVisited>(n, instances, shader, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_instance_paths(size_t n, const Instances<T>& instances, const Shader& shader, void* workspace, size_t workspace_bytes,
                              void* on_stream) const {
        instance_path_batch<IsRobust, TieLastVisited>("trace_instance_paths", n, instances,
                                                      detail::InstanceShader<T, Shader> { shader, instances.records, prim_ids },
                                                      workspace, workspace_bytes, on_stream);
    }
    // The same through a top-level tree of moving placements, each path at its own time: see "Motion blur" at the top of
    // this file.  The shader's start also gives the path's time, which holds for all its segments.
    template <bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_instance_paths(size_t n, const MotionInstances<T>& instances, const Shader& shader, void* workspace,
                              size_t workspace_bytes) const {
        trace_instance_paths<IsRobust, TieLastVisited>(n, instances, shader, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_instance_paths(size_t n, const MotionInstances<T>& instances, const Shader& shader, void* workspace, size_t workspace_bytes,
                              void* on_stream) const {
        using MS = detail::MotionShader<T, Shader>;
        instance_path_batch<IsRobust, TieLastVisited>("trace_instance_paths (motion)", n, instances,
                                                      detail::InstanceShader<T, MS> { MS { shader }, instances.records, prim_ids },
                                                      workspace, workspace_bytes, on_stream);
    }

    // The same through a scene that mixes static and deforming bottoms under moving placements, each ray at its own
    // time: see "Deforming instances" at the top of this file.  The shader is a motion form's (start also gives the time).
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_instances(size_t n, const DeformingInstances<T>& instances, const Shader& shader, void* workspace,
                         size_t workspace_bytes) const {
        trace_instances<IsAnyHit, IsRobust, TieLastVisited>(n, instances, shader, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_instances(size_t n, const DeformingInstances<T>& instances, const Shader& shader, void* workspace, size_t workspace_bytes,
                         void* on_stream) const {
        using MS = detail::MotionShader<T, detail::WithDeformingBottoms<T, Shader>>;
        instance_batch<IsAnyHit, IsRobust, TieLastVisited>(
            "trace_instances (deforming)", n, instances,
            detail::InstanceShader<T, MS> { MS { detail::WithDeformingBottoms<T, Shader> { shader } }, instances.records, prim_ids },
            workspace, workspace_bytes, on_stream);
    }
    // Whole paths through such a scene, each path at its own time.
    template <bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_instance_paths(size_t n, const DeformingInstances<T>& instances, const Shader& shader, void* workspace,
                              size_t workspace_bytes) const {
        trace_instance_paths<IsRobust, TieLastVisited>(n, instances, shader, workspace, workspace_bytes, stream);
    }
    // `on_stream` is a cudaStream_t (unused by the host pass)
    template <bool IsRobust, bool TieLastVisited = false, typename Shader>
    void trace_instance_paths(size_t n, const DeformingInstances<T>& instances, const Shader& shader, void* workspace,
                              size_t workspace_bytes, void* on_stream) const {
        using MS = detail::MotionShader<T, detail::WithDeformingBottoms<T, Shader>>;
        instance_path_batch<IsRobust, TieLastVisited>(
            "trace_instance_paths (deforming)", n, instances,
            detail::InstanceShader<T, MS> { MS { detail::WithDeformingBottoms<T, Shader> { shader } }, instances.records, prim_ids },
            workspace, workspace_bytes, on_stream);
    }

    // PrecomputedTri::intersect (reference tri.h:55-74) on BVH-order triangle k: true, with the hit's distance and
    // barycentrics, when the ray meets it at a distance in [ray.tmin, ray.tmax].  The batched kernels' own test.
    BVH_HD bool intersect_tri(size_t k, const Ray& ray, T& t, T& u, T& v) const {
        bvhb200::RayCtx<T> r;
        load(ray, r);
        bvhb200::HitState<T> hit { bvhb200::kInvalidId, r.tmax, T(0), T(0) };
        Tri tri;
        bvhb200::load_tri(tris + k, tri);
        if (!bvhb200::tri_test<T>(tri, static_cast<uint32_t>(k), prim_ids, false, r, hit)) return false;
        t = hit.t; u = hit.u; v = hit.v;
        return true;
    }

private:
    // the shared memory a persistent block may have, as bvhNN_intersect_rays bounds it
    static constexpr size_t kMaxTraceSmem = 200 * 1024;

    // The library's scheduling of a persistent closest-hit or any-hit batch (trace, trace_triangles, trace_paths,
    // trace_instances, trace_instance_paths), with its default
    // settings; `flags` adds kTraceLastVisited.
    template <bool IsAnyHit, bool IsRobust> static bvhb200::TracePlan batch_plan(size_t n, unsigned flags) {
        bvhb200::TraceRequest request {};
        request.flags = bvhb200::kTraceNoTma | (IsAnyHit ? bvhb200::kTraceAnyHit : 0u) | (IsRobust ? bvhb200::kTraceRobust : 0u) | flags;
        request.is_float = sizeof(T) == 4;
        request.n = n;
        return bvhb200::plan_trace(request);
    }

    // trace_triangles of either triangle source (`ts` holds the tree's triangles, or the keys of a deforming mesh with the
    // shader wrapped in detail::MotionShader), named `call` in its errors.
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited, typename Shader>
    void triangle_batch(const char* call, size_t n, const detail::TriangleShader<T, Shader>& ts, void* workspace, size_t workspace_bytes,
                        void* on_stream) const {
        const bvhb200::TracePlan plan = batch_plan<IsAnyHit, IsRobust>(n, TieLastVisited ? bvhb200::kTraceLastVisited : 0u);
#if defined(__CUDACC__)
        run_batch(call, device_view_triangle_kernel<T, IsAnyHit, IsRobust, TieLastVisited, Shader>, ts, n, plan.refill_min,
                  plan.inner_budget, workspace, workspace_bytes, on_stream);
#else
        (void)on_stream; (void)plan;
        batch_stack_bytes(call, workspace, workspace_bytes);
        using Payload = typename Shader::Payload;
        for (size_t i = 0; i < n; ++i) {
            Payload payload;
            const Ray ray = ts.shader.start(i, payload);
            ts.shader.finish(i, static_cast<const Payload&>(payload), host_triangle_ray<IsAnyHit, IsRobust, TieLastVisited>(ts, payload, ray));
        }
#endif
    }

    // trace_paths of either triangle source, as triangle_batch
    template <bool IsRobust, bool TieLastVisited, typename Shader>
    void path_batch(const char* call, size_t n, const detail::TriangleShader<T, Shader>& ts, void* workspace, size_t workspace_bytes,
                    void* on_stream) const {
        const bvhb200::TracePlan plan = batch_plan<false, IsRobust>(n, TieLastVisited ? bvhb200::kTraceLastVisited : 0u);
#if defined(__CUDACC__)
        run_batch(call, device_view_path_kernel<T, IsRobust, TieLastVisited, Shader>, ts, n, plan.refill_min, plan.inner_budget,
                  workspace, workspace_bytes, on_stream);
#else
        (void)on_stream; (void)plan;
        batch_stack_bytes(call, workspace, workspace_bytes);
        using Payload = typename Shader::Payload;
        for (size_t i = 0; i < n; ++i) {
            Payload payload;
            Ray ray;
            PathStep step = ts.shader.start(i, payload, ray);
            while (step != PathStep::End) {
                const Hit hit = step == PathStep::Occlusion ? host_triangle_ray<true, IsRobust, TieLastVisited>(ts, payload, ray)
                                                            : host_triangle_ray<false, IsRobust, TieLastVisited>(ts, payload, ray);
                step = ts.shader.next(i, payload, hit, ray);
            }
            ts.shader.finish(i, static_cast<const Payload&>(payload));
        }
#endif
    }

    // The keys of the motion forms of trace_triangles and trace_paths: one triangle per primitive of this tree, both keys
    void check_motion_triangles(const char* call, const MotionTriangles<T>& motion) const {
        const std::string who = std::string("bvh::v2::cuda::DeviceView::") + call;
        if (!motion.vertices[0] || !motion.vertices[1]) throw std::invalid_argument(who + ": a null key pointer");
        if (motion.count != prim_count)
            throw std::invalid_argument(who + ": " + std::to_string(motion.count) + " triangles for a tree of " +
                                        std::to_string(prim_count) + " primitives");
    }
    // The motion nodes of the motion-node forms: one record per slot of this tree
    void check_motion_nodes(const char* call, const MotionNodes<T>& motion_nodes) const {
        const std::string who = std::string("bvh::v2::cuda::DeviceView::") + call;
        if (!motion_nodes.nodes) throw std::invalid_argument(who + ": a null motion-node pointer");
        if (motion_nodes.node_count != node_count)
            throw std::invalid_argument(who + ": motion nodes of " + std::to_string(motion_nodes.node_count) + " nodes for a tree of " +
                                        std::to_string(node_count) + " nodes");
    }

    // trace_instances of either record kind (Records: Instances<T> or MotionInstances<T>; `is` holds its records and the
    // shader, wrapped in detail::MotionShader for motion records), named `call` in its errors.
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited, typename Records, typename Shader>
    void instance_batch(const char* call, size_t n, const Records& instances, const detail::InstanceShader<T, Shader>& is, void* workspace,
                        size_t workspace_bytes, void* on_stream) const {
        check_instances(call, instances.count, instances.records);
        const bvhb200::TracePlan plan = batch_plan<IsAnyHit, IsRobust>(n, TieLastVisited ? bvhb200::kTraceLastVisited : 0u);
        const size_t extra = instances.max_depth + detail::kInstanceStackExtra;
#if defined(__CUDACC__)
        run_batch(call, device_view_instance_kernel<T, IsAnyHit, IsRobust, TieLastVisited, Shader>, is, n, plan.refill_min,
                  plan.inner_budget, workspace, workspace_bytes, on_stream, extra);
#else
        (void)on_stream; (void)plan;
        batch_stack_bytes(call, workspace, workspace_bytes, extra);
        using Payload = typename Shader::Payload;
        for (size_t i = 0; i < n; ++i) {
            Payload payload;
            const Ray ray = is.shader.start(i, payload);
            uint32_t hit_inst = detail::kNoInstance;
            const Hit hit = host_instance_ray<IsAnyHit, IsRobust, TieLastVisited>(is, payload, ray, hit_inst);
            is.shader.finish(i, static_cast<const Payload&>(payload), hit, hit_inst);
        }
#endif
    }

    // trace_instance_paths of either record kind, as instance_batch
    template <bool IsRobust, bool TieLastVisited, typename Records, typename Shader>
    void instance_path_batch(const char* call, size_t n, const Records& instances, const detail::InstanceShader<T, Shader>& is,
                             void* workspace, size_t workspace_bytes, void* on_stream) const {
        check_instances(call, instances.count, instances.records);
        const bvhb200::TracePlan plan = batch_plan<false, IsRobust>(n, TieLastVisited ? bvhb200::kTraceLastVisited : 0u);
        const size_t extra = instances.max_depth + detail::kInstanceStackExtra;
#if defined(__CUDACC__)
        run_batch(call, device_view_instance_path_kernel<T, IsRobust, TieLastVisited, Shader>, is, n, plan.refill_min,
                  plan.inner_budget, workspace, workspace_bytes, on_stream, extra);
#else
        (void)on_stream; (void)plan;
        batch_stack_bytes(call, workspace, workspace_bytes, extra);
        using Payload = typename Shader::Payload;
        for (size_t i = 0; i < n; ++i) {
            Payload payload;
            Ray ray;
            PathStep step = is.shader.start(i, payload, ray);
            while (step != PathStep::End) {
                uint32_t hit_inst = detail::kNoInstance;
                const Hit hit = step == PathStep::Occlusion ? host_instance_ray<true, IsRobust, TieLastVisited>(is, payload, ray, hit_inst)
                                                            : host_instance_ray<false, IsRobust, TieLastVisited>(is, payload, ray, hit_inst);
                step = is.shader.next(i, payload, hit, hit_inst, ray);
            }
            is.shader.finish(i, static_cast<const Payload&>(payload));
        }
#endif
    }

    // The record count of trace_instances and trace_instance_paths: the top tree's primitive count
    void check_instances(const char* call, size_t count, const void* records) const {
        if (count != prim_count || (count && !records))
            throw std::invalid_argument(std::string("bvh::v2::cuda::DeviceView::") + call + ": " + std::to_string(count) +
                                        " instance records for a top tree of " + std::to_string(prim_count) + " primitives");
    }

    // One ray of trace_triangles, and one segment of trace_paths, on the host: the library's traversal with the shader's
    // accept as the leaf's filter, and the record finish (trace_triangles) or next (trace_paths) receives.  A ray whose
    // interval is a NaN gets no accept call and a miss record.
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited, typename Shader, typename Payload>
    Hit host_triangle_ray(const detail::TriangleShader<T, Shader>& ts, Payload& payload, const Ray& ray) const {
        bvhb200::RayCtx<T> r;
        load(ray, r);
        const T tmax_in = r.tmax;
        bvhb200::HitState<T> hit { bvhb200::kInvalidId, r.tmax, T(0), T(0) };
        if (!bvhb200::ray_interval_is_nan(r)) {
            bvhb200::ray_prologue<T, IsRobust>(r);
            detail::VectorStack<Index> stack;
            stack.elems.reserve(stack_bound());
            if constexpr (detail::HasMotionNodes<Shader>::value) {
                // traverse_top_down's loop with the inner step of the motion-node forms (the interval stays a number:
                // a leaf only shrinks tmax to a hit's t)
                const MotionNode<T>* motion_nodes = ts.shader.shader.motion_nodes.nodes;
                Index top = motion_nodes[1].index;
                for (;;) {
                    while (bvhb200::index_count(top) == 0)
                        detail::motion_inner_step<T, IsAnyHit, IsRobust>(motion_nodes, payload.time, r, top, stack);
                    if (top == bvhb200::kTraversalDone<Index>) break;
                    detail::shader_leaf<T, TieLastVisited>(ts, payload, (uint32_t)bvhb200::index_first(top), bvhb200::index_count(top), r, hit);
                    if (IsAnyHit && hit.slot != bvhb200::kInvalidId) break;
                    top = bvhb200::pop_or_done<Index>(stack);
                }
            } else {
                bvhb200::traverse_top_down<T, IsAnyHit, IsRobust>(
                    nodes, r, root_index(), stack,
                    [&](Index begin, Index end) {
                        detail::shader_leaf<T, TieLastVisited>(ts, payload, (uint32_t)begin, (uint32_t)(end - begin), r, hit);
                        return hit.slot != bvhb200::kInvalidId;
                    },
                    [](Index) {});
            }
        }
        return detail::make_hit<T>(bvhb200::make_record(hit, tmax_in, prim_ids));
    }

    // One ray of trace_instances on the host, the nested loop its contract states: Bvh::intersect on the top tree, whose
    // leaf enters its instances in BVH order (skipping singular ones), each with the object-space ray, the current tmax, the
    // bottom tree's Bvh::intersect and the triangle leaf of trace_instances, and carries the shrunk tmax back.  Returns the
    // record; `hit_inst` is the hit's instance.
    template <bool IsAnyHit, bool IsRobust, bool TieLastVisited, typename Shader, typename Payload>
    Hit host_instance_ray(const detail::InstanceShader<T, Shader>& is, Payload& payload, const Ray& ray, uint32_t& hit_inst) const {
        bvhb200::RayCtx<T> r;
        load(ray, r);
        const T tmax_in = r.tmax;
        bvhb200::HitState<T> hit { bvhb200::kInvalidId, r.tmax, T(0), T(0) };
        hit_inst = detail::kNoInstance;
        if (!bvhb200::ray_interval_is_nan(r)) {
            bvhb200::ray_prologue<T, IsRobust>(r);
            detail::VectorStack<Index> stack;
            stack.elems.reserve(stack_bound());
            bvhb200::traverse_top_down<T, IsAnyHit, IsRobust>(
                nodes, r, root_index(), stack,
                [&](Index begin, Index end) {
                    for (Index k = begin; k < end; ++k) {
                        const uint32_t id = prim_ids[k];
                        const auto& rec = is.records[id];
                        bool singular = false;
                        bvhb200::RayCtx<T> o;
                        detail::with_world_to_object(rec, payload, [&](const T* world_to_object) {
                            singular = detail::instance_is_singular(world_to_object);
                            detail::object_ray(world_to_object, r, o);
                        });
                        if (singular) continue;
                        bvhb200::ray_prologue<T, IsRobust>(o);
                        detail::VectorStack<Index> bottom;
                        bottom.elems.reserve(rec.depth + 1);
                        if constexpr (detail::IsDeforming<Shader>::value) {
                            // the record's bottom kind: the leaf of deforming_bottom_leaf, and with motion nodes
                            // traverse_top_down's loop with their inner step (host_triangle_ray's)
                            if (rec.motion_nodes) {
                                Index top = rec.root_index;
                                for (;;) {
                                    while (bvhb200::index_count(top) == 0)
                                        detail::motion_inner_step<T, IsAnyHit, IsRobust>(rec.motion_nodes, payload.time, o, top, bottom);
                                    if (top == bvhb200::kTraversalDone<Index>) break;
                                    detail::deforming_bottom_leaf<T, TieLastVisited>(is.shader, rec, id, payload, (uint32_t)bvhb200::index_first(top),
                                                                                     bvhb200::index_count(top), o, hit, hit_inst);
                                    if (IsAnyHit && hit.slot != bvhb200::kInvalidId) break;
                                    top = bvhb200::pop_or_done<Index>(bottom);
                                }
                            } else {
                                bvhb200::traverse_top_down<T, IsAnyHit, IsRobust>(
                                    rec.nodes, o, rec.root_index, bottom,
                                    [&](Index b, Index e) {
                                        detail::deforming_bottom_leaf<T, TieLastVisited>(is.shader, rec, id, payload, (uint32_t)b,
                                                                                         (uint32_t)(e - b), o, hit, hit_inst);
                                        return hit.slot != bvhb200::kInvalidId;
                                    },
                                    [](Index) {});
                            }
                        } else {
                            bvhb200::traverse_top_down<T, IsAnyHit, IsRobust>(
                                rec.nodes, o, rec.root_index, bottom,
                                [&](Index b, Index e) {
                                    detail::instance_leaf<T, TieLastVisited>(is.shader, rec.tris, rec.prim_ids, id, payload, (uint32_t)b,
                                                                             (uint32_t)(e - b), o, hit, hit_inst);
                                    return hit.slot != bvhb200::kInvalidId;
                                },
                                [](Index) {});
                        }
                        r.tmax = o.tmax;
                        if (IsAnyHit && hit.slot != bvhb200::kInvalidId) return true;
                    }
                    return hit.slot != bvhb200::kInvalidId;
                },
                [](Index) {});
        }
        const uint32_t* ids = hit_inst != detail::kNoInstance ? is.records[hit_inst].prim_ids : prim_ids;
        return detail::make_hit<T>(bvhb200::make_record(hit, tmax_in, ids));
    }

    // The checks of trace, query, trace_triangles, trace_paths, trace_instances and trace_instance_paths (`call`): the
    // workspace, then the shared-memory stack of the batched kernels, sized and bounded as bvhNN_intersect_rays sizes and
    // bounds it, with `extra` entries per thread beyond the tree's own (trace_instances and trace_instance_paths: the
    // bottom trees' and an instance visit's).
    // Returns the stack's bytes per block.
    size_t batch_stack_bytes(const char* call, void* workspace, size_t workspace_bytes, size_t extra = 0) const {
        const std::string who = std::string("bvh::v2::cuda::DeviceView::") + call;
        const size_t need = trace_workspace_bytes();
        if (workspace_bytes < need || !workspace)
            throw std::length_error(who + ": a workspace of " + std::to_string(workspace ? workspace_bytes : 0) + " bytes is too small (" +
                                    std::to_string(need) + " bytes)");
        const size_t entries = depth + extra;
        const size_t smem = entries > kMaxTraceSmem ? kMaxTraceSmem + 1             // (too deep for any stack: no overflow below)
                                                    : (size_t)bvhb200::stack_entries(static_cast<uint32_t>(entries), bvhb200::kDefaultStackRound) *
                                                          bvhb200::kTraceBlock * sizeof(Index);
        if (smem > kMaxTraceSmem)
            throw std::length_error(who + ": a tree of depth " + std::to_string(depth) +
                                    (extra ? " with " + std::to_string(extra) + " more entries per ray for its instances" : std::string()) +
                                    " needs " + std::to_string(smem) + " bytes of shared-memory stack per block, more than " +
                                    std::to_string(kMaxTraceSmem));
        return smem;
    }
#if defined(__CUDACC__)
    // The launch of trace, query, trace_triangles, trace_paths, trace_instances and trace_instance_paths: the checks, then,
    // unless n == 0, the current device switched to the tree's, the run cursor reset, and one resident wave of `kernel`
    // (device_view_trace_kernel, device_view_query_kernel, device_view_triangle_kernel, device_view_path_kernel,
    // device_view_instance_kernel or device_view_instance_path_kernel) on `on_stream` with the run length and grid of
    // bvhNN_intersect_rays' persistent kernel.
    // `extra`: stack entries per thread beyond the tree's own (batch_stack_bytes).
    template <typename Fn>
    void run_batch(const char* call, void (*kernel)(const Node*, unsigned long long, unsigned long long*, uint32_t, uint32_t, uint32_t, Fn),
                   const Fn& fn, size_t n, uint32_t refill_min, uint32_t inner_budget, void* workspace, size_t workspace_bytes,
                   void* on_stream, size_t extra = 0) const {
        const size_t smem = batch_stack_bytes(call, workspace, workspace_bytes, extra);
        if (n == 0) return;
        cudaStream_t s = static_cast<cudaStream_t>(on_stream);
        int previous = 0;
        check(cudaGetDevice(&previous), "cudaGetDevice", call);
        if (previous != device) check(cudaSetDevice(device), "cudaSetDevice", call);
        int sm_count = 0, per_sm = 0;
        cudaError_t e = cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device);
        // (the limit belongs to the kernel function, shared by every caller in the process: always kMaxTraceSmem, so that a
        // concurrent batch on a shallower tree cannot lower it under this launch)
        if (e == cudaSuccess && smem > 48 * 1024)
            e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxTraceSmem);
        if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, bvhb200::kTraceBlock, smem);
        if (e == cudaSuccess) e = cudaMemsetAsync(workspace, 0, trace_workspace_bytes(), s);
        if (e == cudaSuccess) {
            const uint32_t run_rays = bvhb200::persistent_run_rays(bvhb200::kDefaultRunRays, n, sm_count);
            const unsigned long long grid = bvhb200::persistent_grid(sm_count, per_sm, n, 32, bvhb200::kTraceBlock / 32);
            kernel<<<(unsigned)grid, bvhb200::kTraceBlock, smem, s>>>(nodes, n, static_cast<unsigned long long*>(workspace), run_rays,
                                                                     refill_min, inner_budget, fn);
            e = cudaGetLastError();
        }
        if (previous != device) cudaSetDevice(previous);
        check(e, "launch", call);
    }
#endif
#if defined(__CUDACC__)
    static void check(cudaError_t e, const char* what, const char* call = "traverse_bottom_up") {
        if (e != cudaSuccess)
            throw std::runtime_error(std::string("bvh::v2::cuda::DeviceView::") + call + ": " + what + ": " + cudaGetErrorString(e));
    }
#endif
    BVH_HD static void load(const Ray& ray, bvhb200::RayCtx<T>& r) { detail::load_ray<T>(ray, r); }
};

// An instance record of the mesh `view` (which must have triangles) placed by `object_to_world` (12 values, 3 x 4
// row-major), on the host or the device.  world_to_object is NaN and root_index 0 until prepare_instances writes them.
template <typename T> BVH_HD Instance<T> make_instance(const DeviceView<T>& view, const T* object_to_world) {
    using R = bvhb200::Real<T>;
    Instance<T> rec;
    rec.nodes = view.nodes; rec.prim_ids = view.prim_ids; rec.tris = view.tris;
    rec.root_index = 0;                 // (prepare_instances reads it: on the GPU the nodes are not host memory)
    rec.depth = static_cast<uint32_t>(view.depth);
    for (int k = 0; k < 12; ++k) {
        rec.object_to_world[k] = object_to_world[k];
        rec.world_to_object[k] = R::from_bits(~(typename R::UInt)0 >> 1);
    }
    return rec;
}

// For every record of `instances` (one thread each, stream-ordered on `stream`, no host synchronisation): its
// root index and world_to_object, and in bboxes[i] / centers[i] (device arrays of instances.count) the world box of its bottom root box
// and that box's centre, ready for bvhNN_build_boxes or bvhNN_refit_boxes with BVH_DEVICE_POINTERS.  See
// detail::prepare_instance for the arithmetic and the bound.  A matrix without an inverse gets an empty box, so the top
// tree never reaches it, and a NaN world_to_object, so trace_instances skips it in a leaf it shares.  The current device
// must be the records'.  A failed launch throws std::runtime_error.  Compiled as plain host C++, the records are
// prepared serially in place.
template <typename T>
void prepare_instances(const Instances<T>& instances, typename detail::ViewTypes<T>::BBox* bboxes,
                       typename detail::ViewTypes<T>::Vec* centers, void* stream = nullptr) {
    if (instances.count == 0) return;
    if (!instances.records || !bboxes || !centers)
        throw std::invalid_argument("bvh::v2::cuda::prepare_instances: null records, boxes or centres");
#if defined(__CUDACC__)
    const unsigned block = 128, grid = (unsigned)((instances.count + block - 1) / block);
    prepare_instances_kernel<T><<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(instances.records, instances.count, bboxes, centers);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
        throw std::runtime_error(std::string("bvh::v2::cuda::prepare_instances: launch: ") + cudaGetErrorString(e));
#else
    (void)stream;
    for (size_t i = 0; i < instances.count; ++i) detail::prepare_instance<T>(instances.records[i], bboxes[i], centers[i]);
#endif
}

// A motion record of the mesh `view` (which must have triangles) placed by `key0` at time 0 and `key1` at time 1 (12
// values each, 3 x 4 row-major), on the host or the device.  root_index is 0 until prepare_motion_instances writes it.
template <typename T> BVH_HD MotionInstance<T> make_motion_instance(const DeviceView<T>& view, const T* key0, const T* key1) {
    MotionInstance<T> rec;
    rec.nodes = view.nodes; rec.prim_ids = view.prim_ids; rec.tris = view.tris;
    rec.root_index = 0;
    rec.depth = static_cast<uint32_t>(view.depth);
    for (int k = 0; k < 12; ++k) {
        rec.object_to_world[0][k] = key0[k];
        rec.object_to_world[1][k] = key1[k];
    }
    return rec;
}

// prepare_instances for motion records (one thread each, stream-ordered on `stream`, no host synchronisation): every
// root index, and in bboxes[i] / centers[i] a world box that holds record i's bottom root box at every time of the
// shutter, and its centre, ready for bvhNN_build_boxes or bvhNN_refit_boxes with BVH_DEVICE_POINTERS.  See
// detail::prepare_motion_instance for the bound.  A key with a non-finite entry gives an empty box; a key without an
// inverse does not (the rays at times where the placement has none skip the record).  The current device must be the
// records'.  A failed launch throws std::runtime_error.  Compiled as plain host C++, the records are prepared serially
// in place.
template <typename T>
void prepare_motion_instances(const MotionInstances<T>& instances, typename detail::ViewTypes<T>::BBox* bboxes,
                              typename detail::ViewTypes<T>::Vec* centers, void* stream = nullptr) {
    if (instances.count == 0) return;
    if (!instances.records || !bboxes || !centers)
        throw std::invalid_argument("bvh::v2::cuda::prepare_motion_instances: null records, boxes or centres");
#if defined(__CUDACC__)
    const unsigned block = 128, grid = (unsigned)((instances.count + block - 1) / block);
    prepare_motion_instances_kernel<T><<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(instances.records, instances.count, bboxes,
                                                                                           centers);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
        throw std::runtime_error(std::string("bvh::v2::cuda::prepare_motion_instances: launch: ") + cudaGetErrorString(e));
#else
    (void)stream;
    for (size_t i = 0; i < instances.count; ++i) detail::prepare_motion_instance<T>(instances.records[i], bboxes[i], centers[i]);
#endif
}

// A deforming-scene record of the mesh `view` placed by `key0` at time 0 and `key1` at time 1 (12 values each, 3 x 4
// row-major), on the host.  Without motion_tris the bottom is static (the view must have triangles); with them it
// deforms, on the view's tree refitted over prepare_motion_triangles' boxes or, with motion_nodes, on those nodes (the
// view needs no triangles).  Throws std::invalid_argument for a static bottom whose view has no triangles, null keys
// or motion nodes, motion_tris.count other than view.prim_count or motion_nodes.node_count other than
// view.node_count.  root_index is 0 until
// prepare_deforming_instances writes it.
namespace detail {
// make_deforming_instance's record of `view` under the keys, before its bottom kind is set (a static bottom)
template <typename T> DeformingInstance<T> deforming_record(const DeviceView<T>& view, const T* key0, const T* key1) {
    DeformingInstance<T> rec;
    rec.nodes = view.nodes; rec.prim_ids = view.prim_ids; rec.tris = view.tris;
    rec.root_index = 0;
    rec.depth = static_cast<uint32_t>(view.depth);
    for (int k = 0; k < 12; ++k) {
        rec.object_to_world[0][k] = key0[k];
        rec.object_to_world[1][k] = key1[k];
    }
    rec.vertices[0] = rec.vertices[1] = nullptr;
    rec.motion_nodes = nullptr;
    return rec;
}
}
template <typename T> DeformingInstance<T> make_deforming_instance(const DeviceView<T>& view, const T* key0, const T* key1) {
    if (!view.tris)
        throw std::invalid_argument("bvh::v2::cuda::make_deforming_instance: a static bottom needs a view with triangles (built from boxes)");
    return detail::deforming_record(view, key0, key1);
}
template <typename T>
DeformingInstance<T> make_deforming_instance(const DeviceView<T>& view, const T* key0, const T* key1, const MotionTriangles<T>& motion_tris) {
    const std::string who = "bvh::v2::cuda::make_deforming_instance: ";
    if (!motion_tris.vertices[0] || !motion_tris.vertices[1]) throw std::invalid_argument(who + "a null vertex key");
    if (motion_tris.count != view.prim_count)
        throw std::invalid_argument(who + std::to_string(motion_tris.count) + " triangles for a tree of " + std::to_string(view.prim_count) +
                                    " primitives");
    DeformingInstance<T> rec = detail::deforming_record(view, key0, key1);
    rec.vertices[0] = motion_tris.vertices[0];
    rec.vertices[1] = motion_tris.vertices[1];
    return rec;
}
template <typename T>
DeformingInstance<T> make_deforming_instance(const DeviceView<T>& view, const T* key0, const T* key1, const MotionTriangles<T>& motion_tris,
                                             const MotionNodes<T>& motion_nodes) {
    const std::string who = "bvh::v2::cuda::make_deforming_instance: ";
    if (!motion_nodes.nodes) throw std::invalid_argument(who + "a null motion-node pointer");
    if (motion_nodes.node_count != view.node_count)
        throw std::invalid_argument(who + "motion nodes of " + std::to_string(motion_nodes.node_count) + " nodes for a tree of " +
                                    std::to_string(view.node_count) + " nodes");
    DeformingInstance<T> rec = make_deforming_instance(view, key0, key1, motion_tris);
    rec.motion_nodes = motion_nodes.nodes;
    return rec;
}

// prepare_motion_instances for deforming-scene records (one thread each, stream-ordered on `stream`, no host
// synchronisation): every root index (the root motion node's for a bottom with motion nodes, otherwise the view's), and
// in bboxes[i] / centers[i] a world box that holds every finite triangle of record i's bottom at every time of the
// shutter under its placement at that time, and its centre, ready for bvhNN_build_boxes or bvhNN_refit_boxes with
// BVH_DEVICE_POINTERS.  See detail::prepare_deforming_instance for the bottom box and the argument.  Each deforming
// bottom's own step (prepare_motion_triangles and bvhNN_refit_boxes, or prepare_motion_nodes) must come first on the
// stream.  The current device must be the records'.  A failed launch throws std::runtime_error.  Compiled as plain
// host C++, the records are prepared serially in place.
template <typename T>
void prepare_deforming_instances(const DeformingInstances<T>& instances, typename detail::ViewTypes<T>::BBox* bboxes,
                                 typename detail::ViewTypes<T>::Vec* centers, void* stream = nullptr) {
    if (instances.count == 0) return;
    if (!instances.records || !bboxes || !centers)
        throw std::invalid_argument("bvh::v2::cuda::prepare_deforming_instances: null records, boxes or centres");
#if defined(__CUDACC__)
    const unsigned block = 128, grid = (unsigned)((instances.count + block - 1) / block);
    prepare_deforming_instances_kernel<T><<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(instances.records, instances.count, bboxes,
                                                                                              centers);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
        throw std::runtime_error(std::string("bvh::v2::cuda::prepare_deforming_instances: launch: ") + cudaGetErrorString(e));
#else
    (void)stream;
    for (size_t i = 0; i < instances.count; ++i) detail::prepare_deforming_instance<T>(instances.records[i], bboxes[i], centers[i]);
#endif
}

// For every triangle of a deforming mesh (one thread each, stream-ordered on `stream`, no host synchronisation): in
// bboxes[id] / centers[id] (device arrays of tris.count, original order) a box that holds triangle_at(tris, id, tau) at
// every tau of the shutter, and the centre of the triangle at 0.5, ready for bvhNN_build_boxes or bvhNN_refit_boxes with
// BVH_DEVICE_POINTERS.  See detail::prepare_motion_triangle for the bound; with equal keys, box and centre are
// tri_bounds_center's of the key bit for bit.  A key with a non-finite entry gives an empty box.  The current device must
// be the keys'.  A null pointer throws std::invalid_argument, a failed launch std::runtime_error.  Compiled as plain host
// C++, the triangles are prepared serially.
template <typename T>
void prepare_motion_triangles(const MotionTriangles<T>& tris, typename detail::ViewTypes<T>::BBox* bboxes,
                              typename detail::ViewTypes<T>::Vec* centers, void* stream = nullptr) {
    if (tris.count == 0) return;
    if (!tris.vertices[0] || !tris.vertices[1] || !bboxes || !centers)
        throw std::invalid_argument("bvh::v2::cuda::prepare_motion_triangles: null keys, boxes or centres");
#if defined(__CUDACC__)
    const unsigned block = 128, grid = (unsigned)((tris.count + block - 1) / block);
    prepare_motion_triangles_kernel<T><<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(tris, bboxes, centers);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
        throw std::runtime_error(std::string("bvh::v2::cuda::prepare_motion_triangles: launch: ") + cudaGetErrorString(e));
#else
    (void)stream;
    for (size_t i = 0; i < tris.count; ++i) detail::prepare_motion_triangle<T>(tris, i, bboxes[i], centers[i]);
#endif
}

// The motion nodes of `view`'s topology for a deforming mesh (stream-ordered on `stream`, the view's by default, no host
// synchronisation): into out[1 .. view.node_count] (a device array of view.node_count + 1 records; slot 0 is not
// written) each node's bounds at time 0 and at time 1 from the two vertex keys, and its packed index, for the
// motion-node forms of trace_triangles and trace_paths.  One pass of view.traverse_bottom_up (its two kernels, on
// `workspace` of view.bottom_up_workspace_bytes() bytes); see detail::MotionNodeBuilder for the boxes and the widening
// bound.  With equal keys both keys of every record are the view's node bounds after bvhNN_refit_boxes over
// prepare_motion_triangles' boxes, bit for bit.  The topology is the view's: build it once (bvhNN_build_boxes over
// prepare_motion_triangles' boxes) and call this once per frame.  A null pointer or a triangle count other than the
// tree's throws std::invalid_argument, a small workspace std::length_error, a failed launch std::runtime_error, each
// naming prepare_motion_nodes.  Compiled as plain host C++, the pass runs serially.
template <typename T>
void prepare_motion_nodes(const DeviceView<T>& view, const MotionTriangles<T>& tris, MotionNode<T>* out, void* workspace,
                          size_t workspace_bytes, void* stream) {
    const std::string who = "bvh::v2::cuda::prepare_motion_nodes: ";
    if (!tris.vertices[0] || !tris.vertices[1] || !out) throw std::invalid_argument(who + "null keys or motion nodes");
    if (tris.count != view.prim_count)
        throw std::invalid_argument(who + std::to_string(tris.count) + " triangles for a tree of " + std::to_string(view.prim_count) +
                                    " primitives");
    const size_t need = view.bottom_up_workspace_bytes();
    if (workspace_bytes < need || !workspace)
        throw std::length_error(who + "a workspace of " + std::to_string(workspace ? workspace_bytes : 0) + " bytes is too small for " +
                                std::to_string(view.node_count) + " nodes (" + std::to_string(need) + " bytes)");
    const detail::MotionNodeBuilder<T> builder { view.nodes, view.prim_ids, tris, out };
    try {
        view.traverse_bottom_up(workspace, workspace_bytes, builder, builder, stream);
    } catch (const std::runtime_error& e) {
        throw std::runtime_error(who + e.what());
    }
}
template <typename T>
void prepare_motion_nodes(const DeviceView<T>& view, const MotionTriangles<T>& tris, MotionNode<T>* out, void* workspace,
                          size_t workspace_bytes) {
    prepare_motion_nodes(view, tris, out, workspace, workspace_bytes, view.stream);
}

} // namespace bvh::v2::cuda
