"""ctypes binding of ``libbvh_c.so`` — the host-side mirror of the reference interface used by the
tests and ``bench.py``.

Names follow the reference: :class:`Bvh` is ``bvh::v2::Bvh<Node<T,3>>`` (reference bvh.h:17-89) as the
C shim exposes it (reference c_api/bvh.h:90-295) plus the batched GPU entry points of
``include/bvh_b200.h``.  There is no CPU fallback here: if the CUDA library is missing or no device is
visible, the batched calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("BVH_B200_LIB") or os.path.join(HERE, "libbvh_c.so")     # (the override: A/B builds of experiments)

ANY_HIT = 1 << 0
ROBUST = 1 << 1
TIE_LAST_VISITED = 1 << 2
DEVICE_POINTERS = 1 << 3
KERNEL_SIMPLE = 1 << 8
KERNEL_NO_TMA = 1 << 9
KERNEL_TMA = 1 << 10
KERNEL_PAIR = 1 << 11
KERNEL_WIDE = 1 << 12
SORT_RAYS = 1 << 13
KERNELS = (KERNEL_PAIR, KERNEL_NO_TMA, KERNEL_TMA, KERNEL_SIMPLE)
INVALID_ID = 0xFFFFFFFF

QUALITY = {"low": 0, "medium": 1, "high": 2}

HIT3F = np.dtype([("prim_id", np.uint32), ("t", np.float32), ("u", np.float32), ("v", np.float32)])
HIT3D = np.dtype([("prim_id", np.uint64), ("t", np.float64), ("u", np.float64), ("v", np.float64)])
STATS = np.dtype([("inner_steps", np.uint32), ("leaves", np.uint32), ("prim_tests", np.uint32)])


class BuildConfig(C.Structure):
    """``struct bvh_build_config`` (reference c_api/bvh.h:53-58)."""
    _fields_ = [("quality", C.c_int), ("min_leaf_size", C.c_size_t), ("max_leaf_size", C.c_size_t),
                ("parallel_threshold", C.c_size_t)]


class DeviceView(C.Structure):
    """``struct bvh_device_view3f`` / ``bvh_device_view3d`` (include/bvh_b200.h): the same layout for both."""
    _fields_ = [("device", C.c_int), ("stream", C.c_void_p), ("nodes", C.c_void_p), ("prim_ids", C.c_void_p),
                ("tris", C.c_void_p), ("node_count", C.c_size_t), ("prim_count", C.c_size_t), ("depth", C.c_size_t)]


class BvhError(RuntimeError):
    pass


_lib = None


def lib() -> C.CDLL:
    """Loads the CUDA library; fails loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise BvhError(f"{LIB_PATH} is missing: build it with `python -m bvh_b200.build_ext` "
                       "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    P, SZ, U = C.c_void_p, C.c_size_t, C.c_uint
    L.bvh_last_error.restype = C.c_char_p
    L.bvh_cuda_device_count.restype = C.c_int
    L.bvh_cuda_set_device.argtypes = [C.c_int]
    L.bvh_cuda_set_stream.argtypes = [P]
    L.bvh_cuda_reset_stream.argtypes = []
    L.bvh_host_alloc.restype = P
    L.bvh_host_alloc.argtypes = [SZ]
    L.bvh_host_free.argtypes = [P]
    L.bvh_cuda_trim.restype = C.c_int
    L.bvh_cuda_trim.argtypes = [C.c_int]
    L.bvh_set_option.restype = C.c_int
    L.bvh_set_option.argtypes = [C.c_char_p, C.c_long]
    L.bvh_thread_pool_create.restype = P
    L.bvh_thread_pool_create.argtypes = [SZ]
    L.bvh_thread_pool_destroy.argtypes = [P]
    for s in ("3f", "3d"):
        f = lambda name: getattr(L, f"bvh{s}_{name}")
        f("build").restype = P
        f("build").argtypes = [P, P, P, SZ, C.POINTER(BuildConfig)]
        f("build_triangles").restype = P
        f("build_triangles").argtypes = [P, SZ, C.POINTER(BuildConfig), U]
        f("destroy").argtypes = [P]
        f("get_node").restype = P
        f("get_node").argtypes = [P, SZ]
        f("get_prim_id").restype = SZ
        f("get_prim_id").argtypes = [P, SZ]
        f("get_prim_count").restype = SZ
        f("get_prim_count").argtypes = [P]
        f("get_node_count").restype = SZ
        f("get_node_count").argtypes = [P]
        f("refit").argtypes = [P]
        f("optimize").argtypes = [P, P]
        f("append_node").argtypes = [P]
        f("remove_last_node").argtypes = [P]
        f("set_triangles").restype = C.c_int
        f("set_triangles").argtypes = [P, P, SZ, U]
        f("refit_triangles").restype = C.c_int
        f("refit_triangles").argtypes = [P, P, SZ, U]
        f("intersect_rays").restype = C.c_int
        f("intersect_rays").argtypes = [P, P, SZ, P, U]
        f("intersect_rays_gather").restype = C.c_int
        f("intersect_rays_gather").argtypes = [P, P, SZ, P, C.POINTER(C.c_void_p), C.c_int, SZ, P, U]
        f("intersect_rays_stats").restype = C.c_int
        f("intersect_rays_stats").argtypes = [P, P, SZ, P, P, U]
        f("sync").restype = C.c_int
        f("sync").argtypes = [P]
        f("get_depth").restype = SZ
        f("get_depth").argtypes = [P]
        f("get_property").restype = SZ
        f("get_property").argtypes = [P, C.c_int]
        f("get_prim_ids").restype = P
        f("get_prim_ids").argtypes = [P]
        f("get_device_view").restype = C.c_int
        f("get_device_view").argtypes = [P, C.POINTER(DeviceView)]
        for name in ("intersect_ray", "intersect_ray_any", "intersect_ray_robust", "intersect_ray_any_robust"):
            f(name).argtypes = [P, P, P]
        n = lambda name: getattr(L, f"bvh_node{s}_{name}")
        n("is_leaf").restype = C.c_bool
        n("is_leaf").argtypes = [P]
        n("get_prim_count").restype = SZ
        n("get_prim_count").argtypes = [P]
        n("get_first_id").restype = SZ
        n("get_first_id").argtypes = [P]
        n("set_prim_count").argtypes = [P, SZ]
        n("set_first_id").argtypes = [P, SZ]
    _lib = L
    return L


def last_error() -> str:
    return lib().bvh_last_error().decode()


def device_count() -> int:
    return lib().bvh_cuda_device_count()


def set_device(device: int) -> None:
    if lib().bvh_cuda_set_device(device):
        raise BvhError(last_error())


def set_stream(cuda_stream: int | None) -> None:
    """Use a caller-owned CUDA stream (e.g. ``torch.cuda.current_stream().cuda_stream``; 0 is the legacy
    default stream) for handles created from now on; ``None`` restores one private stream per handle."""
    if cuda_stream is None:
        lib().bvh_cuda_reset_stream()
    else:
        lib().bvh_cuda_set_stream(C.c_void_p(int(cuda_stream)))


def set_option(name: str, value: int) -> None:
    """``bvh_set_option``: process-wide experiment / test switches (``include/bvh_b200.h``)."""
    if lib().bvh_set_option(name.encode(), int(value)):
        raise BvhError(last_error())


def trim(device: int = 0) -> None:
    """Hands the library's cached device memory back to the driver (``bvh_cuda_trim``)."""
    if lib().bvh_cuda_trim(device):
        raise BvhError(last_error())


PROPERTIES = {"depth": 0, "node_slots": 1, "morton_bits": 2, "quality": 3, "treelets": 4, "wide_nodes": 5,
              "last_kernel": 6, "stream": 7}
KERNEL_NAMES = {0: None, 1: "trace_persistent_kernel<kTma=true>", 2: "trace_persistent_kernel<kTma=false>",
                3: "trace_simple_kernel", 4: "trace_simple_kernel<kStats=true>", 5: "trace_pair_kernel", 6: "trace_wide_kernel"}


def _sfx(dtype) -> str:
    dtype = np.dtype(dtype)
    if dtype == np.float32:
        return "3f"
    if dtype == np.float64:
        return "3d"
    raise TypeError(f"unsupported scalar type {dtype}")


def _config(quality, min_leaf_size, max_leaf_size):
    if quality is None and min_leaf_size is None and max_leaf_size is None:
        return None
    return C.byref(BuildConfig(QUALITY.get(quality, 2) if isinstance(quality, str) or quality is None else int(quality),
                               1 if min_leaf_size is None else min_leaf_size,
                               8 if max_leaf_size is None else max_leaf_size, 1024))


def _addr(x):
    """numpy array -> host address; int -> address passed through (device pointer / pinned buffer)."""
    if isinstance(x, np.ndarray):
        return C.c_void_p(x.ctypes.data)
    return C.c_void_p(int(x))


class Bvh:
    """A BVH handle (``struct bvh3f`` / ``struct bvh3d``)."""

    def __init__(self, handle, dtype):
        if not handle:
            raise BvhError(last_error() or "BVH construction failed")
        self.handle = handle
        self.dtype = np.dtype(dtype)
        self.s = _sfx(dtype)

    def _f(self, name):
        return getattr(lib(), f"bvh{self.s}_{name}")

    # -- construction ---------------------------------------------------------------------------
    @classmethod
    def build(cls, bboxes: np.ndarray, centers: np.ndarray, quality=None, min_leaf_size=None,
              max_leaf_size=None, thread_pool=None) -> "Bvh":
        """``bvhNN_build`` (reference c_api/bvh.h:99-125): boxes are ``(n, 6)`` as ``min3, max3``
        (``struct bvh_bbox3f``), centres ``(n, 3)``.  The thread pool is accepted and ignored."""
        bboxes = np.ascontiguousarray(bboxes)
        centers = np.ascontiguousarray(centers, dtype=bboxes.dtype)
        s = _sfx(bboxes.dtype)
        h = getattr(lib(), f"bvh{s}_build")(thread_pool, _addr(bboxes), _addr(centers), bboxes.shape[0],
                                            _config(quality, min_leaf_size, max_leaf_size))
        return cls(h, bboxes.dtype)

    @classmethod
    def build_triangles(cls, vertices, count: int | None = None, dtype=None, quality=None,
                        min_leaf_size=None, max_leaf_size=None, flags: int = 0) -> "Bvh":
        """``bvhNN_build_triangles``: ``vertices`` is ``(n, 9)`` (or a device pointer with
        ``flags=DEVICE_POINTERS`` plus ``count`` and ``dtype``)."""
        if isinstance(vertices, np.ndarray):
            vertices = np.ascontiguousarray(vertices)
            count, dtype = vertices.shape[0], vertices.dtype
        s = _sfx(dtype)
        h = getattr(lib(), f"bvh{s}_build_triangles")(_addr(vertices), count,
                                                      _config(quality, min_leaf_size, max_leaf_size), flags)
        bvh = cls(h, dtype)
        bvh._keep = vertices
        return bvh

    def set_triangles(self, vertices, flags: int = 0) -> None:
        n = vertices.shape[0] if isinstance(vertices, np.ndarray) else self.prim_count
        if isinstance(vertices, np.ndarray):
            vertices = np.ascontiguousarray(vertices, dtype=self.dtype)
        if self._f("set_triangles")(self.handle, _addr(vertices), n, flags):
            raise BvhError(last_error())

    def refit_triangles(self, vertices, flags: int = 0) -> None:
        """``bvhNN_refit_triangles``: GPU refit after the vertices moved (same count and order)."""
        n = vertices.shape[0] if isinstance(vertices, np.ndarray) else self.prim_count
        if isinstance(vertices, np.ndarray):
            vertices = np.ascontiguousarray(vertices, dtype=self.dtype)
        if self._f("refit_triangles")(self.handle, _addr(vertices), n, flags):
            raise BvhError(last_error())

    def destroy(self) -> None:
        if self.handle:
            self._f("destroy")(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass

    # -- batched traversal ----------------------------------------------------------------------
    def intersect_rays(self, rays, count: int | None = None, hits=None, flags: int = 0, stats: bool = False):
        """``bvhNN_intersect_rays``.  With numpy rays returns a structured hit array (and the per-ray
        counters when ``stats``); with device pointers (``flags & DEVICE_POINTERS``) writes into ``hits``."""
        hit_dtype = HIT3F if self.s == "3f" else HIT3D
        if isinstance(rays, np.ndarray):
            rays = np.ascontiguousarray(rays, dtype=self.dtype)
            count = rays.shape[0]
            if hits is None:
                hits = np.empty(count, hit_dtype)
        st = np.zeros(count, STATS) if stats else None
        if stats:
            rc = self._f("intersect_rays_stats")(self.handle, _addr(rays), count, _addr(hits), _addr(st), flags)
        else:
            rc = self._f("intersect_rays")(self.handle, _addr(rays), count, _addr(hits), flags)
        if rc:
            raise BvhError(last_error())
        return (hits, st) if stats else hits

    def intersect_rays_gather(self, rays_ptr: int, count: int, gathered_ptrs, shard_offset: int, hits_ptr: int = 0,
                              multicast_ptr: int = 0, flags: int = 0) -> None:
        """``bvhNN_intersect_rays_gather``: trace a device-resident shard and let the kernel store each hit
        record into the gathered array of every rank (``gathered_ptrs[r]``: that array as mapped here)."""
        arr = (C.c_void_p * len(gathered_ptrs))(*[int(p) for p in gathered_ptrs])
        rc = self._f("intersect_rays_gather")(self.handle, C.c_void_p(int(rays_ptr)), count,
                                              C.c_void_p(int(hits_ptr)) if hits_ptr else None, arr, len(gathered_ptrs),
                                              shard_offset, C.c_void_p(int(multicast_ptr)) if multicast_ptr else None, flags)
        if rc:
            raise BvhError(last_error())

    def sync(self) -> None:
        if self._f("sync")(self.handle):
            raise BvhError(last_error())

    def device_view(self) -> dict:
        """``bvhNN_get_device_view``: the device tree for CUDA kernels of your own (include/bvh/v2/cuda/intersect.cuh), as
        ints: device, stream, the device addresses nodes / prim_ids / tris (0 without triangles), node_count,
        prim_count and depth.  The addresses stay valid until the tree is rebuilt, re-uploaded after a mirror edit or
        destroyed, and tris until set_triangles."""
        v = DeviceView()
        if self._f("get_device_view")(self.handle, C.byref(v)):
            raise BvhError(last_error())
        return {name: int(getattr(v, name) or 0) for name, _ in DeviceView._fields_}

    # -- reference-style introspection (host mirror) -------------------------------------------
    @property
    def prim_count(self) -> int:
        return self._f("get_prim_count")(self.handle)

    @property
    def node_count(self) -> int:
        return self._f("get_node_count")(self.handle)

    @property
    def depth(self) -> int:
        return self._f("get_depth")(self.handle)

    def get_property(self, name: str) -> int:
        v = self._f("get_property")(self.handle, PROPERTIES[name])
        if v == C.c_size_t(-1).value:
            raise BvhError(last_error() or f"unknown property {name}")
        return v

    def properties(self) -> dict:
        """Provenance of the device tree and the kernel of the last batched call (``bvhNN_get_property``)."""
        p = {k: self.get_property(k) for k in PROPERTIES}
        q = p["quality"] if p["quality"] < 3 else None
        p["last_kernel"] = KERNEL_NAMES.get(p["last_kernel"])
        bits = p["morton_bits"]
        if bits:
            p["pipeline"] = (f"LBVH ({bits}-bit Morton, SAH leaf collapse, max_leaf_size 8)"
                             + (f" + SAH treelet pass ({p['treelets']} subtrees of <= 64 primitives)" if p["treelets"] else "")
                             + f", quality {('low', 'medium', 'high')[q] if q is not None else '?'}")
        else:
            p["pipeline"] = "tree uploaded from the host mirror"
        return p

    def arrays(self):
        """(bounds[n,6] as minx,maxx,miny,maxy,minz,maxz; index_values[n] u64; prim_ids[p] u64) read
        through ``bvhNN_get_node`` / ``bvhNN_get_prim_id`` — the mirror is the reference's Node array,
        so the whole block is viewed at once through the pointer to node 0."""
        n, p = self.node_count, self.prim_count
        if n == 0:
            raise BvhError(last_error())
        base = self._f("get_node")(self.handle, 0)
        if self.s == "3f":
            rec = np.dtype([("bounds", np.float32, 6), ("index", np.uint32)])
        else:
            rec = np.dtype([("bounds", np.float64, 6), ("index", np.uint64)])
        buf = (C.c_char * (n * rec.itemsize)).from_address(base)
        nodes = np.frombuffer(buf, dtype=rec, count=n)
        bounds = nodes["bounds"].copy()
        index_values = nodes["index"].astype(np.uint64)
        base_ids = self._f("get_prim_ids")(self.handle)
        if not base_ids:
            raise BvhError(last_error())
        ids = np.frombuffer((C.c_char * (p * 8)).from_address(base_ids), dtype=np.uint64, count=p).copy()
        return bounds, index_values, ids

    def refit(self) -> None:
        self._f("refit")(self.handle)

    def save(self, path: str) -> None:
        libc = C.CDLL(None)
        libc.fopen.restype = C.c_void_p
        libc.fopen.argtypes = [C.c_char_p, C.c_char_p]
        libc.fclose.argtypes = [C.c_void_p]
        fp = libc.fopen(path.encode(), b"wb")
        if not fp:
            raise OSError(f"cannot open {path}")
        fn = self._f("save")
        fn.argtypes = [C.c_void_p, C.c_void_p]
        fn(self.handle, fp)
        libc.fclose(fp)

    @classmethod
    def load(cls, path: str, dtype=np.float32) -> "Bvh":
        libc = C.CDLL(None)
        libc.fopen.restype = C.c_void_p
        libc.fopen.argtypes = [C.c_char_p, C.c_char_p]
        libc.fclose.argtypes = [C.c_void_p]
        fp = libc.fopen(path.encode(), b"rb")
        if not fp:
            raise OSError(f"cannot open {path}")
        fn = getattr(lib(), f"bvh{_sfx(dtype)}_load")
        fn.restype = C.c_void_p
        fn.argtypes = [C.c_void_p]
        h = fn(fp)
        libc.fclose(fp)
        return cls(h, dtype)
