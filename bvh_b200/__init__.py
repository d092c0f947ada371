"""bvh_b200 — H100-native BVH construction and batched ray traversal behind the madmann91/bvh v2
API surface.  The compute path is hand-written CUDA for sm_90a in ``bvh_b200/csrc`` exposed through
a C ABI (``include/bvh_b200.h``); this package is the thin Python binding used by the tests and
``bench.py``.  There is no CPU fallback: importing :mod:`bvh_b200.api` without the built library
raises."""
__all__ = ["scenes"]
