"""bvh2f_load / bvh2d_load on corrupt headers: a header that announces more nodes or primitives than the file holds
is rejected before anything is allocated, as bvh3f_load / bvh3d_load reject it, and a valid file still loads and saves
back byte for byte."""
import subprocess
import sys

import numpy as np
import pytest

from tests.helpers import reference_tree
from tests.test_c_abi_2d import OURS, Api2, scene2

# Loads one file through bvh<s>_load in a child process whose address space is capped at 2 GiB, so that a load that
# tried to allocate what a corrupt header announces would fail there instead of exhausting the machine's memory.
LOAD_IN_CHILD = r"""
import ctypes as C, resource, sys
resource.setrlimit(resource.RLIMIT_AS, (2 << 30, 2 << 30))
lib, libc = C.CDLL(sys.argv[1]), C.CDLL(None)
libc.fopen.restype = C.c_void_p; libc.fopen.argtypes = [C.c_char_p, C.c_char_p]; libc.fclose.argtypes = [C.c_void_p]
load = getattr(lib, "bvh%s_load" % sys.argv[2]); load.restype = C.c_void_p; load.argtypes = [C.c_void_p]
lib.bvh_last_error.restype = C.c_char_p
fp = libc.fopen(sys.argv[3].encode(), b"rb"); h = load(fp); libc.fclose(fp)
print("NULL" if h is None else "handle", lib.bvh_last_error().decode())
"""


@pytest.mark.parametrize("s", ["2f", "2d"])
def test_load_rejects_a_header_that_announces_more_than_the_file_holds(tmp_path, s):
    ours = Api2(OURS, s)
    boxes, _, _ = scene2(700, 3, ours.dtype)
    good = reference_tree(f"c_abi_2d_{s}", boxes, 2, ours.dtype)
    it = np.uint32 if s == "2f" else np.uint64
    node_count = int(np.frombuffer(good[:it().itemsize], it)[0])
    corrupt = {"huge": np.array([0xFFFFFFFF if s == "2f" else 1 << 40, 700], it).tobytes() + bytes(64),
               "one_node_more": np.array([node_count + 1], it).tobytes() + good[it().itemsize:]}
    for name, data in corrupt.items():
        path = tmp_path / f"{name}.bin"
        path.write_bytes(data)
        out = subprocess.run([sys.executable, "-c", LOAD_IN_CHILD, OURS, s, str(path)], capture_output=True, text=True)
        assert out.returncode == 0, out.stderr
        assert out.stdout.startswith("NULL") and "announces more nodes" in out.stdout, (name, out.stdout)
    # a valid file still loads, and saves back byte for byte
    path = tmp_path / "good.bin"
    path.write_bytes(good)
    h = ours.load(str(path))
    assert h
    ours.save(h, str(tmp_path / "again.bin"))
    ours.f("destroy")(h)
    assert (tmp_path / "again.bin").read_bytes() == good
