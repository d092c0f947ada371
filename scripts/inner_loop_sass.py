#!/usr/bin/env python
"""Instruction count and opcode histogram of a traversal kernel's inner-node loop, from the built library's SASS.

    python scripts/inner_loop_sass.py [LIB] [--kernel 'trace_persistent_kernel<float, false, false, false, false>']

The inner loop is the innermost backward branch whose body holds the four 128-bit node loads of one sibling pair
(LDG.E.128.CONSTANT).  Counting it needs no GPU: cuobjdump reads the sm_90a cubin embedded in the library.  The script
also reports the kernel's local-memory traffic (LDL / STL anywhere in the kernel), which is where spills show up.
"""
from __future__ import annotations

import argparse
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
DEFAULT_KERNEL = "trace_persistent_kernel<float, false, false, false, false>"


def functions(lib: str) -> dict[str, list[tuple[int, str]]]:
    """Demangled kernel name -> [(address, instruction text)] for every kernel in the library."""
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", lib], capture_output=True, text=True, check=True).stdout
    chunks = re.split(r"\n\s*Function : ", sass)[1:]
    mangled = [c.split("\n", 1)[0].strip() for c in chunks]
    demangled = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.split("\n")
    out = {}
    for name, chunk in zip(demangled, chunks):
        name = re.sub(r"^void |bvhb200::|\(anonymous namespace\)::", "", name)
        name = re.sub(r"\(.*\)$", "", name)                      # the parameter list
        out[name] = [(int(m.group(1), 16), m.group(2)) for m in map(INSN.match, chunk.split("\n")) if m]
    return out


def opcode(text: str) -> str:
    words = text.split()
    if words[0].startswith("@"):
        words = words[1:]
    return words[0]


def inner_loop(insns: list[tuple[int, str]]) -> list[tuple[int, str]]:
    """The smallest [target, branch] range closed by a backward BRA that contains the four node loads."""
    best = None
    for addr, text in insns:
        m = re.search(r"\bBRA\b.*\b0x([0-9a-f]+)$", text)       # (also `BRA P5, 0x...`: the branch on two predicates)
        if not m or int(m.group(1), 16) >= addr:
            continue
        body = [(a, t) for a, t in insns if int(m.group(1), 16) <= a <= addr]
        if sum(opcode(t).startswith("LDG.E.128.CONSTANT") for _, t in body) == 4 and (best is None or len(body) < len(best)):
            best = body
    if best is None:
        raise SystemExit("no backward branch encloses four LDG.E.128.CONSTANT node loads")
    return best


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("lib", nargs="?", default=os.path.join(ROOT, "bvh_b200", "libbvh_c.so"))
    ap.add_argument("--kernel", default=DEFAULT_KERNEL)
    ap.add_argument("--list", action="store_true", help="print the loop's instructions too")
    args = ap.parse_args()
    funcs = functions(args.lib)
    if args.kernel not in funcs:
        sys.exit(f"{args.kernel} not in {args.lib}; traversal kernels: " + ", ".join(sorted(f for f in funcs if f.startswith("trace_"))))
    insns = funcs[args.kernel]
    loop = inner_loop(insns)
    print(f"{args.kernel}: inner loop 0x{loop[0][0]:04x}-0x{loop[-1][0]:04x}, {len(loop)} instructions per step")
    for op, n in sorted(collections.Counter(opcode(t) for _, t in loop).items(), key=lambda kv: (-kv[1], kv[0])):
        print(f"  {n:3d}  {op}")
    local = collections.Counter(opcode(t).split(".")[0] for _, t in insns if opcode(t).split(".")[0] in ("LDL", "STL"))
    print("local memory in the kernel: " + (", ".join(f"{k} x{v}" for k, v in sorted(local.items())) or "none"))
    if args.list:
        for a, t in loop:
            print(f"  {a:04x}  {t}")


if __name__ == "__main__":
    main()
