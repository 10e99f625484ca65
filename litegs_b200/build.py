"""Builds liblitegs_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

One translation unit per .cu, compiled in parallel, linked into a single C-ABI shared library that
depends on nothing but cudart.  ``python -m litegs_b200.build`` or ``__graft_entry__.build()``.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "liblitegs_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# the system g++ is preferred as nvcc's host compiler: a $CXX set by the environment may lack libgomp.
HOST_CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-ccbin", HOST_CXX, "--expt-relaxed-constexpr"]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers_mtime():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    return max([os.path.getmtime(h) for h in hs] + [os.path.getmtime(__file__)])


def _compile(src: str, verbose: bool) -> str:
    obj = os.path.join(OBJ, src[:-3] + ".o")
    spath = os.path.join(CSRC, src)
    if os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(spath), _headers_mtime()):
        return obj
    cmd = [NVCC, *FLAGS, "-c", spath, "-o", obj]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        sys.stderr.write(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), _sources()))
    if force or not os.path.exists(LIB) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        cmd = [NVCC, "-shared", "-ccbin", HOST_CXX, "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB, *objs,
               "-cudart", "shared"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
