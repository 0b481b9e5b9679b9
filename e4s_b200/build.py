"""In-tree build of libe4s_b200.so (hand-written sm_90a CUDA behind the C ABI of include/e4s_b200.h).

    python -m e4s_b200.build [--force] [--verbose]

nvcc cross-compiles without a GPU.  Objects go to e4s_b200/csrc/_obj/, the shared library to
e4s_b200/libe4s_b200.so (both git-ignored build products).
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(CSRC, "_obj")
LIB = os.path.join(PKG, "libe4s_b200.so")
INCLUDE = os.path.join(os.path.dirname(PKG), "include")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--expt-relaxed-constexpr",
          "-I", INCLUDE]


def _newer(src_list, target):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in src_list)


def _compile(src, verbose, objdir=None, extra=()):
    obj = os.path.join(objdir or OBJ, os.path.basename(src)[:-3] + ".o")
    deps = [src] + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(INCLUDE, "*.h"))
    if not _newer(deps, obj):
        return obj, ""
    cmd = [NVCC] + ARCH + CFLAGS + list(extra) + ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        print(r.stderr)
    return obj, r.stderr


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    if force:
        for f in glob.glob(os.path.join(OBJ, "*.o")):
            os.remove(f)
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile(s, verbose), srcs))
    objs = [o for o, _ in results]
    log = "\n".join(l for _, l in results if l)
    if log:
        with open(os.path.join(OBJ, "ptxas.log"), "w") as f:
            f.write(log)
    if force or _newer(objs, LIB):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart", "-lcuda"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
