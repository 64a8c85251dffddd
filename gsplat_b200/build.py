"""Builds gsplat_b200/libgsplat_b200.so in-tree with nvcc for sm_90a (no torch headers involved).

    python -m gsplat_b200.build [--force]

The library is a plain C-ABI shared object (include/gsplat_b200.h); the per-gaussian kernels are
compiled with -fmad=false so that they can be checked bit for bit against the CPU oracle.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libgsplat_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "--expt-extended-lambda"]
UNITS = {
    # file: extra flags
    "raster.cu": [],
    "pergauss.cu": ["-fmad=false"],
    "isect.cu": ["-fmad=false"],
    "sort.cu": [],
    "nvls.cu": [],
    "loss.cu": [],
    "surfel.cu": ["-fmad=false"],
    "ut.cu": ["-fmad=false"],
}
HEADERS = ["camera.cuh", "common.cuh", "gaussmath.cuh", "indices.cuh", "isect.cuh", "pixels.cuh", "rowrec.cuh", os.path.join("..", "..", "include", "gsplat_b200.h")]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def source_hash() -> str:
    """sha256 over the CUDA sources and headers the library is built from (sorted by name): compiled into the library
    (gsb200_source_hash()) so that a shipped binary can be matched against the tree it sits in."""
    import hashlib

    h = hashlib.sha256()
    names = sorted(UNITS) + sorted(os.path.basename(x) for x in HEADERS)
    for name in names:
        path = os.path.join(CSRC, name) if name != "gsplat_b200.h" else os.path.join(CSRC, "..", "..", "include", name)
        h.update(name.encode())
        with open(path, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS] + [os.path.abspath(__file__)]
    nvcc = _nvcc()
    jobs = []
    objs = []
    for unit, extra in UNITS.items():
        src = os.path.join(CSRC, unit)
        obj = os.path.join(OBJ, unit.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, [src] + hdrs):
            jobs.append([nvcc, *ARCH, *COMMON, *extra, "-c", src, "-o", obj])
    # the hash of ALL sources, in its own tiny unit so that it is refreshed whenever anything is rebuilt
    stamp_src, stamp_obj = os.path.join(OBJ, "source_hash.cu"), os.path.join(OBJ, "source_hash.o")
    digest = source_hash()
    text = f'extern "C" const char *gsb200_source_hash(void) {{ return "{digest}"; }}\n'
    if not os.path.exists(stamp_src) or open(stamp_src).read() != text:
        with open(stamp_src, "w") as f:
            f.write(text)
    objs.append(stamp_obj)
    if force or _stale(stamp_obj, [stamp_src]):
        jobs.append([nvcc, *ARCH, "-O1", "-Xcompiler", "-fPIC", "-c", stamp_src, "-o", stamp_obj])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 2)) as ex:
            list(ex.map(run, jobs))
    if force or jobs or _stale(LIB, objs):
        run([nvcc, *ARCH, "-shared", "-o", LIB, *objs, "-cudart", "static"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
