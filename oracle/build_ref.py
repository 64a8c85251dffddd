#!/usr/bin/env python
"""Builds the REAL reference's 3DGS CUDA operators into oracle/_ref/gsplat_ref.so (test / bench
infrastructure only; never imported by gsplat_b200).

The sources are compiled where they lie under /root/reference/gsplat/cuda (nothing is copied into
this repository) with a recipe written here -- the reference's own build system (gsplat/cuda/build.py,
JIT via torch.utils.cpp_extension.load) is NOT run; its flag set for a "3DGS only" release build is
restated: -std=c++20 -O3 -DNDEBUG -use_fast_math -DGSPLAT_BUILD_3DGS=1 (every other module then defaults
to off, csrc/Config.h:28-60) and -DGSPLAT_NUM_CHANNELS=1,3,4 (Config.h:70-72) to keep compile time sane.
Target: sm_90a.  Only runs where the reference sources exist; the resulting .so is
git-ignored; tests/golden/make_ref_cuda_golden.py (which records tests/golden/ref_cuda.npz) and bench.py load it
with torch.ops.load_library and call torch.ops.gsplat.* directly.  The pybind module inside is named ``csrc``
(TORCH_EXTENSION_NAME), so that baseline/install_ref.py can also place a copy as the prebuilt ``gsplat/csrc.so``
the reference's Python package imports first (gsplat/cuda/_backend.py:30) -- one process must load only ONE of
the two copies (oracle/refcuda.py picks), else the TORCH_LIBRARY registration would run twice.

    python oracle/build_ref.py [-j JOBS] [--full]
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

REF = "/root/reference/gsplat/cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
OBJ = os.path.join(OUT, "obj")
LIB = os.path.join(OUT, "gsplat_ref.so")
NUM_CHANNELS = "1,3,4"


def main():
    if not os.path.isdir(REF):
        print("build_ref: /root/reference not present -- nothing to do")
        return 0
    import torch
    from torch.utils import cpp_extension as ce

    jobs = int(sys.argv[sys.argv.index("-j") + 1]) if "-j" in sys.argv else (os.cpu_count() or 4)
    os.makedirs(OBJ, exist_ok=True)
    sources = sorted(glob.glob(os.path.join(REF, "csrc", "*.cu")) + glob.glob(os.path.join(REF, "csrc", "*.cpp")))
    sources = [s for s in sources if not s.endswith("CameraWrappers.cu")] + [os.path.join(REF, "ext.cpp")]
    inc = [os.path.join(REF, "include"), os.path.join(REF, "csrc", "third_party", "glm"), os.path.join(REF, "csrc")]
    inc += ce.include_paths("cuda") if "device_type" in ce.include_paths.__code__.co_varnames else ce.include_paths(True)
    inc += [sysconfig.get_paths()["include"]]
    incf = [f"-I{p}" for p in inc]
    defs = [
        "-DTORCH_EXTENSION_NAME=csrc", "-DTORCH_API_INCLUDE_EXTENSION_H", "-DNDEBUG", "-DGSPLAT_BUILD_3DGS=1",
        "-DGSPLAT_BUILD_ADAM=1", "-DGSPLAT_BUILD_RELOC=1",
        f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}",
    ]
    cxx = ["/usr/bin/g++", "-std=c++20", "-O3", "-fPIC", "-Wno-attributes", "-Wno-unknown-pragmas", "-w",
           f"-DGSPLAT_NUM_CHANNELS={NUM_CHANNELS}"]
    nvcc = [
        "/usr/local/cuda/bin/nvcc", "-ccbin", "/usr/bin/g++", "-std=c++20", "-O3", "-use_fast_math", "--expt-relaxed-constexpr",
        "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-diag-suppress", "3189,20012,186", "-w",
        "-DGSPLAT_NUM_CHANNELS=" + NUM_CHANNELS.replace(",", "\\,"),
        "-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__", "-D__CUDA_NO_BFLOAT16_CONVERSIONS__",
        "-D__CUDA_NO_HALF2_OPERATORS__",
    ]
    # --full: the configuration the reference's own hot-path tests need to RUN rather than skip (tests/refsuite):
    #   GSPLAT_BUILD_3DGUT=1          two tests of the 3DGS path (test_basic.py test_isect / the eval3d twins) are gated on it
    #   GSPLAT_BUILD_CAMERA_WRAPPERS  tests/test_rasterization.py imports tests/test_cameras.py, which skips itself without them
    #   GSPLAT_NUM_CHANNELS           the channel counts the reference's pytest.ini builds for its tests (1,3,4,6,8,21,23,24,32,128)
    # None of this changes the 3DGS kernels that get timed; it adds instantiations.  Objects go to obj_full/.
    full = "--full" in sys.argv
    objdir = OBJ
    if full:
        defs += ["-DGSPLAT_BUILD_3DGUT=1", "-DGSPLAT_BUILD_CAMERA_WRAPPERS=1"]
        channels = "1,3,4,6,8,21,23,24,32,128"  # the reference's own test configuration (pytest.ini: NUM_CHANNELS)
        cxx[-1] = f"-DGSPLAT_NUM_CHANNELS={channels}"
        nvcc[nvcc.index("-DGSPLAT_NUM_CHANNELS=" + NUM_CHANNELS.replace(",", "\\,"))] = "-DGSPLAT_NUM_CHANNELS=" + channels.replace(",", "\\,")
        sources.insert(0, os.path.join(REF, "csrc", "CameraWrappers.cu"))
        objdir = OBJ + "_full"
        os.makedirs(objdir, exist_ok=True)
    # objects are reused only when they were compiled with the same flags (a changed -gencode rebuilds everything)
    stamp = os.path.join(objdir, "flags.txt")
    flags = "\n".join(" ".join(x) for x in (nvcc, cxx, defs, incf))
    same_flags = os.path.exists(stamp) and open(stamp).read() == flags
    cmds, objs = [], []
    for s in sources:
        o = os.path.join(objdir, os.path.basename(s) + ".o")
        objs.append(o)
        if same_flags and os.path.exists(o) and os.path.getmtime(o) > os.path.getmtime(s):
            continue
        base = nvcc if s.endswith(".cu") else cxx
        cmds.append((s, base + defs + incf + ["-c", s, "-o", o]))

    def run(item):
        s, cmd = item
        # note: nvcc splits -D values at commas, so it must RECEIVE the backslash-escaped form (no shell here)
        r = subprocess.run(cmd, capture_output=True, text=True)
        tag = "ok " if r.returncode == 0 else "ERR"
        print(f"[{tag}] {os.path.basename(s)}", flush=True)
        if r.returncode != 0:
            print(r.stderr[-3000:], flush=True)
        return r.returncode

    with ThreadPoolExecutor(max_workers=jobs) as ex:
        rcs = list(ex.map(run, cmds))
    if any(rcs):
        print("build_ref: compilation failed")
        return 1
    with open(stamp, "w") as f:
        f.write(flags)
    tlib = os.path.join(os.path.dirname(torch.__file__), "lib")
    out_lib = LIB
    link = ["/usr/bin/g++", "-shared", "-o", out_lib] + objs + [
        f"-L{tlib}", "-L/usr/local/cuda/lib64", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
        "-lcudart", f"-Wl,-rpath,{tlib}",
    ]
    r = subprocess.run(link, capture_output=True, text=True)
    if r.returncode != 0:
        print(r.stderr[-4000:])
        return 1
    print("built", out_lib, os.path.getsize(out_lib) // 1024, "kB")
    return 0


if __name__ == "__main__":
    sys.exit(main())
