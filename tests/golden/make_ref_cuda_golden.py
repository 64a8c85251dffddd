#!/usr/bin/env python
"""Records the reference outputs tests/test_gpu_vs_reference_cuda.py compares against.  Needs a GPU and a build of
the reference's CUDA operators (oracle/build_ref.py, from the reference's sources) in oracle/_ref/.

    python tests/golden/make_ref_cuda_golden.py [OUT.npz]            # its CUDA ops -> tests/golden/ref_cuda.npz
    python tests/golden/make_ref_cuda_golden.py --stock [OUT.npz]    # its stock rasterization() -> ref_cuda_stock.npz

--stock drives the reference's Python package, which oracle/refcuda.py looks for in baseline/_ref (the package
installed there with its csrc.so being the oracle/_ref build).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    import gsplat_b200
    from oracle import refcuda
    from tests import test_gpu_vs_reference_cuda as T

    stock = "--stock" in sys.argv
    args = [a for a in sys.argv[1:] if a != "--stock"]
    out = args[0] if args else (T.GOLDEN_STOCK if stock else T.GOLDEN)
    if stock:
        recorders = T.STOCK_RECORDERS(refcuda.import_package())
    else:
        recorders = T.RECORDERS(refcuda.load_ops(), gsplat_b200)
    arrays = {}
    for name, fn in recorders.items():
        for k, v in fn().items():
            arrays[f"{name}/{k}"] = v
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **arrays)
    print(out, os.path.getsize(out), "bytes,", len(arrays), "arrays")


if __name__ == "__main__":
    main()
