#!/usr/bin/env python
"""Records tests/golden/ref_indices.npz: the reference's own rasterize_to_indices_3dgs op on the garden crop at
256 x 256 with two cameras, for tests/test_indices_gpu.py.  Needs a GPU and the build of the reference's CUDA operators
in oracle/_ref/ (oracle/build_ref.py).

    python tests/golden/make_ref_indices_golden.py [OUT.npz]

The inputs (projected with gsplat_b200, intersected with its ellipse test) are stored with the outputs, so that the
comparison does not depend on the projection staying bit-identical.  Cases: the full range with T = 1, the batches
[1, 3) with T = 1, and the full range from seeded per-pixel transmittances in [1e-3, 1] (regenerated from the stored
seed by the test).  Per case the reference's pairs are stored as per-pixel counts and gaussian ids (its output is
pixel-major, front to back).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

W = H = 256
N_MAX = 8000
CASES = {"full": (0, 2**30, -1), "range_1_3": (1, 3, -1), "given_t": (0, 2**30, 7)}


def transmittances(seed, shape):
    """T = 1 for seed < 0, else seeded log-uniform values in [1e-3, 1]"""
    if seed < 0:
        return np.ones(shape, np.float32)
    return np.exp(np.random.RandomState(seed).uniform(np.log(1e-3), 0.0, shape)).astype(np.float32)


def main():
    import torch

    import gsplat_b200
    from oracle import refcuda
    from tests.test_indices_gpu import _n, garden_view

    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "ref_indices.npz")
    ops = refcuda.load_ops()
    v = garden_view(gsplat_b200, W, H, batch=(1, 2), n_max=N_MAX)
    sq = lambda t: t.reshape(t.shape[1:])  # noqa: E731  (image dims [1, 2] -> [2])
    m2, con, op, off = (sq(v[k]) for k in ("means2d", "conics", "opacities", "isect_offsets"))
    fl = v["flatten_ids"]
    N = m2.shape[-2]
    assert N < 65536
    arrays = dict(W=W, H=H, means2d=_n(m2), conics=_n(con), opacities=_n(op), isect_offsets=_n(off), flatten_ids=_n(fl),
                  cases=np.array(list(CASES)))
    for name, (rs, re_, seed) in CASES.items():
        T = torch.from_numpy(transmittances(seed, (2, H, W))).cuda()
        g, p, i = ops.rasterize_to_indices_3dgs(rs, re_, T, m2, con, op, W, H, 16, off, fl)
        lin = _n(i) * H * W + _n(p)
        assert (np.diff(lin) >= 0).all(), "the reference's output is pixel-major"
        arrays[f"{name}/range"] = np.array([rs, re_], np.int64)
        arrays[f"{name}/t_seed"] = np.array(seed, np.int64)
        arrays[f"{name}/counts"] = np.bincount(lin, minlength=2 * H * W).astype(np.uint16)
        arrays[f"{name}/gaussian_ids"] = _n(g).astype(np.uint16)
        print(f"{name}: {len(lin)} pairs")
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **arrays)
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
