#!/usr/bin/env python
"""Records tests/golden/ref_contrib.npz: the reference's own rasterize_num_contributing_gaussians,
rasterize_contributing_gaussian_ids and rasterize_top_contributing_gaussian_ids (K = 4) ops on the garden crop at
64 x 64 with two cameras, for tests/test_contrib_gpu.py.  Needs a GPU and the build of the reference's CUDA operators
in oracle/_ref/ (oracle/build_ref.py).

    python tests/golden/make_ref_contrib_golden.py [OUT.npz]

The inputs (projected with gsplat_b200, intersected with its ellipse test) are stored with the outputs.  The padded id
lists are stored as their valid entries only: per-pixel counts, then the ids and weights pixel-major, front to back.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

W = H = 64
N_MAX = 4000
TOP_K = 4


def main():
    import gsplat_b200
    from oracle import refcuda
    from tests.test_indices_gpu import _n, garden_view

    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "ref_contrib.npz")
    ops = refcuda.load_ops()
    v = garden_view(gsplat_b200, W, H, batch=(1, 2), n_max=N_MAX)
    sq = lambda t: t.reshape(t.shape[1:])  # noqa: E731  (image dims [1, 2] -> [2])
    m2, con, op, off = (sq(v[k]) for k in ("means2d", "conics", "opacities", "isect_offsets"))
    fl = v["flatten_ids"]
    assert m2.shape[-2] < 65536
    counts, alphas = ops.rasterize_num_contributing_gaussians(m2, con, op, off, fl, W, H, 16)
    ids, weights = ops.rasterize_contributing_gaussian_ids(m2, con, op, off, fl, W, H, 16, counts)
    top_ids, top_weights = ops.rasterize_top_contributing_gaussian_ids(m2, con, op, off, fl, W, H, 16, TOP_K)
    valid = _n(ids) >= 0
    c = _n(counts)
    assert np.array_equal(valid.sum(-1), c), "the reference's ids are its counts' pairs, then -1"
    arrays = dict(
        W=W, H=H, means2d=_n(m2), conics=_n(con), opacities=_n(op), isect_offsets=_n(off), flatten_ids=_n(fl),
        counts=c.astype(np.uint16), alphas=_n(alphas), ids=_n(ids)[valid].astype(np.uint16), weights=_n(weights)[valid],
        top_ids=_n(top_ids).astype(np.int32), top_weights=_n(top_weights),
    )
    print(f"{int(c.sum())} pairs, max count {int(c.max())}")
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **arrays)
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
