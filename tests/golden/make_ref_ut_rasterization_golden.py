#!/usr/bin/env python
"""Records the reference's own 3DGUT orchestrator for the tests of rasterization(with_ut=True, with_eval3d=True).

    python tests/golden/make_ref_ut_rasterization_golden.py     (GPU; needs oracle/_ref from
                                                                 python oracle/build_ref.py --full)

Writes only tests/golden/ref_ut_rasterization.npz.  The reference build's torch.ops.gsplat.rasterization_3dgs is called
with the arguments gsplat/rendering.py:601-650 passes it for rasterization(..., packed=False, tile_size=16,
with_ut=True, with_eval3d=True, render_mode="RGB+ED", sh_degree=3), on the seeded 96x64 garden crop of
make_ref_ut_golden.py with SH degree 3, two cameras and a background, for every camera of RASTER_CAMERAS.  Per camera
it records the colours and alphas, the meta radii / means2d / depths / isect_offsets / flatten_ids, and the gradients
of a seeded cotangent with respect to means, quats, scales, opacities, the SH coefficients and the backgrounds.
"""
import os
import sys

import numpy as np

from make_ref_ut_golden import CAMERA_IDS, HERE, N_GAUSS, ROOT, SCALE, H, W

# name -> (camera model, coefficients), the same coefficients for both cameras
RASTER_CAMERAS = {
    "pinhole": ("pinhole", {}),
    "pinhole_distorted": ("pinhole", {"radial": [0.08, -0.03, 0.005, 0.01, 0.0, 0.0], "tangential": [0.004, -0.003],
                                      "thin": [0.002, -0.001, 0.001, 0.0005]}),
    "fisheye_radial": ("fisheye", {"radial": [0.04, -0.01, 0.002, -0.0003]}),
}
RASTER_C, RASTER_SH_DEGREE = 2, 3


def record_rasterization():
    sys.path.insert(0, ROOT)
    import torch

    from oracle import refcuda
    from tests import scene

    ops = refcuda.load_ops()
    dev = "cuda"
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    # the crop of make_ref_ut_golden.small_scene (same seed: the SH draw comes after every other parameter), SH degree
    # 3, two cameras
    sc = scene.make_scene(n_max=N_GAUSS, sh_degree=RASTER_SH_DEGREE, seed=0)
    C = RASTER_C
    inputs = dict(means=sc["means"], quats=sc["quats"], scales=(sc["scales"] * SCALE).astype(np.float32),
                  opacities=sc["opacities"], sh=sc["sh"], viewmats=sc["viewmats"][:C],
                  Ks=scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:C].astype(np.float32))
    rng = np.random.RandomState(11)
    bg = rng.random_sample((C, 3)).astype(np.float32)
    v_rc = rng.standard_normal((C, H, W, 4)).astype(np.float32)  # RGB+ED: four channels
    v_ra = rng.standard_normal((C, H, W, 1)).astype(np.float32)
    out = dict(inputs, backgrounds=bg, v_render_colors=v_rc, v_render_alphas=v_ra, width=W, height=H,
               sh_degree=RASTER_SH_DEGREE)
    utp = torch.classes.gsplat.UnscentedTransformParameters()
    ftheta = torch.classes.gsplat.FThetaCameraDistortionParameters()
    keys = {"radial": "radial_coeffs", "tangential": "tangential_coeffs", "thin": "thin_prism_coeffs"}
    for name, (model, coeffs) in RASTER_CAMERAS.items():
        co = {keys[k]: np.tile(np.float32(v), (C, 1)) for k, v in coeffs.items()}
        for k, v in co.items():
            out[f"{name}/{k}"] = v
        ct = {k: t(v) for k, v in co.items()}
        leaves = {k: t(inputs[k]).requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "sh")}
        leaves["backgrounds"] = t(bg).requires_grad_(True)
        # the argument list of gsplat/rendering.py:601-650 for packed=False, tile_size=16, render_mode="RGB+ED",
        # rasterize_mode="classic", with_eval3d=with_ut=True, one process
        res = ops.rasterization_3dgs(
            leaves["means"], None, leaves["quats"], leaves["scales"], leaves["opacities"], leaves["sh"], t(inputs["viewmats"]),
            t(inputs["Ks"]), W, H, 16, 0.3, 0.01, 1e10, 0.0, leaves["backgrounds"], False, False, False, False, True,
            CAMERA_IDS[model], False, 32, True, RASTER_SH_DEGREE, None, -1, True, True, True, True, None, None, utp, 4,
            ct.get("radial_coeffs"), ct.get("tangential_coeffs"), ct.get("thin_prism_coeffs"), ftheta, None, None, True,
            False, False, 0, None, 1,
        )
        rc, ra = res[0], res[1]
        radii, m2, d = res[8], res[9], res[10]
        flatten_ids, isect_offsets = res[15], res[16]
        ((rc * t(v_rc)).sum() + (ra * t(v_ra)).sum()).backward()
        culled = (radii == 0).all(-1)
        # the reference leaves the float outputs of a culled row unwritten; this library zeroes them
        m2, d = m2.masked_fill(culled[..., None], 0), d.masked_fill(culled, 0)
        rec = dict(render_colors=rc, render_alphas=ra, radii=radii, means2d=m2, depths=d, isect_offsets=isect_offsets,
                   flatten_ids=flatten_ids)
        for k, v in rec.items():
            out[f"{name}/{k}"] = v.detach().cpu().numpy()
        for k, leaf in leaves.items():
            out[f"{name}/v_{k}"] = leaf.grad.detach().cpu().numpy()
        print(name, "visible", int((~culled).sum()), "pairs", flatten_ids.numel(), "alpha mean", ra.mean().item())
    np.savez_compressed(os.path.join(HERE, "ref_ut_rasterization.npz"), **out)


if __name__ == "__main__":
    record_rasterization()
