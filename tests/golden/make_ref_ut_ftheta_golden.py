#!/usr/bin/env python
"""Records the reference's FTheta 3DGUT for the tests.

    python tests/golden/make_ref_ut_ftheta_golden.py     (GPU; needs oracle/_ref from python oracle/build_ref.py --full)

Writes tests/golden/ref_ut_ftheta.npz and tests/golden/ref_ut_ftheta_rasterization.npz on the seeded 96x64 garden
crop of make_ref_ut_golden.py, through the calibrations of tests/golden/ftheta_calibrations.json scaled to 96 pixels
wide (tests/scene.scaled; each camera's Ks holds the scaled principal point, fx = fy = 1 unused).

ref_ut_ftheta.npz: for every calibration, both reference polynomials (ptoa: pixel distance -> angle, atop: angle ->
pixel distance) and both depth orders (z: global_z_order=True, dist: False), and for one top-to-bottom
rolling-shutter case per calibration (ptoa, dist, the end pose of make_ref_ut_rs_golden.end_poses): the reference
build's torch.ops.gsplat.projection_ut_3dgs_fused and rasterize_to_pixels_from_world_3dgs (MixedBatch): the
projection outputs the tests compare (radii, means2d, depths), the tile lists built from them
(gsplat_b200.isect_tiles / isect_offset_encode), the eval3d colour (one channel) and alphas, and the gradients of a
seeded cotangent (make_ref_ut_rs_golden.cotangents) with respect to means, quats, scales, colors, opacities and
backgrounds.  Keys: "<calibration>/<ptoa|atop>/<z|dist>[/rs]/<output>".

ref_ut_ftheta_rasterization.npz: one rasterization_3dgs record through the cross-left calibration, ptoa,
global_z_order=False: SH degree 3, RGB+ED, two cameras with distinct principal points and a background, with its
gradients.

The backgrounds and cotangents are not stored: cotangents(seed, ...) redraws them from the recorded seed.
"""
import os
import sys

import numpy as np

from make_ref_ut_golden import HERE, N_GAUSS, ROOT, SCALE, H, W, small_scene
from make_ref_ut_rs_golden import cotangents, end_poses

FTHETA = 3  # the reference's CameraModelType.FTHETA
POLYS = {"ptoa": 0, "atop": 1}
ORDERS = {"z": True, "dist": False}
COTANGENT_SEED, RASTER_COTANGENT_SEED = 13, 17
RASTER_CALIBRATION, RASTER_C, RASTER_SH_DEGREE = "cross_left_120fov", 2, 3


def ftheta_K(pp, C=1, shift=(0.0, 0.0)):
    """[C, 3, 3] intrinsics holding the principal point (camera i moved by i * shift), fx = fy = 1 (unused)."""
    K = np.zeros((C, 3, 3), np.float32)
    for i in range(C):
        K[i] = [[1, 0, pp[0] + i * shift[0]], [0, 1, pp[1] + i * shift[1]], [0, 0, 1]]
    return K


def record():
    sys.path.insert(0, ROOT)
    import torch

    import gsplat_b200 as gs
    from oracle import refcuda
    from tests import scene

    ops = refcuda.load_ops()
    dev = "cuda"
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    sc = small_scene()
    sc["colors"] = np.ascontiguousarray(sc["colors"][:, :1])
    vm_rs = end_poses(sc["viewmats"])
    bg, v_rc, v_ra = cotangents(COTANGENT_SEED, 1, 1, 1)
    out = dict(sc, viewmats_rs=vm_rs, cotangent_seed=COTANGENT_SEED, width=W, height=H)
    out.pop("Ks")
    utp = torch.classes.gsplat.UnscentedTransformParameters()
    tw, th = (W + 15) // 16, (H + 15) // 16

    def ftheta_obj(params, ref):
        return torch.classes.gsplat.FThetaCameraDistortionParameters(
            ref, params["pixeldist_to_angle_poly"], params["angle_to_pixeldist_poly"], params["max_angle"],
            params["linear_cde"])

    for cname, cal in scene.calibrations().items():
        params, pp, _ = scene.scaled(cal, W)
        K = ftheta_K(pp)
        out[f"{cname}/Ks"] = K
        cases = [(p, o, 4) for p in POLYS for o in ORDERS] + [("ptoa", "dist", 0)]
        for pname, oname, rs in cases:
            name = f"{cname}/{pname}/{oname}" + ("/rs" if rs != 4 else "")
            ft = ftheta_obj(params, POLYS[pname])
            vrs = t(vm_rs) if rs != 4 else None
            radii, m2, d, _, _ = ops.projection_ut_3dgs_fused(
                t(sc["means"]), t(sc["quats"]), t(sc["scales"]), t(sc["opacities"]), t(sc["viewmats"]), vrs, t(K),
                W, H, 0.3, 0.01, 1e10, 0.0, True, FTHETA, ORDERS[oname], utp, rs, None, None, None, ft, None, None,
            )
            culled = (radii == 0).all(-1)
            # the reference leaves the float outputs of a culled row unwritten; this library zeroes them
            m2, d = m2.masked_fill(culled[..., None], 0), d.masked_fill(culled, 0)
            _, isect_ids, flatten_ids = gs.isect_tiles(m2, radii, d, 16, tw, th)
            offsets = gs.isect_offset_encode(isect_ids, 1, tw, th)
            leaves = [t(x).requires_grad_(True) for x in (sc["means"], sc["quats"], sc["scales"], sc["colors"][None], sc["opacities"][None], bg)]
            rc, ra, *_ = ops.rasterize_to_pixels_from_world_3dgs(
                leaves[0], leaves[1], leaves[2], leaves[3], leaves[4], leaves[5], None, W, H, 16, t(sc["viewmats"]), vrs,
                t(K), FTHETA, utp, rs, None, None, None, None, ft, None, None, offsets, flatten_ids, False, False, False,
                0, True, False,
            )
            ((rc * t(v_rc)).sum() + (ra * t(v_ra)).sum()).backward()
            rec = dict(radii=radii, means2d=m2, depths=d, isect_offsets=offsets, flatten_ids=flatten_ids,
                       render_colors=rc, render_alphas=ra)
            for k, v in rec.items():
                out[f"{name}/{k}"] = v.detach().cpu().numpy()
            for k, leaf in zip(("means", "quats", "scales", "colors", "opacities", "backgrounds"), leaves):
                out[f"{name}/v_{k}"] = leaf.grad.detach().cpu().numpy()
            print(name, "visible", int((~culled).sum()), "pairs", flatten_ids.numel(), "alpha mean", float(ra.detach().mean()))
    np.savez_compressed(os.path.join(HERE, "ref_ut_ftheta.npz"), **out)

    # ---- rasterization_3dgs: SH degree 3, RGB+ED, two cameras with distinct principal points, a background
    full = scene.make_scene(n_max=N_GAUSS, sh_degree=RASTER_SH_DEGREE, seed=0)
    C = RASTER_C
    params, pp, _ = scene.scaled(scene.calibrations()[RASTER_CALIBRATION], W)
    inputs = dict(means=full["means"], quats=full["quats"], scales=(full["scales"] * SCALE).astype(np.float32),
                  opacities=full["opacities"], sh=full["sh"], viewmats=full["viewmats"][:C].astype(np.float32),
                  Ks=ftheta_K(pp, C, shift=(3.0, -2.0)))
    bg2, v_rc2, v_ra2 = cotangents(RASTER_COTANGENT_SEED, C, 3, 4)  # RGB+ED: four channels
    out = dict(inputs, width=W, height=H, cotangent_seed=RASTER_COTANGENT_SEED, sh_degree=RASTER_SH_DEGREE)
    leaves = {k: t(inputs[k]).requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "sh")}
    leaves["backgrounds"] = t(bg2).requires_grad_(True)
    res = ops.rasterization_3dgs(
        leaves["means"], None, leaves["quats"], leaves["scales"], leaves["opacities"], leaves["sh"], t(inputs["viewmats"]),
        t(inputs["Ks"]), W, H, 16, 0.3, 0.01, 1e10, 0.0, leaves["backgrounds"], False, False, False, False, True,
        FTHETA, False, 32, True, RASTER_SH_DEGREE, None, -1, True, True, True, True, None, None,
        utp, 4, None, None, None, ftheta_obj(params, 0), None, None, False, False, False, 0, None, 1,
    )
    rc, ra = res[0], res[1]
    radii, m2, d = res[8], res[9], res[10]
    ((rc * t(v_rc2)).sum() + (ra * t(v_ra2)).sum()).backward()
    culled = (radii == 0).all(-1)
    m2, d = m2.masked_fill(culled[..., None], 0), d.masked_fill(culled, 0)
    for k, v in dict(render_colors=rc, render_alphas=ra, radii=radii, means2d=m2, depths=d).items():
        out[k] = v.detach().cpu().numpy()
    for k, leaf in leaves.items():
        out[f"v_{k}"] = leaf.grad.detach().cpu().numpy()
    print("raster visible", int((~culled).sum()), "alpha mean", ra.mean().item())
    np.savez_compressed(os.path.join(HERE, "ref_ut_ftheta_rasterization.npz"), **out)


if __name__ == "__main__":
    record()
