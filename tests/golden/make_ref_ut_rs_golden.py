#!/usr/bin/env python
"""Records the reference's rolling-shutter 3DGUT for the tests.

    python tests/golden/make_ref_ut_rs_golden.py     (GPU; needs oracle/_ref from python oracle/build_ref.py --full)

Writes tests/golden/ref_ut_rs.npz and tests/golden/ref_ut_rs_rasterization.npz, on the seeded 96x64 garden crop of
make_ref_ut_golden.py.  The end pose is the start pose moved by a seeded rotation of about 2 degrees and a small
translation (the script prints the largest image displacement of a visible mean between the two poses, which should be
several pixels).

ref_ut_rs.npz: for every camera of RS_CAMERAS and every rolling shutter type, the reference build's
torch.ops.gsplat.projection_ut_3dgs_fused and rasterize_to_pixels_from_world_3dgs (MixedBatch), both given viewmats1:
the projection outputs, the tile lists built from them (gsplat_b200.isect_tiles / isect_offset_encode), the eval3d
colour (one channel: the shutter is what these records are about, and one channel keeps the file small) and alphas,
and the gradients of a seeded cotangent with respect to means, quats, scales, colors, opacities and backgrounds.

ref_ut_rs_rasterization.npz: one rasterization_3dgs record with SH degree 3, RGB+ED, two cameras and a background with
a top-to-bottom shutter through the distorted pinhole, with gradients for viewmats and viewmats_rs as well.

The backgrounds and cotangents are not stored: cotangents(seed, ...) redraws them from the recorded seed.
"""
import os
import sys

import numpy as np

from make_ref_ut_golden import CAMERA_IDS, HERE, N_GAUSS, ROOT, SCALE, H, W, small_scene

RS_CAMERAS = {
    "pinhole": ("pinhole", {}),
    "pinhole_distorted": ("pinhole", {"radial": [0.08, -0.03, 0.005, 0.01, 0.0, 0.0], "tangential": [0.004, -0.003]}),
    "fisheye_radial": ("fisheye", {"radial": [0.04, -0.01, 0.002, -0.0003]}),
}
SHUTTERS = {"top_to_bottom": 0, "left_to_right": 1, "bottom_to_top": 2, "right_to_left": 3}
RASTER_CAMERA, RASTER_SHUTTER, RASTER_C, RASTER_SH_DEGREE = "pinhole_distorted", 0, 2, 3
KEYS = {"radial": "radial_coeffs", "tangential": "tangential_coeffs", "thin": "thin_prism_coeffs"}
COTANGENT_SEED, RASTER_COTANGENT_SEED = 7, 11


def end_poses(viewmats, seed=3, degrees=2.0, shift=0.03):
    """viewmats [C, 4, 4] moved in the camera frame by a seeded rotation of `degrees` about a random axis and a
    translation of length `shift`."""
    rng = np.random.RandomState(seed)
    out = []
    for vm in viewmats:
        axis = rng.standard_normal(3)
        axis /= np.linalg.norm(axis)
        th = np.deg2rad(degrees)
        k = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
        delta = np.eye(4)
        delta[:3, :3] = np.eye(3) + np.sin(th) * k + (1 - np.cos(th)) * (k @ k)
        d = rng.standard_normal(3)
        delta[:3, 3] = shift * d / np.linalg.norm(d)
        out.append(delta @ vm.astype(np.float64))
    return np.stack(out).astype(np.float32)


def cotangents(seed, images, bg_channels, channels):
    """The seeded background [images, bg_channels] and cotangents of the colours [images, H, W, channels] and of the
    alphas [images, H, W, 1], drawn in that order."""
    rng = np.random.RandomState(seed)
    bg = rng.random_sample((images, bg_channels)).astype(np.float32)
    v_rc = rng.standard_normal((images, H, W, channels)).astype(np.float32)
    v_ra = rng.standard_normal((images, H, W, 1)).astype(np.float32)
    return bg, v_rc, v_ra


def displacement(means, vm0, vm1, K):
    """Largest pinhole image displacement of a mean in front of both poses and inside the image."""
    def proj(vm):
        pc = means @ vm[:3, :3].T + vm[:3, 3]
        uv = pc[:, :2] / pc[:, 2:] * np.diag(K)[:2] + K[:2, 2]
        return uv, pc[:, 2] > 0.1

    a, oka = proj(vm0.astype(np.float64))
    b, okb = proj(vm1.astype(np.float64))
    inside = oka & okb & (a[:, 0] >= 0) & (a[:, 0] < W) & (a[:, 1] >= 0) & (a[:, 1] < H)
    return float(np.linalg.norm(a - b, axis=1)[inside].max())


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
    vm_rs = end_poses(sc["viewmats"])
    print("largest image displacement between the start and end poses: "
          f"{displacement(sc['means'].astype(np.float64), sc['viewmats'][0], vm_rs[0], sc['Ks'][0].astype(np.float64)):.2f} px")
    sc["colors"] = np.ascontiguousarray(sc["colors"][:, :1])
    bg, v_rc, v_ra = cotangents(COTANGENT_SEED, 1, 1, 1)
    out = dict(sc, viewmats_rs=vm_rs, cotangent_seed=COTANGENT_SEED, width=W, height=H)
    utp = torch.classes.gsplat.UnscentedTransformParameters()
    ftheta = torch.classes.gsplat.FThetaCameraDistortionParameters()
    tw, th = (W + 15) // 16, (H + 15) // 16
    for cname, (model, coeffs) in RS_CAMERAS.items():
        co = {KEYS[k]: np.float32([v]) for k, v in coeffs.items()}
        for k, v in co.items():
            out[f"{cname}/{k}"] = v
        ct = {k: t(v) for k, v in co.items()}
        cam = CAMERA_IDS[model]
        for sname, rs in SHUTTERS.items():
            name = f"{cname}/{sname}"
            radii, m2, d, conics, comps = ops.projection_ut_3dgs_fused(
                t(sc["means"]), t(sc["quats"]), t(sc["scales"]), t(sc["opacities"]), t(sc["viewmats"]), t(vm_rs), t(sc["Ks"]),
                W, H, 0.3, 0.01, 1e10, 0.0, True, cam, True, utp, rs, ct.get("radial_coeffs"), ct.get("tangential_coeffs"),
                ct.get("thin_prism_coeffs"), None, None, None,
            )
            culled = (radii == 0).all(-1)
            # the reference leaves the float outputs of a culled row unwritten; this library zeroes them
            m2, d, conics, comps = (x.masked_fill(culled[..., None] if x.dim() == 3 else culled, 0) for x in (m2, d, conics, comps))
            _, isect_ids, flatten_ids = gs.isect_tiles(m2, radii, d, 16, tw, th)
            offsets = gs.isect_offset_encode(isect_ids, 1, tw, th)
            leaves = [t(x).requires_grad_(True) for x in (sc["means"], sc["quats"], sc["scales"], sc["colors"][None], sc["opacities"][None], bg)]
            rc, ra, *_ = ops.rasterize_to_pixels_from_world_3dgs(
                leaves[0], leaves[1], leaves[2], leaves[3], leaves[4], leaves[5], None, W, H, 16, t(sc["viewmats"]), t(vm_rs),
                t(sc["Ks"]), cam, utp, rs, None, ct.get("radial_coeffs"), ct.get("tangential_coeffs"),
                ct.get("thin_prism_coeffs"), ftheta, None, None, offsets, flatten_ids, False, False, False, 0, True, False,
            )
            ((rc * t(v_rc)).sum() + (ra * t(v_ra)).sum()).backward()
            rec = dict(radii=radii, means2d=m2, depths=d, conics=conics, compensations=comps, isect_offsets=offsets,
                       flatten_ids=flatten_ids, render_colors=rc, render_alphas=ra)
            for k, v in rec.items():
                out[f"{name}/{k}"] = v.detach().cpu().numpy()
            for k, leaf in zip(("means", "quats", "scales", "colors", "opacities", "backgrounds"), leaves):
                out[f"{name}/v_{k}"] = leaf.grad.detach().cpu().numpy()
            print(name, "visible", int((~culled).sum()), "pairs", flatten_ids.numel(), "alpha mean", float(ra.detach().mean()))

    np.savez_compressed(os.path.join(HERE, "ref_ut_rs.npz"), **out)

    # ---- rasterization_3dgs: SH degree 3, RGB+ED, two cameras, a background, gradients for both poses
    full = scene.make_scene(n_max=N_GAUSS, sh_degree=RASTER_SH_DEGREE, seed=0)
    C = RASTER_C
    vm0 = full["viewmats"][:C].astype(np.float32)
    vm1 = end_poses(vm0, seed=5)
    inputs = dict(means=full["means"], quats=full["quats"], scales=(full["scales"] * SCALE).astype(np.float32),
                  opacities=full["opacities"], sh=full["sh"], viewmats=vm0, viewmats_rs=vm1,
                  Ks=scene.rescale_K(full["Ks"], full["width"], full["height"], W, H)[:C].astype(np.float32))
    bg2, v_rc2, v_ra2 = cotangents(RASTER_COTANGENT_SEED, C, 3, 4)  # RGB+ED: four channels
    model, coeffs = RS_CAMERAS[RASTER_CAMERA]
    co = {KEYS[k]: np.tile(np.float32(v), (C, 1)) for k, v in coeffs.items()}
    out = dict(inputs, **co, width=W, height=H, sh_degree=RASTER_SH_DEGREE, rolling_shutter=RASTER_SHUTTER,
               cotangent_seed=RASTER_COTANGENT_SEED)
    ct = {k: t(v) for k, v in co.items()}
    leaves = {k: t(inputs[k]).requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "sh", "viewmats", "viewmats_rs")}
    leaves["backgrounds"] = t(bg2).requires_grad_(True)
    res = ops.rasterization_3dgs(
        leaves["means"], None, leaves["quats"], leaves["scales"], leaves["opacities"], leaves["sh"], leaves["viewmats"],
        t(inputs["Ks"]), W, H, 16, 0.3, 0.01, 1e10, 0.0, leaves["backgrounds"], False, False, False, False, True,
        CAMERA_IDS[model], False, 32, True, RASTER_SH_DEGREE, None, -1, True, True, True, True, None, leaves["viewmats_rs"],
        utp, RASTER_SHUTTER, ct.get("radial_coeffs"), ct.get("tangential_coeffs"), ct.get("thin_prism_coeffs"), ftheta, None,
        None, True, False, False, 0, None, 1,
    )
    rc, ra = res[0], res[1]
    radii, m2, d = res[8], res[9], res[10]
    flatten_ids, isect_offsets = res[15], res[16]
    ((rc * t(v_rc2)).sum() + (ra * t(v_ra2)).sum()).backward()
    culled = (radii == 0).all(-1)
    m2, d = m2.masked_fill(culled[..., None], 0), d.masked_fill(culled, 0)
    rec = dict(render_colors=rc, render_alphas=ra, radii=radii, means2d=m2, depths=d, isect_offsets=isect_offsets,
               flatten_ids=flatten_ids)
    for k, v in rec.items():
        out[k] = v.detach().cpu().numpy()
    for k, leaf in leaves.items():
        out[f"v_{k}"] = (leaf.grad if leaf.grad is not None else torch.zeros_like(leaf)).detach().cpu().numpy()
    print("raster visible", int((~culled).sum()), "pairs", flatten_ids.numel(), "alpha mean", ra.mean().item(),
          "|v_viewmats|", float(np.abs(out["v_viewmats"]).sum()), "|v_viewmats_rs|", float(np.abs(out["v_viewmats_rs"]).sum()))
    np.savez_compressed(os.path.join(HERE, "ref_ut_rs_rasterization.npz"), **out)


if __name__ == "__main__":
    record()
