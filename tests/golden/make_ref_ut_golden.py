#!/usr/bin/env python
"""Records the reference's 3DGUT behaviour for the tests.

    python tests/golden/make_ref_ut_golden.py --signatures REFERENCE_ROOT     (no GPU; reads the reference's source)
    python tests/golden/make_ref_ut_golden.py                                  (GPU; needs oracle/_ref from
                                                                                python oracle/build_ref.py --full)

--signatures writes tests/golden/ref_signatures_ut.json: the parameter names and default values (as source text) of
fully_fused_projection_with_ut and rasterize_to_pixels_eval3d, read with ast from the reference's _wrapper.py.

Without it, the reference build's torch.ops.gsplat.projection_ut_3dgs_fused and rasterize_to_pixels_from_world_3dgs
(MixedBatch) run on a small seeded garden crop at 96x64 for every camera of CAMERAS, and tests/golden/ref_ut.npz gets,
per camera: the projection outputs, the tile lists built from them (gsplat_b200.isect_tiles / isect_offset_encode,
whose lists equal the reference's), the eval3d colours and alphas, and the gradients of a seeded cotangent with
respect to means, quats, scales, colors, opacities and backgrounds.
"""
import ast
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
NAMES = ("fully_fused_projection_with_ut", "rasterize_to_pixels_eval3d")
W, H, N_GAUSS, SCALE = 96, 64, 400, 4.0
# name -> (camera model, coefficients)
CAMERAS = {
    "pinhole": ("pinhole", {}),
    "pinhole_radial": ("pinhole", {"radial": [0.08, -0.03, 0.005, 0.01, 0.0, 0.0]}),
    "pinhole_tangential": ("pinhole", {"tangential": [0.004, -0.003]}),
    "pinhole_thin_prism": ("pinhole", {"thin": [0.002, -0.001, 0.001, 0.0005]}),
    "fisheye": ("fisheye", {}),
    "fisheye_radial": ("fisheye", {"radial": [0.04, -0.01, 0.002, -0.0003]}),
}
CAMERA_IDS = {"pinhole": 0, "fisheye": 2}  # reference CameraModelType


def signatures(root):
    tree = ast.parse(open(os.path.join(root, "gsplat", "cuda", "_wrapper.py")).read())
    out = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name in NAMES:
            names = [x.arg for x in node.args.args]
            defaults = [ast.unparse(d) for d in node.args.defaults]
            out[node.name] = {"params": names, "defaults": dict(zip(names[len(names) - len(defaults):], defaults))}
    with open(os.path.join(HERE, "ref_signatures_ut.json"), "w") as f:
        json.dump({"params": out}, f, indent=1)
        f.write("\n")


def small_scene():
    sys.path.insert(0, ROOT)
    from tests import scene

    sc = scene.make_scene(n_max=N_GAUSS, sh_degree=0, seed=0)
    K = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:1].astype(np.float32)
    return dict(means=sc["means"], quats=sc["quats"], scales=(sc["scales"] * SCALE).astype(np.float32),
                opacities=sc["opacities"], colors=sc["colors"].astype(np.float32), viewmats=sc["viewmats"][:1], Ks=K)


def record():
    sys.path.insert(0, ROOT)
    import torch

    import gsplat_b200 as gs
    from oracle import refcuda

    ops = refcuda.load_ops()
    dev = "cuda"
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    sc = small_scene()
    rng = np.random.RandomState(7)
    bg = rng.random_sample((1, 3)).astype(np.float32)
    v_rc = rng.standard_normal((1, H, W, 3)).astype(np.float32)
    v_ra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    out = {k: v for k, v in sc.items()}
    out.update(backgrounds=bg, v_render_colors=v_rc, v_render_alphas=v_ra, width=W, height=H)
    utp = torch.classes.gsplat.UnscentedTransformParameters()
    ftheta = torch.classes.gsplat.FThetaCameraDistortionParameters()
    keys = {"radial": "radial_coeffs", "tangential": "tangential_coeffs", "thin": "thin_prism_coeffs"}
    tw, th = (W + 15) // 16, (H + 15) // 16
    for name, (model, coeffs) in CAMERAS.items():
        co = {keys[k]: np.float32([v]) for k, v in coeffs.items()}
        for k, v in co.items():
            out[f"{name}/{k}"] = v
        ct = {k: t(v) for k, v in co.items()}
        cam = CAMERA_IDS[model]
        radii, m2, d, conics, comps = ops.projection_ut_3dgs_fused(
            t(sc["means"]), t(sc["quats"]), t(sc["scales"]), t(sc["opacities"]), t(sc["viewmats"]), None, t(sc["Ks"]), W, H,
            0.3, 0.01, 1e10, 0.0, True, cam, True, utp, 4, ct.get("radial_coeffs"), ct.get("tangential_coeffs"),
            ct.get("thin_prism_coeffs"), None, None, None,
        )
        culled = (radii == 0).all(-1)
        # the reference leaves the float outputs of a culled row unwritten; this library zeroes them
        m2, d, conics, comps = (x.masked_fill(culled[..., None] if x.dim() == 3 else culled, 0) for x in (m2, d, conics, comps))
        _, isect_ids, flatten_ids = gs.isect_tiles(m2, radii, d, 16, tw, th)
        offsets = gs.isect_offset_encode(isect_ids, 1, tw, th)
        leaves = [t(x).requires_grad_(True) for x in (sc["means"], sc["quats"], sc["scales"], sc["colors"][None], sc["opacities"][None], bg)]
        rc, ra, *_ = ops.rasterize_to_pixels_from_world_3dgs(
            leaves[0], leaves[1], leaves[2], leaves[3], leaves[4], leaves[5], None, W, H, 16, t(sc["viewmats"]), None,
            t(sc["Ks"]), cam, utp, 4, None, ct.get("radial_coeffs"), ct.get("tangential_coeffs"),
            ct.get("thin_prism_coeffs"), ftheta, None, None, offsets, flatten_ids, False, False, False, 0, True, False,
        )
        ((rc * t(v_rc)).sum() + (ra * t(v_ra)).sum()).backward()
        rec = dict(radii=radii, means2d=m2, depths=d, conics=conics, compensations=comps, isect_offsets=offsets,
                   flatten_ids=flatten_ids, render_colors=rc, render_alphas=ra)
        for k, v in rec.items():
            out[f"{name}/{k}"] = v.detach().cpu().numpy()
        for k, leaf in zip(("means", "quats", "scales", "colors", "opacities", "backgrounds"), leaves):
            out[f"{name}/v_{k}"] = leaf.grad.detach().cpu().numpy()
        print(name, "visible", int((~culled).sum()), "pairs", flatten_ids.numel(), "alpha mean", float(ra.mean()))
    np.savez_compressed(os.path.join(HERE, "ref_ut.npz"), **out)


if __name__ == "__main__":
    if "--signatures" in sys.argv:
        rest = [a for a in sys.argv[1:] if a != "--signatures"]
        if not rest:
            sys.exit("--signatures needs the reference checkout's root directory")
        signatures(rest[0])
    else:
        record()
