"""Self-check of the float64 oracle chain ``gso.rasterization_fwd_bwd`` (CPU only, runs without a GPU).

The GPU tests of rasterization() compare every gradient against this chain, so the chain itself has to be right:
here each of its gradients is checked against a float64 central difference of its own forward, one random
direction per parameter tensor, on a tiny scene (a few hundred garden Gaussians seen through a 48 x 32 crop).

The central difference is only meaningful while no discrete decision flips inside the step (alpha >= 1/255, the
T <= 1e-4 stop, tile and cull cuts): the flatten lists and radii must be identical at +h and -h, and pixels
with a decision within 1e-3 of its threshold get no cotangent (their last_ids must not change either).

Two differences are expected and bounded explicitly:
  * the compensation backward divides by (comp + 1e-6) -- the reference's rule, not the exact derivative -- so
    the part of the gradient that flows through the compensation may be off by a factor 1e-6 / min(comp);
  * in the ED modes, acc / max(alpha, 1e-10) is arbitrarily steep as alpha -> 0: the depth cotangent is only put
    on pixels whose alpha is above 1e-2.
"""

import numpy as np
import pytest

from oracle import gso
from tests import scene

W, H = 48, 32
STEP = 1e-6


def _tiny_scene(camera_model="pinhole", n_cams=1, per_cam=160, batch=0, seed=0):
    """Gaussians of the garden scene that are visible in a 48 x 32 crop of the first ``n_cams`` cameras."""
    sc = scene.make_scene(sh_degree=3)
    Ks = sc["Ks"][:n_cams].astype(np.float64).copy()
    Ks[:, 0, 2], Ks[:, 1, 2] = W / 2, H / 2
    if camera_model == "ortho":
        Ks[:, 0, 0], Ks[:, 1, 1] = 60.0, 60.0
    vm = sc["viewmats"][:n_cams].astype(np.float64)
    f8 = lambda k: sc[k].astype(np.float64)  # noqa: E731
    radii = gso.fully_fused_projection(
        f8("means"), None, f8("quats"), f8("scales"), vm, Ks, W, H, 0.3, 0.01, 1e10, 0.0, False, camera_model,
        f8("opacities"),
    )[0]
    rng = np.random.RandomState(seed)
    sel = set()
    for c in range(n_cams):
        vis = np.nonzero((radii[c] > 0).all(-1))[0]
        assert len(vis) >= per_cam
        sel.update(rng.choice(vis, per_cam, replace=False).tolist())
    sel = np.array(sorted(sel))
    P = {k: np.ascontiguousarray(f8(k)[sel]) for k in ("means", "quats", "scales", "opacities", "sh", "colors")}
    P["viewmats"], P["Ks"] = vm, Ks
    if batch:
        # batch element b sees the scene shifted by 0.01 b along x
        shift = np.array([0.01, 0.0, 0.0])
        for k in ("means", "quats", "scales", "opacities"):
            P[k] = np.stack([P[k] + (shift * b if k == "means" else 0.0) for b in range(batch)])
        P["viewmats"], P["Ks"] = np.stack([vm] * batch), np.stack([Ks] * batch)
    return P


def _run(P, cfg, v_rc=None, v_ra=None):
    colors = P.get("sh") if cfg.get("sh_degree") is not None else P.get("colors")
    return gso.rasterization_fwd_bwd(
        P["means"], P.get("quats"), P.get("scales"), P["opacities"], colors, P["viewmats"], P["Ks"], W, H,
        cfg.get("sh_degree"), v_rc, v_ra, backgrounds=P.get("backgrounds"), covars=P.get("covars"),
        **{k: v for k, v in cfg.items() if k not in ("sh_degree",)},
    )


def _check(P, cfg, params, seed=0):
    fwd, _ = _run(P, cfg)
    rng = np.random.RandomState(seed)
    v_rc = rng.standard_normal(fwd["render_colors"].shape)
    v_ra = rng.standard_normal(fwd["render_alphas"].shape)
    if cfg.get("render_mode") in ("ED", "RGB+ED"):
        v_rc[..., -1:] *= fwd["render_alphas"] > 1e-2
    # a decision that flips in the middle of a pixel's list leaves last_ids alone: pixels with any decision within
    # 1e-3 (relative) of its threshold get no cotangent.  The steps below move alpha by well under 1e-4 relative.
    keep = fwd["margins"] > 1e-3
    assert keep.mean() > 0.8
    v_rc, v_ra = v_rc * keep[..., None], v_ra * keep[..., None]
    _, g = _run(P, cfg, v_rc, v_ra)
    assert fwd["flatten_ids"].shape[0] >= 300, f"only {fwd['flatten_ids'].shape[0]} intersections"

    def loss(f):
        return (f["render_colors"] * v_rc).sum() + (f["render_alphas"] * v_ra).sum()

    # the part of each gradient that flows through the compensation: the same backward with only v_compensations
    g_comp = None
    if cfg.get("rasterize_mode") == "antialiased":
        z = np.zeros_like
        vc = gso.fully_fused_projection_bwd(
            P["means"], P.get("covars"), P.get("quats"), P.get("scales"), P["viewmats"], P["Ks"], W, H,
            cfg.get("eps2d", 0.3), fwd["radii"], fwd["conics"], fwd["compensations"], z(fwd["means2d"]),
            z(fwd["depths"]), z(fwd["conics"]), g["v_compensations"], cfg.get("viewmats_requires_grad", False),
            cfg.get("camera_model", "pinhole"),
        )
        g_comp = dict(v_means=vc[0], v_covars=vc[1], v_quats=vc[2], v_scales=vc[3], v_viewmats=vc[4])
        comp_rel = 1e-6 / fwd["compensations"][(fwd["radii"] > 0).all(-1)].min()
    for name, key in params:
        p = P[name]
        d = rng.standard_normal(p.shape)
        if name in ("scales", "covars", "opacities"):
            # relative steps keep tiny scales positive, covariances positive definite and faint alphas off 1/255
            d *= np.abs(p)
        if name in ("means", "viewmats"):
            # one world unit is ~400 pixels here: a 1e-6 shift would move alpha by ~1e-3 relative and flip decisions
            d *= 1e-2
        if name == "viewmats":
            d[..., 3, :] = 0.0
        outs = []
        for s in (1.0, -1.0):
            Q = dict(P)
            Q[name] = p + s * STEP * d
            outs.append(_run(Q, cfg)[0])
        for k in ("flatten_ids", "radii", "last_ids"):
            a, b, c = outs[0][k], outs[1][k], fwd[k]
            if k == "last_ids":
                a, b, c = a[keep], b[keep], c[keep]
            assert np.array_equal(a, b) and np.array_equal(a, c), f"{name}: {k} changed within the step; pick another scene"
        fd = (loss(outs[0]) - loss(outs[1])) / (2 * STEP)
        an = float((g[key] * d).sum())
        mag = float(np.abs(g[key] * d).sum())
        bound = 1e-6 * abs(an) + 1e-9 * mag
        if g_comp is not None and g_comp.get(key) is not None:
            bound += comp_rel * float(np.abs(g_comp[key] * d).sum())
        assert abs(fd - an) <= bound, f"{name}: finite difference {fd:.10e} vs oracle {an:.10e} (bound {bound:.2e})"


GEOM = [("means", "v_means"), ("quats", "v_quats"), ("scales", "v_scales"), ("opacities", "v_opacities")]


def test_fd_classic_rgb_sh():
    P = _tiny_scene()
    _check(P, dict(sh_degree=3), GEOM + [("sh", "v_sh")])


def test_fd_antialiased_sh_backgrounds_pose():
    P = _tiny_scene(n_cams=2)
    P["backgrounds"] = np.random.RandomState(1).random_sample((2, 3))
    cfg = dict(sh_degree=3, rasterize_mode="antialiased", viewmats_requires_grad=True)
    _check(P, cfg, GEOM + [("sh", "v_sh"), ("viewmats", "v_viewmats"), ("backgrounds", "v_backgrounds")])


@pytest.mark.parametrize("render_mode", ["D", "RGB+D"])
def test_fd_depth_modes(render_mode):
    P = _tiny_scene(n_cams=2)
    P["backgrounds"] = np.random.RandomState(2).random_sample((2, 3))
    params = GEOM + ([("colors", "v_colors"), ("backgrounds", "v_backgrounds")] if render_mode == "RGB+D" else [])
    _check(P, dict(render_mode=render_mode, viewmats_requires_grad=True), params + [("viewmats", "v_viewmats")])


@pytest.mark.parametrize("render_mode", ["ED", "RGB+ED"])
def test_fd_expected_depth_antialiased(render_mode):
    P = _tiny_scene(n_cams=2)
    P["colors"] = np.random.RandomState(3).random_sample((2,) + P["colors"].shape)  # [C, N, D]
    params = GEOM + ([("colors", "v_colors")] if render_mode == "RGB+ED" else [])
    _check(P, dict(render_mode=render_mode, rasterize_mode="antialiased"), params)


def test_fd_covars():
    P = _tiny_scene(n_cams=2)
    P["covars"] = gso.quat_scale_to_covar_preci(P.pop("quats"), P.pop("scales"), True, False, True)[0]
    _check(P, dict(sh_degree=2, rasterize_mode="antialiased"), [("means", "v_means"), ("covars", "v_covars")])


def test_fd_batch_and_clipping():
    P = _tiny_scene(n_cams=2, batch=2)
    cfg = dict(sh_degree=1, viewmats_requires_grad=True, near_plane=0.5, far_plane=50.0, radius_clip=0.5, eps2d=0.1)
    _check(P, cfg, GEOM + [("sh", "v_sh"), ("viewmats", "v_viewmats")])


@pytest.mark.parametrize("camera_model", ["ortho", "fisheye"])
def test_fd_camera_models(camera_model):
    P = _tiny_scene(camera_model=camera_model, per_cam=320)
    cfg = dict(sh_degree=1, camera_model=camera_model, rasterize_mode="antialiased", viewmats_requires_grad=True)
    _check(P, cfg, GEOM + [("sh", "v_sh"), ("viewmats", "v_viewmats")])
