"""FTheta 3DGUT on the GPU: the UT projection and the eval3d compositing (forward and gradients) against the float64
oracle (oracle/ut.py) and the reference's records (ref_ut_ftheta.npz, make_ref_ut_ftheta_golden.py), for
both reference polynomials and both depth orders; a lens beyond 180 degrees; rolling shutter; rasterization() against
the hand chain; batch dims and cameras sharing one parameter set; the drop-in and a short fit."""
import os
import sys
import types

import numpy as np
import pytest
import torch

import gsplat_b200 as gs
from tests import scene
from oracle import ut as U

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_NPZ = os.path.join(ROOT, "tests", "golden", "ref_ut_ftheta.npz")
REF_RASTER_NPZ = os.path.join(ROOT, "tests", "golden", "ref_ut_ftheta_rasterization.npz")
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_ref_ut_ftheta_golden import POLYS, ORDERS, ftheta_K  # noqa: E402
from make_ref_ut_rs_golden import cotangents, end_poses  # noqa: E402

W, H = 96, 64
TW, TH = (W + 15) // 16, (H + 15) // 16
CALS = list(scene.calibrations())


def _t(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)


def _cal(name, ref):
    params, pp, _ = scene.scaled(scene.calibrations()[name], W)
    return dict(params, reference_poly=ref), pp


def _obj(params):
    return gs.FThetaCameraDistortionParameters(**params)


def _small(n=400, C=1):
    sc = scene.make_scene(n_max=n, sh_degree=3, seed=0)
    vm = sc["viewmats"][:C].astype(np.float32)
    return dict(means=sc["means"], quats=sc["quats"], scales=(sc["scales"] * 4.0).astype(np.float32),
                opacities=sc["opacities"], colors=sc["colors"].astype(np.float32), sh=sc["sh"], viewmats=vm,
                viewmats_rs=end_poses(vm))


def _project(p, params, K, gzo=True, shutter=4):
    rs = dict(rolling_shutter=shutter, viewmats_rs=_t(p["viewmats_rs"])) if shutter != 4 else {}
    return gs.fully_fused_projection_with_ut(_t(p["means"]), _t(p["quats"]), _t(p["scales"]), _t(p["opacities"]),
                                             _t(p["viewmats"]), _t(K), W, H, calc_compensations=True,
                                             camera_model="ftheta", ftheta_coeffs=_obj(params), global_z_order=gzo, **rs)


def _lists(r, m2, d, C=1):
    _, ii, fl = gs.isect_tiles(m2, r, d, 16, TW, TH)
    return gs.isect_offset_encode(ii, C, TW, TH).reshape(C, TH, TW), fl


def _check_projection(out, o, ref_rows=None):
    r, m2, d, co, _ = out
    r = r[0].cpu().numpy()
    ro = o["radii"].numpy() if ref_rows is None else ref_rows["radii"]
    frac = o["radii_unrounded"].numpy()
    # a radius at an integer, or a sigma point at the image margin or max_angle, may round either way in float32
    loose = (np.abs(frac - np.round(frac)) < 1e-3).any(-1) | o["rs_edge"].numpy()
    diff = (r != ro).any(-1)
    assert (diff & ~loose).sum() <= max(2, len(r) // 100), (diff & ~loose).sum()
    ok = (r > 0).all(-1) & (ro > 0).all(-1) & ~loose
    assert ok.sum() > 20, ok.sum()
    m2o = o["means2d"].numpy() if ref_rows is None else ref_rows["means2d"]
    do = o["depths"].numpy() if ref_rows is None else ref_rows["depths"]
    err = np.abs(m2[0].cpu().numpy()[ok] - m2o[ok]).max(-1)
    assert (err > 5e-3 + 1e-4 * np.abs(m2o[ok]).max(-1)).sum() <= max(1, ok.sum() // 100)
    # float32 pose interpolation under a rolling shutter moves the depth by a few 1e-6 relative
    np.testing.assert_allclose(d[0].cpu().numpy()[ok], do[ok], rtol=5e-5)
    return ok


# ---- projection against the oracle
@pytest.mark.parametrize("gzo", [True, False])
@pytest.mark.parametrize("ref", [0, 1])
@pytest.mark.parametrize("cname", CALS)
def test_projection_against_oracle(cname, ref, gzo):
    p = _small()
    params, pp = _cal(cname, ref)
    K = ftheta_K(pp)
    out = _project(p, params, K, gzo)
    cam = U.FThetaCamera(params, K[0], W, H)
    o = U.ut_projection(p["means"], p["quats"], p["scales"], p["opacities"], p["viewmats"][0], cam, global_z_order=gzo)
    ok = _check_projection(out, o)
    if not gzo:
        # the depth is the distance from the camera centre
        vm = p["viewmats"][0].astype(np.float64)
        dist = np.linalg.norm(p["means"].astype(np.float64) @ vm[:3, :3].T + vm[:3, 3], axis=-1)
        np.testing.assert_allclose(out[2][0].cpu().numpy()[ok], dist[ok], rtol=1e-5)


# ---- eval3d forward and gradients against the oracle
def _eval_case(p, params, K, offs, fl, bg, shutter=4):
    rs = dict(rolling_shutter=shutter, viewmats_rs=_t(p["viewmats_rs"])) if shutter != 4 else {}
    leaves = [_t(x, True) for x in (p["means"], p["quats"], p["scales"], p["colors"][None], p["opacities"][None], bg)]
    rc, ra = gs.rasterize_to_pixels_eval3d(*leaves[:5], _t(p["viewmats"]), _t(K), W, H, 16, offs, fl,
                                           backgrounds=leaves[5], camera_model="ftheta", ftheta_coeffs=_obj(params), **rs)
    return leaves, rc, ra


def _check_eval(p, params, K, offs, fl, bg, leaves, rc, ra, v_rc, v_ra, ref=None, shutter=4):
    N = len(p["means"])
    cam = U.FThetaCamera(params, K[0], W, H)
    f8 = [torch.from_numpy(np.asarray(x, np.float64)).requires_grad_(True)
          for x in (p["means"], p["quats"], p["scales"], p["colors"], p["opacities"], bg[0])]
    pose = p["viewmats"][0] if shutter == U.GLOBAL else U.ShutterPoses(p["viewmats"][0], p["viewmats_rs"][0], shutter)
    oc, oa, margin = U.eval3d_render(*f8[:5], pose, cam, offs.cpu(), fl.cpu().tolist(), 1, N, 0, background=f8[5])
    ((oc * torch.from_numpy(v_rc[0].astype(np.float64))).sum() + (oa * torch.from_numpy(v_ra[0].astype(np.float64))).sum()).backward()
    # pixels whose Newton step sits near the 1e-6 convergence threshold may converge in one precision only
    step = cam.last_step.reshape(H, W).numpy()
    newton_edge = (step > 1e-7) & (step < 1e-5)
    clear = (margin > 1e-3).numpy() & ~newton_edge
    target_c = oc.detach().numpy() if ref is None else ref["render_colors"][0]
    target_a = oa[..., 0].detach().numpy() if ref is None else ref["render_alphas"][0][..., 0]
    err = np.abs(rc[0].detach().cpu().numpy() - target_c).max(-1)
    aerr = np.abs(ra[0, ..., 0].detach().cpu().numpy() - target_a)
    bad = err > 2e-4
    assert (bad & clear).sum() <= max(1, clear.size // 1000), (bad & clear).sum()
    assert (bad & ~clear).sum() <= max(8, clear.size // 50), ((bad & ~clear).sum(), newton_edge.sum())
    assert ((aerr > 2e-4) & clear).sum() <= max(1, clear.size // 1000)
    for i, name in enumerate(("means", "quats", "scales", "colors", "opacities", "backgrounds")):
        g = leaves[i].grad.detach().cpu().numpy().reshape(-1)
        gr = (f8[i].grad.numpy() if ref is None else ref[f"v_{name}"]).reshape(-1)
        rel = np.linalg.norm(g - gr) / max(np.linalg.norm(gr), 1e-12)
        assert rel < 2e-2, (name, rel)


@pytest.mark.parametrize("gzo", [True, False])
@pytest.mark.parametrize("ref", [0, 1])
@pytest.mark.parametrize("cname", CALS)
def test_eval3d_against_oracle(cname, ref, gzo):
    p = _small()
    params, pp = _cal(cname, ref)
    K = ftheta_K(pp)
    r, m2, d, _, _ = _project(p, params, K, gzo)
    offs, fl = _lists(r, m2, d)
    assert fl.numel() > 20
    rng = np.random.RandomState(1)
    bg = rng.random_sample((1, 3)).astype(np.float32)
    leaves, rc, ra = _eval_case(p, params, K, offs, fl, bg)
    v_rc = rng.standard_normal(rc.shape).astype(np.float32)
    v_ra = rng.standard_normal(ra.shape).astype(np.float32)
    ((rc * _t(v_rc)).sum() + (ra * _t(v_ra)).sum()).backward()
    _check_eval(p, params, K, offs, fl, bg, leaves, rc, ra, v_rc, v_ra)


# ---- rolling shutter through the FTheta lens
@pytest.mark.parametrize("gzo", [True, False])
@pytest.mark.parametrize("cname", ["cross_left_120fov", "synthetic_wide_190"])
def test_rolling_shutter_against_oracle(cname, gzo):
    p = _small()
    params, pp = _cal(cname, 0)
    K = ftheta_K(pp)
    out = _project(p, params, K, gzo, shutter=0)
    cam = U.FThetaCamera(params, K[0], W, H)
    o = U.ut_projection(p["means"], p["quats"], p["scales"], p["opacities"],
                        U.ShutterPoses(p["viewmats"][0], p["viewmats_rs"][0], 0), cam, global_z_order=gzo)
    _check_projection(out, o)
    offs, fl = _lists(*out[:3])
    rng = np.random.RandomState(2)
    bg = rng.random_sample((1, 3)).astype(np.float32)
    leaves, rc, ra = _eval_case(p, params, K, offs, fl, bg, shutter=0)
    v_rc = rng.standard_normal(rc.shape).astype(np.float32)
    v_ra = rng.standard_normal(ra.shape).astype(np.float32)
    ((rc * _t(v_rc)).sum() + (ra * _t(v_ra)).sum()).backward()
    _check_eval(p, params, K, offs, fl, bg, leaves, rc, ra, v_rc, v_ra, shutter=0)


# ---- against the reference's records
def _golden_cases():
    cases = [(c, pn, on, False) for c in CALS for pn in POLYS for on in ORDERS]
    return cases + [(c, "ptoa", "dist", True) for c in CALS]


@pytest.mark.parametrize("cname,pname,oname,rolling", _golden_cases())
def test_kernels_against_reference(cname, pname, oname, rolling):
    z = np.load(REF_NPZ)
    name = f"{cname}/{pname}/{oname}" + ("/rs" if rolling else "")
    p = {k: z[k] for k in ("means", "quats", "scales", "opacities", "colors", "viewmats", "viewmats_rs")}
    params, _ = _cal(cname, POLYS[pname])
    K = z[f"{cname}/Ks"]
    gzo, shutter = ORDERS[oname], (0 if rolling else 4)
    out = _project(p, params, K, gzo, shutter)
    cam = U.FThetaCamera(params, K[0], W, H)
    pose = p["viewmats"][0] if shutter == U.GLOBAL else U.ShutterPoses(p["viewmats"][0], p["viewmats_rs"][0], shutter)
    o = U.ut_projection(p["means"], p["quats"], p["scales"], p["opacities"], pose, cam, global_z_order=gzo)
    rows = {k: z[f"{name}/{k}"][0] for k in ("radii", "means2d", "depths")}
    _check_projection(out, o, rows)
    # the oracle reproduces the reference's rows too
    _check_projection((torch.from_numpy(rows["radii"])[None], torch.from_numpy(rows["means2d"])[None],
                       torch.from_numpy(rows["depths"])[None], None, None), o)
    offs, fl = _t(z[f"{name}/isect_offsets"]), _t(z[f"{name}/flatten_ids"])
    bg, v_rc, v_ra = cotangents(int(z["cotangent_seed"]), 1, 1, 1)
    leaves, rc, ra = _eval_case(p, params, K, offs, fl, bg, shutter)
    ((rc * _t(v_rc)).sum() + (ra * _t(v_ra)).sum()).backward()
    ref = {k: z[f"{name}/{k}"] for k in ("render_colors", "render_alphas", "v_means", "v_quats", "v_scales", "v_colors",
                                          "v_opacities", "v_backgrounds")}
    ref["v_colors"], ref["v_opacities"] = ref["v_colors"][0], ref["v_opacities"][0]
    _check_eval(p, params, K, offs, fl, bg, leaves, rc, ra, v_rc, v_ra, ref=ref, shutter=shutter)


# ---- a lens beyond 180 degrees: Gaussians behind the camera plane inside max_angle
def test_beyond_180_degrees():
    params, pp = _cal("synthetic_wide_190", 0)
    K = ftheta_K(pp)
    rng = np.random.RandomState(4)
    n = 64
    th = rng.uniform(1.62, 1.8, n)  # beyond pi / 2, inside max_angle 1.9
    ph = rng.uniform(-0.4, 0.4, n) + np.where(np.arange(n) % 2 == 0, 0.0, np.pi)  # left and right of the axis
    dist = rng.uniform(2.0, 4.0, n)
    means = np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1) * dist[:, None]
    assert (means[:, 2] < 0).all()
    quats = np.tile(np.float32([1, 0, 0, 0]), (n, 1))
    p = dict(means=means.astype(np.float32), quats=quats, scales=np.full((n, 3), 0.05, np.float32),
             opacities=np.full(n, 0.9, np.float32), viewmats=np.eye(4, dtype=np.float32)[None])
    r_far, _, d_far, _, _ = _project(p, params, K, gzo=False)
    r_z, _, _, _, _ = _project(p, params, K, gzo=True)
    seen = (r_far[0] > 0).all(-1).cpu().numpy()
    assert seen.sum() > n // 2, seen.sum()
    np.testing.assert_allclose(d_far[0].cpu().numpy()[seen], np.linalg.norm(means, axis=-1)[seen], rtol=1e-5)
    assert (r_z[0] == 0).all()  # z < near_plane: culled in the global z order
    cam = U.FThetaCamera(params, K[0], W, H)
    o = U.ut_projection(p["means"], p["quats"], p["scales"], p["opacities"], p["viewmats"][0], cam, global_z_order=False)
    assert ((o["radii"].numpy() > 0).all(-1) == seen).mean() > 0.95


# ---- rasterization() equals the hand chain
def _hand_chain(p, params, K, gzo, bg):
    """UT projection, SH + clamp, isect_tiles + isect_offset_encode, eval3d compositing."""
    C, N = K.shape[0], len(p["means"])
    args = [_t(p[k]) for k in ("means", "quats", "scales", "opacities")]
    vm = _t(p["viewmats"])
    r, m2, d, _, _ = gs.fully_fused_projection_with_ut(*args, vm, _t(K), W, H, camera_model="ftheta",
                                                      ftheta_coeffs=_obj(params), global_z_order=gzo)
    feat = gs.spherical_harmonics(3, args[0], vm, _t(p["sh"]), masks=(r > 0).all(-1))
    feat = torch.clamp_min(feat + 0.5, 0.0)
    offs, fl = _lists(r, m2, d, C)
    opac = torch.broadcast_to(args[3][None], (C, N))
    return gs.rasterize_to_pixels_eval3d(args[0], args[1], args[2], feat, opac, vm, _t(K), W, H, 16, offs, fl,
                                         backgrounds=bg, camera_model="ftheta", ftheta_coeffs=_obj(params))


@pytest.mark.parametrize("gzo", [True, False])
def test_rasterization_equals_hand_chain(gzo):
    p = _small(C=2)
    params, pp = _cal("cross_left_120fov", 0)
    K = ftheta_K(pp, 2, shift=(3.0, -2.0))
    bg = _t(np.float32([[0.1, 0.2, 0.3], [0.3, 0.2, 0.1]]))
    rc, ra, meta = gs.rasterization(_t(p["means"]), _t(p["quats"]), _t(p["scales"]), _t(p["opacities"]), _t(p["sh"]),
                                    _t(p["viewmats"]), _t(K), W, H, sh_degree=3, packed=False, backgrounds=bg,
                                    with_ut=True, with_eval3d=True, camera_model="ftheta",
                                    ftheta_coeffs=_obj(params), global_z_order=gzo)
    hc, ha = _hand_chain(p, params, K, gzo, bg)
    assert torch.equal(ra, ha)
    assert torch.equal(rc, hc)
    assert (ra > 0).float().mean() > 0.05
    # the two cameras share the parameters and differ in their principal points
    assert not torch.equal(rc[0], rc[1])
    if not gzo:
        vm = p["viewmats"].astype(np.float64)
        ok = (meta["radii"] > 0).all(-1).cpu().numpy()
        dist = np.linalg.norm(np.einsum("cij,nj->cni", vm[:, :3, :3], p["means"].astype(np.float64)) + vm[:, None, :3, 3], axis=-1)
        np.testing.assert_allclose(meta["depths"].cpu().numpy()[ok], dist[ok], rtol=1e-5)


def test_rasterization_against_reference():
    z = np.load(REF_RASTER_NPZ)
    params, _ = _cal("cross_left_120fov", 0)
    p = {k: z[k] for k in ("means", "quats", "scales", "opacities", "sh", "viewmats", "Ks")}
    C = p["viewmats"].shape[0]
    bg, v_rc, v_ra = cotangents(int(z["cotangent_seed"]), C, 3, 4)
    leaves = {k: _t(p[k], True) for k in ("means", "quats", "scales", "opacities", "sh")}
    leaves["backgrounds"] = _t(bg, True)
    rc, ra, meta = gs.rasterization(leaves["means"], leaves["quats"], leaves["scales"], leaves["opacities"], leaves["sh"],
                                    _t(p["viewmats"]), _t(p["Ks"]), W, H, sh_degree=3, packed=False,
                                    backgrounds=leaves["backgrounds"], render_mode="RGB+ED", with_ut=True,
                                    with_eval3d=True, camera_model="ftheta", ftheta_coeffs=_obj(params),
                                    global_z_order=False)
    ((rc * _t(v_rc)).sum() + (ra * _t(v_ra)).sum()).backward()
    r, rr = meta["radii"].cpu().numpy(), z["radii"]
    assert ((r != rr).any(-1)).mean() < 0.02
    ok = (r > 0).all(-1) & (rr > 0).all(-1)
    np.testing.assert_allclose(meta["depths"].cpu().numpy()[ok], z["depths"][ok], rtol=1e-5)
    err = np.abs(rc[..., :3].detach().cpu().numpy() - z["render_colors"][..., :3]).max(-1)
    assert (err > 1e-3).mean() < 0.01, (err > 1e-3).mean()
    aerr = np.abs(ra.detach().cpu().numpy() - z["render_alphas"])
    assert (aerr > 1e-3).mean() < 0.01
    for k, leaf in leaves.items():
        g, gr = leaf.grad.cpu().numpy().reshape(-1), z[f"v_{k}"].reshape(-1)
        assert np.linalg.norm(g - gr) / max(np.linalg.norm(gr), 1e-12) < 5e-2, k


# ---- batch dims and cameras sharing one parameter set
def test_batch_dims_match_single_calls():
    p = _small(C=2)
    params, pp = _cal("front_tele_30fov", 1)
    K = ftheta_K(pp, 2, shift=(-4.0, 3.0))
    B = 2
    ex = lambda a: np.stack([a] * B)  # noqa: E731
    args = [_t(ex(p[k])) for k in ("means", "quats", "scales", "opacities")]
    r, m2, d, cn, _ = gs.fully_fused_projection_with_ut(*args, _t(ex(p["viewmats"])), _t(ex(K)), W, H,
                                                       camera_model="ftheta", ftheta_coeffs=_obj(params),
                                                       global_z_order=False)
    assert r.shape == (B, 2, len(p["means"]), 2)
    for c in range(2):
        r1, m1, d1, _, _ = gs.fully_fused_projection_with_ut(*[a[0] for a in args], _t(p["viewmats"][c:c + 1]),
                                                           _t(K[c:c + 1]), W, H, camera_model="ftheta",
                                                           ftheta_coeffs=_obj(params), global_z_order=False)
        for b in range(B):
            assert torch.equal(r[b, c], r1[0]) and torch.equal(m2[b, c], m1[0]) and torch.equal(d[b, c], d1[0])
    assert not torch.equal(m2[0, 0], m2[0, 1])
    offs, fl = gs.isect_tiles(m2, r, d, 16, TW, TH)[1:]
    offs = gs.isect_offset_encode(offs, B * 2, TW, TH).reshape(B, 2, TH, TW)
    col = _t(np.stack([np.stack([p["colors"]] * 2)] * B))
    rc, ra = gs.rasterize_to_pixels_eval3d(args[0], args[1], args[2], col, args[3][:, None].expand(B, 2, -1).contiguous(),
                                           _t(ex(p["viewmats"])), _t(ex(K)), W, H, 16, offs, fl, camera_model="ftheta",
                                           ftheta_coeffs=_obj(params))
    assert torch.equal(rc[0], rc[1]) and (ra > 0).any()


# ---- the drop-in serves a call that carries coefficients
def test_dropin_serves_ftheta(monkeypatch):
    from gsplat_b200 import dropin

    calls = []

    def stock(*a, **k):
        calls.append(k.get("camera_model"))
        return "stock"

    g = types.ModuleType("gsplat")
    g.__path__ = []
    g.__file__ = "gsplat/__init__.py"
    wrapper = types.ModuleType("gsplat.cuda._wrapper")
    for name in dropin._OPS + ("adam",):
        setattr(wrapper, name, stock)
    rendering = types.ModuleType("gsplat.rendering")
    rendering.rasterization = stock
    mods = {"gsplat": g, "gsplat.cuda": types.ModuleType("gsplat.cuda"), "gsplat.cuda._wrapper": wrapper,
            "gsplat.rendering": rendering, "gsplat.relocation": types.ModuleType("gsplat.relocation"),
            "gsplat.strategy": types.ModuleType("gsplat.strategy"), "gsplat.strategy.ops": types.ModuleType("gsplat.strategy.ops"),
            "gsplat.optimizers": types.ModuleType("gsplat.optimizers")}
    mods["gsplat.relocation"].compute_relocation = stock
    mods["gsplat.strategy.ops"].compute_relocation = stock
    mods["gsplat.optimizers"].SelectiveAdam = object
    g.rasterization = stock
    for k, v in mods.items():
        monkeypatch.setitem(sys.modules, k, v)
    dropin.apply(losses=False)
    try:
        st = dropin.stats["rasterization"]
        b0, s0 = st["b200"], st["stock"]
        p = _small()
        params, pp = _cal("cross_left_120fov", 0)
        args = [_t(p[k]) for k in ("means", "quats", "scales", "opacities", "sh", "viewmats")] + [_t(ftheta_K(pp)), W, H]
        rc, ra, _ = g.rasterization(*args, sh_degree=3, packed=False, with_ut=True, with_eval3d=True,
                                    camera_model="ftheta", ftheta_coeffs=_obj(params), global_z_order=False)
        assert rc.shape == (1, H, W, 3) and (ra > 0).any()
        assert st["b200"] == b0 + 1 and st["stock"] == s0 and calls == []
    finally:
        dropin.undo()


# ---- a short fit through an FTheta camera
def test_short_fit_reduces_loss():
    p = _small(n=300)
    params, pp = _cal("cross_left_120fov", 0)
    K = _t(ftheta_K(pp))
    vm = _t(p["viewmats"])
    with torch.no_grad():
        target, _, _ = gs.rasterization(_t(p["means"]), _t(p["quats"]), _t(p["scales"]), _t(p["opacities"]), _t(p["sh"]),
                                        vm, K, W, H, sh_degree=3, packed=False, with_ut=True, with_eval3d=True,
                                        camera_model="ftheta", ftheta_coeffs=_obj(params), global_z_order=False)
    rng = np.random.RandomState(9)
    leaves = {"means": _t(p["means"] + rng.normal(0, 0.02, p["means"].shape).astype(np.float32), True),
              "sh": _t(p["sh"] * 0.5, True), "opacities": _t(p["opacities"] * 0.8, True)}
    opt = torch.optim.Adam(leaves.values(), lr=5e-3)
    losses = []
    for _ in range(60):
        rc, _, _ = gs.rasterization(leaves["means"], _t(p["quats"]), _t(p["scales"]), leaves["opacities"].clamp(0, 1),
                                    leaves["sh"], vm, K, W, H, sh_degree=3, packed=False, with_ut=True, with_eval3d=True,
                                    camera_model="ftheta", ftheta_coeffs=_obj(params), global_z_order=False)
        loss = (rc - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert np.isfinite(losses).all() and losses[-1] < 0.6 * losses[0], (losses[0], losses[-1])
