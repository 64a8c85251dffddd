"""Rolling-shutter 3DGUT on the GPU: the UT projection and the eval3d compositing (forward and gradients) against the
float64 oracle and against the reference's records (ref_ut_rs.npz, make_ref_ut_rs_golden.py), the row and column
identity with global-shutter renders at interpolated poses, no motion equal to the global shutter, and
rasterization(): the hand chain, the reference's orchestrator with both pose gradients, batch dims, the drop-in and a
short fit."""
import os
import sys
import types

import numpy as np
import pytest
import torch

import gsplat_b200 as gs
from oracle import gso
from oracle import ut as U
from tests import scene
from tests.test_ut_gpu import CAMS, KEYS, H, W

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_NPZ = os.path.join(ROOT, "tests", "golden", "ref_ut_rs.npz")
REF_RASTER_NPZ = os.path.join(ROOT, "tests", "golden", "ref_ut_rs_rasterization.npz")
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_ref_ut_rs_golden import cotangents, end_poses  # noqa: E402
TW, TH = (W + 15) // 16, (H + 15) // 16
SHUTTERS = [0, 1, 2, 3]
# a pinhole, a distorted pinhole and a distorted fisheye for the slower oracle compositing
CAMS3 = [CAMS[0], CAMS[1], CAMS[5]]
SNAMES = {"top_to_bottom": 0, "left_to_right": 1, "bottom_to_top": 2, "right_to_left": 3}


def _t(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)


def _end_pose(vm, seed=3, degrees=2.0, shift=0.03):
    """[C, 4, 4] view matrices moved in the camera frame by a seeded rotation and translation (as the golden script)."""
    return end_poses(vm, seed=seed, degrees=degrees, shift=shift)


def _small(n=400, C=1):
    sc = scene.make_scene(n_max=n, sh_degree=3, seed=0)
    K = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:C].astype(np.float32)
    vm = sc["viewmats"][:C].astype(np.float32)
    return dict(means=sc["means"], quats=sc["quats"], scales=(sc["scales"] * 4.0).astype(np.float32),
                opacities=sc["opacities"], colors=sc["colors"].astype(np.float32), sh=sc["sh"], viewmats=vm,
                viewmats_rs=_end_pose(vm), Ks=K)


def _coeffs(coeffs, shape=(1,)):
    return {KEYS[k]: _t(np.tile(np.float32(v), shape + (1,))) for k, v in coeffs.items()}


def _project(p, kind, co, shutter, vm_rs=None):
    vm_rs = p["viewmats_rs"] if vm_rs is None else vm_rs
    rs = dict(rolling_shutter=shutter, viewmats_rs=_t(vm_rs)) if shutter != 4 else {}
    return gs.fully_fused_projection_with_ut(_t(p["means"]), _t(p["quats"]), _t(p["scales"]), _t(p["opacities"]),
                                             _t(p["viewmats"]), _t(p["Ks"]), W, H, calc_compensations=True,
                                             camera_model=kind, **co, **rs)


def _lists(r, m2, d, C=1):
    _, ii, fl = gs.isect_tiles(m2, r, d, 16, TW, TH)
    return gs.isect_offset_encode(ii, C, TW, TH).reshape(C, TH, TW), fl


# ---- projection against the oracle
@pytest.mark.parametrize("shutter", SHUTTERS)
@pytest.mark.parametrize("kind,coeffs", CAMS)
def test_projection_against_oracle(kind, coeffs, shutter):
    p = _small()
    r, m2, d, co, cp = _project(p, kind, _coeffs(coeffs), shutter)
    cam = U.Camera(kind, p["Ks"][0], W, H, **coeffs)
    o = U.ut_projection(p["means"], p["quats"], p["scales"], p["opacities"],
                        U.ShutterPoses(p["viewmats"][0], p["viewmats_rs"][0], shutter), cam)
    r, ro = r[0].cpu().numpy(), o["radii"].numpy()
    frac = o["radii_unrounded"].numpy()
    edge = o["rs_edge"].numpy()
    on_int = (np.abs(frac - np.round(frac)) < 1e-3).any(-1)
    diff = (r != ro).any(-1)
    assert (diff & ~(on_int | edge)).sum() <= max(2, len(r) // 200), (diff & ~(on_int | edge)).sum()
    ok = (r > 0).all(-1) & (ro > 0).all(-1)
    assert ok.sum() > 50
    clean = ok & ~edge
    np.testing.assert_allclose(m2[0].cpu().numpy()[clean], o["means2d"].numpy()[clean], rtol=1e-4, atol=5e-3)
    np.testing.assert_allclose(d[0].cpu().numpy()[ok], o["depths"].numpy()[ok], rtol=1e-5)
    c, cref = co[0].cpu().numpy()[clean], o["conics"].numpy()[clean]
    np.testing.assert_allclose(c, cref, rtol=5e-3, atol=5e-3 * np.abs(cref).max())
    # a sigma point on a row boundary may take the neighbouring row's pose: one row's worth of motion, a fraction of
    # a pixel here, bounds its mean's shift
    if (ok & edge).any():
        assert np.abs(m2[0].cpu().numpy()[ok & edge] - o["means2d"].numpy()[ok & edge]).max() < 0.5


# ---- eval3d forward and gradients against the oracle
def _eval_case(p, kind, coeffs, shutter, offs, fl, bg):
    co = _coeffs(coeffs)
    leaves = [_t(x, True) for x in (p["means"], p["quats"], p["scales"], p["colors"][None], p["opacities"][None], bg)]
    rc, ra = gs.rasterize_to_pixels_eval3d(*leaves[:5], _t(p["viewmats"]), _t(p["Ks"]), W, H, 16, offs, fl,
                                           backgrounds=leaves[5], camera_model=kind, rolling_shutter=shutter,
                                           viewmats_rs=_t(p["viewmats_rs"]), **co)
    return leaves, rc, ra


def _check_against_oracle(p, kind, coeffs, shutter, offs, fl, bg, leaves, rc, ra, v_rc, v_ra, ref=None):
    N = len(p["means"])
    cam = U.Camera(kind, p["Ks"][0], W, H, **coeffs)
    f8 = [torch.from_numpy(np.asarray(x, np.float64)).requires_grad_(True)
          for x in (p["means"], p["quats"], p["scales"], p["colors"], p["opacities"], bg[0])]
    oc, oa, margin = U.eval3d_render(*f8[:5], U.ShutterPoses(p["viewmats"][0], p["viewmats_rs"][0], shutter), cam, offs.cpu(),
                                     fl.cpu().tolist(), 1, N, 0, background=f8[5])
    ((oc * torch.from_numpy(v_rc[0].astype(np.float64))).sum() + (oa * torch.from_numpy(v_ra[0].astype(np.float64))).sum()).backward()
    clear = (margin > 1e-3).numpy()
    target_c = oc.detach().numpy() if ref is None else ref["render_colors"][0]
    target_a = oa[..., 0].detach().numpy() if ref is None else ref["render_alphas"][0][..., 0]
    err = np.abs(rc[0].detach().cpu().numpy() - target_c).max(-1)
    aerr = np.abs(ra[0, ..., 0].detach().cpu().numpy() - target_a)
    bad = err > 2e-4
    assert (bad & clear).sum() <= max(1, clear.size // 1000), (bad & clear).sum()
    assert (bad & ~clear).sum() <= max(8, clear.size // 50), (bad & ~clear).sum()
    assert ((aerr > 2e-4) & clear).sum() <= max(1, clear.size // 1000)
    for i, name in enumerate(("means", "quats", "scales", "colors", "opacities", "backgrounds")):
        g = leaves[i].grad.detach().cpu().numpy().reshape(-1)
        gr = (f8[i].grad.numpy() if ref is None else ref[f"v_{name}"]).reshape(-1)
        rel = np.linalg.norm(g - gr) / max(np.linalg.norm(gr), 1e-12)
        assert rel < 2e-2, (name, rel)


@pytest.mark.parametrize("shutter", SHUTTERS)
@pytest.mark.parametrize("kind,coeffs", CAMS3)
def test_eval3d_against_oracle(kind, coeffs, shutter):
    p = _small()
    r, m2, d, _, _ = _project(p, kind, _coeffs(coeffs), shutter)
    offs, fl = _lists(r, m2, d)
    assert fl.numel() > 50
    rng = np.random.RandomState(1)
    bg = rng.random_sample((1, 3)).astype(np.float32)
    leaves, rc, ra = _eval_case(p, kind, coeffs, shutter, offs, fl, bg)
    v_rc = rng.standard_normal(rc.shape).astype(np.float32)
    v_ra = rng.standard_normal(ra.shape).astype(np.float32)
    ((rc * _t(v_rc)).sum() + (ra * _t(v_ra)).sum()).backward()
    _check_against_oracle(p, kind, coeffs, shutter, offs, fl, bg, leaves, rc, ra, v_rc, v_ra)


# ---- against the reference's records
@pytest.mark.parametrize("sname", list(SNAMES))
@pytest.mark.parametrize("cname", ["pinhole", "pinhole_distorted", "fisheye_radial"])
def test_kernels_against_reference(cname, sname):
    z = np.load(REF_NPZ)
    model = "fisheye" if cname.startswith("fisheye") else "pinhole"
    coeffs = {short: z[f"{cname}/{k}"][0] for short, k in KEYS.items() if f"{cname}/{k}" in z.files}
    p = {k: z[k] for k in ("means", "quats", "scales", "opacities", "colors", "viewmats", "viewmats_rs", "Ks")}
    name, shutter = f"{cname}/{sname}", SNAMES[sname]
    r, m2, d, cn, cp = _project(p, model, _coeffs(coeffs), shutter)
    cam = U.Camera(model, p["Ks"][0], W, H, **coeffs)
    o = U.ut_projection(p["means"], p["quats"], p["scales"], p["opacities"],
                        U.ShutterPoses(p["viewmats"][0], p["viewmats_rs"][0], shutter), cam)
    frac = o["radii_unrounded"].numpy()
    loose = o["rs_edge"].numpy() | (np.abs(frac - np.round(frac)) < 1e-3).any(-1)
    r, rr = r[0].cpu().numpy(), z[f"{name}/radii"][0]
    diff = (r != rr).any(-1)
    assert (diff & ~loose).sum() <= max(1, len(r) // 200), (diff & ~loose).sum()
    ok = (r > 0).all(-1) & (rr > 0).all(-1) & ~loose
    np.testing.assert_allclose(m2[0].cpu().numpy()[ok], z[f"{name}/means2d"][0][ok], rtol=1e-4, atol=5e-3)
    np.testing.assert_allclose(d[0].cpu().numpy()[ok], z[f"{name}/depths"][0][ok], rtol=1e-5)
    # compositing with the reference's own lists
    offs, fl = _t(z[f"{name}/isect_offsets"]), _t(z[f"{name}/flatten_ids"])
    bg, v_rc, v_ra = cotangents(int(z["cotangent_seed"]), 1, p["colors"].shape[-1], p["colors"].shape[-1])
    leaves, rc, ra = _eval_case(p, model, coeffs, shutter, offs, fl, bg)
    ((rc * _t(v_rc)).sum() + (ra * _t(v_ra)).sum()).backward()
    ref = {k: z[f"{name}/{k}"] for k in ("render_colors", "render_alphas", "v_means", "v_quats", "v_scales", "v_colors",
                                          "v_opacities", "v_backgrounds")}
    ref["v_colors"] = ref["v_colors"][0]
    ref["v_opacities"] = ref["v_opacities"][0]
    _check_against_oracle(p, model, coeffs, shutter, offs, fl, bg, leaves, rc, ra, v_rc, v_ra, ref=ref)


# ---- row (column) identity: each row of a rolling render is the global render at that row's pose
@pytest.mark.parametrize("shutter", [0, 1])
def test_rows_and_columns_are_global_renders_at_their_pose(shutter):
    p = _small()
    kind, coeffs = CAMS[1]
    co = _coeffs(coeffs)
    r, m2, d, _, _ = _project(p, kind, co, shutter)
    offs, fl = _lists(r, m2, d)
    args = (_t(p["means"]), _t(p["quats"]), _t(p["scales"]), _t(p["colors"][None]), _t(p["opacities"][None]))
    bg = _t(np.float32([[0.2, 0.4, 0.6]]))
    rc, ra = gs.rasterize_to_pixels_eval3d(*args, _t(p["viewmats"]), _t(p["Ks"]), W, H, 16, offs, fl, backgrounds=bg,
                                           camera_model=kind, rolling_shutter=shutter, viewmats_rs=_t(p["viewmats_rs"]), **co)
    poses = U.ShutterPoses(p["viewmats"][0], p["viewmats_rs"][0], shutter)
    n = H if shutter == 0 else W
    R, tt = poses.at(torch.arange(n, dtype=torch.float64) / (n - 1))
    worst = 0.0
    for k in range(n):
        vm = np.eye(4)
        vm[:3, :3], vm[:3, 3] = R[k].numpy(), tt[k].numpy()
        gc, ga = gs.rasterize_to_pixels_eval3d(*args, _t(vm[None].astype(np.float32)), _t(p["Ks"]), W, H, 16, offs, fl,
                                               backgrounds=bg, camera_model=kind, **co)
        a_row = rc[0, k] if shutter == 0 else rc[0, :, k]
        g_row = gc[0, k] if shutter == 0 else gc[0, :, k]
        worst = max(worst, float((a_row - g_row).abs().max()))
        al = ra[0, k] if shutter == 0 else ra[0, :, k]
        gl = ga[0, k] if shutter == 0 else ga[0, :, k]
        assert torch.allclose(al, gl, atol=1e-4, rtol=0), k
    assert worst < 1e-4, worst
    assert (ra > 0).any()


# ---- no motion: the rolling path is the global path
@pytest.mark.parametrize("shutter", SHUTTERS)
def test_no_motion_matches_global(shutter):
    p = _small()
    kind, coeffs = CAMS[5]
    co = _coeffs(coeffs)
    g = _project(p, kind, co, 4)
    rs = _project(p, kind, co, shutter, vm_rs=p["viewmats"])
    same = (g[0] == rs[0]).all(-1)[0]
    assert same.float().mean() > 0.99
    vis = same & (g[0][0] > 0).all(-1)
    assert vis.sum() > 50
    # the rotation comes from the pose's quaternion: the tolerances of test_projection_against_oracle
    for a, b in zip(g[1:], rs[1:]):
        torch.testing.assert_close(b[0][vis], a[0][vis], rtol=2e-3, atol=2e-3 * float(a[0][vis].abs().max()))
    offs, fl = _lists(*[x for x in (g[0], g[1], g[2])])
    args = (_t(p["means"]), _t(p["quats"]), _t(p["scales"]), _t(p["colors"][None]), _t(p["opacities"][None]), _t(p["viewmats"]),
            _t(p["Ks"]), W, H, 16, offs, fl)
    gc, ga = gs.rasterize_to_pixels_eval3d(*args, camera_model=kind, **co)
    rc, ra = gs.rasterize_to_pixels_eval3d(*args, camera_model=kind, rolling_shutter=shutter, viewmats_rs=_t(p["viewmats"]), **co)
    torch.testing.assert_close(rc, gc, rtol=0, atol=1e-4)
    torch.testing.assert_close(ra, ga, rtol=0, atol=1e-4)


# ---- rasterization()
def _rast(p, kind, co, vm, vm_rs, shutter=0, colour="sh", **kw):
    L = kw.pop("L")
    return gs.rasterization(L["means"], L["quats"], L["scales"], L["opacities"], L[colour], vm, _t(p["Ks"]), W, H,
                            sh_degree=3 if colour == "sh" else None, packed=False, with_ut=True, with_eval3d=True,
                            camera_model=kind, rolling_shutter=shutter, viewmats_rs=vm_rs, **co, **kw)


def test_rasterization_equals_hand_chain():
    C = 2
    p = _small(C=C)
    kind, coeffs = CAMS[1]
    co = _coeffs(coeffs, (C,))
    L = {k: _t(p[k]) for k in ("means", "quats", "scales", "opacities", "sh")}
    vm, vm_rs = _t(p["viewmats"]), _t(p["viewmats_rs"])
    bg = _t(np.float32([[0.1, 0.2, 0.3], [0.3, 0.2, 0.1]]))
    rc, ra, meta = _rast(p, kind, co, vm, vm_rs, L=L, backgrounds=bg)
    rs = dict(rolling_shutter=0, viewmats_rs=vm_rs)
    r, m2, d, _, _ = gs.fully_fused_projection_with_ut(L["means"], L["quats"], L["scales"], L["opacities"], vm, _t(p["Ks"]), W, H,
                                                      camera_model=kind, **co, **rs)
    feat = torch.clamp_min(gs.spherical_harmonics(3, L["means"], vm, L["sh"], masks=(r > 0).all(-1), viewmats_rs=vm_rs) + 0.5, 0.0)
    offs, fl = _lists(r, m2, d, C)
    opac = torch.broadcast_to(L["opacities"][None], (C, len(p["means"])))
    hc, ha = gs.rasterize_to_pixels_eval3d(L["means"], L["quats"], L["scales"], feat, opac, vm, _t(p["Ks"]), W, H, 16, offs, fl,
                                           backgrounds=bg, camera_model=kind, **co, **rs)
    assert torch.equal(meta["flatten_ids"], fl) and torch.equal(meta["isect_offsets"], offs)
    assert torch.equal(rc, hc) and torch.equal(ra, ha) and (ra > 0).any()


def test_rasterization_against_reference_orchestrator():
    z = np.load(REF_RASTER_NPZ)
    C = z["viewmats"].shape[0]
    q = {k: z[k] for k in ("means", "quats", "scales", "opacities", "sh", "viewmats", "viewmats_rs", "Ks")}
    co = {k: _t(z[k]) for k in KEYS.values() if k in z.files}
    L = {k: _t(q[k], True) for k in ("means", "quats", "scales", "opacities", "sh", "viewmats", "viewmats_rs")}
    bg_np, v_rc, v_ra = cotangents(int(z["cotangent_seed"]), C, 3, 4)
    bg = _t(bg_np, True)
    rc, ra, meta = gs.rasterization(L["means"], L["quats"], L["scales"], L["opacities"], L["sh"], L["viewmats"], _t(q["Ks"]), W, H,
                                    sh_degree=int(z["sh_degree"]), packed=False, backgrounds=bg, render_mode="RGB+ED",
                                    with_ut=True, with_eval3d=True, camera_model="pinhole",
                                    rolling_shutter=int(z["rolling_shutter"]), viewmats_rs=L["viewmats_rs"], **co)
    ((rc * _t(v_rc)).sum() + (ra * _t(v_ra)).sum()).backward()
    ref_r = z["radii"]
    diff = (meta["radii"].cpu().numpy() != ref_r).any(-1)
    assert diff.sum() <= max(2, diff.size // 100), diff.sum()
    vis = (ref_r > 0).all(-1) & ~diff
    np.testing.assert_allclose(meta["depths"].cpu().numpy()[vis], z["depths"][vis], rtol=1e-5)
    np.testing.assert_allclose(meta["means2d"].cpu().numpy()[vis], z["means2d"][vis], rtol=1e-4, atol=5e-3)
    got_c, got_a = rc.detach().cpu().numpy(), ra.detach().cpu().numpy()
    ref_c, ref_a = z["render_colors"], z["render_alphas"]
    err = np.abs(got_c[..., :3] - ref_c[..., :3]).max(-1)
    assert (err > 2e-4).mean() < 0.01, (err > 2e-4).mean()
    assert (np.abs(got_a - ref_a) > 2e-4).mean() < 0.01
    for k, leaf in list(L.items()) + [("backgrounds", bg)]:
        g, gr = leaf.grad.detach().cpu().numpy().reshape(-1), z[f"v_{k}"].reshape(-1)
        rel = np.linalg.norm(g - gr) / max(np.linalg.norm(gr), 1e-12)
        assert rel < 2e-2, (k, rel)
    # the poses' gradients come from the SH view directions only
    assert float(L["viewmats_rs"].grad.abs().sum()) > 0


def test_sh_gradient_splits_between_the_poses():
    p = _small(C=2)
    m = _t(p["means"])
    vm, vm_rs = _t(p["viewmats"], True), _t(p["viewmats_rs"], True)
    sh = _t(p["sh"])
    out = gs.spherical_harmonics(3, m, vm, sh, viewmats_rs=vm_rs)
    # the same as the global SH seen from the mean camera position
    mid = U.rs_sh_viewmat(p["viewmats"], p["viewmats_rs"]).float().to(DEV)
    torch.testing.assert_close(out, gs.spherical_harmonics(3, m, mid, sh), rtol=1e-5, atol=1e-5)
    x = gso.spherical_harmonics(3, p["means"].astype(np.float64), mid.cpu().double().numpy(), p["sh"].astype(np.float64))
    np.testing.assert_allclose(out.detach().cpu().numpy(), x, rtol=1e-4, atol=1e-5)
    out.square().sum().backward()
    assert float(vm.grad.abs().sum()) > 0 and float(vm_rs.grad.abs().sum()) > 0


def test_batch_dims_and_cameras():
    p = _small(C=2, n=300)
    kind, coeffs = CAMS[1]
    N = len(p["means"])
    means = np.stack([p["means"], p["means"] + 0.01])
    quats, scales, opac = (np.stack([p[k]] * 2) for k in ("quats", "scales", "opacities"))
    vm, vm_rs, K = np.stack([p["viewmats"]] * 2), np.stack([p["viewmats_rs"], p["viewmats"]]), np.stack([p["Ks"]] * 2)
    rng = np.random.RandomState(9)
    colors = rng.random_sample((2, 2, N, 3)).astype(np.float32)
    co = {KEYS[k]: np.tile(np.float32(v), (2, 2, 1)) for k, v in coeffs.items()}
    rc, ra, meta = gs.rasterization(_t(means), _t(quats), _t(scales), _t(opac), _t(colors), _t(vm), _t(K), W, H, packed=False,
                                    with_ut=True, with_eval3d=True, camera_model=kind, rolling_shutter=2,
                                    viewmats_rs=_t(vm_rs), **{k: _t(v) for k, v in co.items()})
    assert rc.shape == (2, 2, H, W, 3) and meta["n_batches"] == 2 and meta["n_cameras"] == 2
    for b in range(2):
        for c in range(2):
            one_c, one_a, _ = gs.rasterization(
                _t(means[b]), _t(quats[b]), _t(scales[b]), _t(opac[b]), _t(colors[b, c : c + 1]), _t(vm[b, c : c + 1]),
                _t(K[b, c : c + 1]), W, H, packed=False, with_ut=True, with_eval3d=True, camera_model=kind, rolling_shutter=2,
                viewmats_rs=_t(vm_rs[b, c : c + 1]), **{k: _t(v[b, c : c + 1]) for k, v in co.items()},
            )
            assert torch.equal(one_c[0], rc[b, c]) and torch.equal(one_a[0], ra[b, c]), (b, c)
            assert (one_a > 0).any()


def test_dropin_serves_rolling_shutter(monkeypatch):
    from gsplat_b200 import dropin

    calls = []

    def stock_rasterization(*a, **k):
        calls.append(k.get("camera_model"))
        return "stock"

    Wm = types.ModuleType("gsplat.cuda._wrapper")
    for n in dropin._OPS:
        setattr(Wm, n, lambda *a, **k: None)
    Wm.adam = lambda *a, **k: None
    R = types.ModuleType("gsplat.rendering")
    R.rasterization = stock_rasterization
    G = types.ModuleType("gsplat")
    G.__file__ = "stub"
    rel = types.ModuleType("gsplat.relocation")
    rel.compute_relocation = lambda *a, **k: None
    sops = types.ModuleType("gsplat.strategy.ops")
    sops.compute_relocation = rel.compute_relocation
    for name, mod in (("gsplat", G), ("gsplat.cuda", types.ModuleType("gsplat.cuda")), ("gsplat.cuda._wrapper", Wm),
                      ("gsplat.rendering", R), ("gsplat.relocation", rel), ("gsplat.strategy", types.ModuleType("gsplat.strategy")),
                      ("gsplat.strategy.ops", sops), ("gsplat.losses", types.ModuleType("gsplat.losses")),
                      ("gsplat.optimizers", types.ModuleType("gsplat.optimizers"))):
        monkeypatch.setitem(sys.modules, name, mod)
    dropin.apply(losses=False)
    try:
        st = dropin.stats["rasterization"]
        b0, s0 = st["b200"], st["stock"]
        p = _small()
        kind, coeffs = CAMS[1]
        args = (_t(p["means"]), _t(p["quats"]), _t(p["scales"]), _t(p["opacities"]), _t(p["sh"]), _t(p["viewmats"]), _t(p["Ks"]), W, H)
        rc, ra, meta = R.rasterization(*args, sh_degree=3, packed=False, with_ut=True, with_eval3d=True, camera_model=kind,
                                       rolling_shutter=gs.RollingShutterType.ROLLING_LEFT_TO_RIGHT,
                                       viewmats_rs=_t(p["viewmats_rs"]), **_coeffs(coeffs))
        assert rc.shape == (1, H, W, 3) and (ra > 0).any()
        assert calls == [] and st["b200"] == b0 + 1 and st["stock"] == s0
    finally:
        dropin.undo()


def test_fit_to_a_rolling_shutter_target():
    p = _small()
    kind, coeffs = CAMS[1]
    co = _coeffs(coeffs)
    shutter = 0
    N = len(p["means"])
    # the target: the float64 oracle's projection, its tile lists, and its compositing of the colours
    cam = U.Camera(kind, p["Ks"][0], W, H, **coeffs)
    o = U.ut_projection(p["means"], p["quats"], p["scales"], p["opacities"],
                        U.ShutterPoses(p["viewmats"][0], p["viewmats_rs"][0], shutter), cam)
    offs, fl = _lists(_t(o["radii"].numpy().astype(np.int32)[None]), _t(o["means2d"].numpy().astype(np.float32)[None]),
                      _t(o["depths"].numpy().astype(np.float32)[None]))
    f8 = [torch.from_numpy(np.asarray(p[k], np.float64)) for k in ("means", "quats", "scales", "colors", "opacities")]
    with torch.no_grad():
        gt, _, _ = U.eval3d_render(*f8, U.ShutterPoses(p["viewmats"][0], p["viewmats_rs"][0], shutter), cam, offs.cpu(),
                                   fl.cpu().tolist(), 1, N, 0)
    gt = gt.float().to(DEV)[None]
    g = torch.Generator(device="cpu").manual_seed(13)
    params = {
        "means": _t(p["means"] + 0.01 * torch.randn((N, 3), generator=g).numpy(), True),
        "quats": _t(p["quats"], True),
        "log_scales": _t(np.log(p["scales"] * 0.7), True),
        "logit_opac": _t(np.full(N, 0.0, np.float32), True),
        "colors": _t(np.full((N, 3), 0.5, np.float32), True),
    }
    opt = torch.optim.Adam([
        {"params": [params["means"]], "lr": 2e-3}, {"params": [params["quats"]], "lr": 1e-2},
        {"params": [params["log_scales"]], "lr": 1e-2}, {"params": [params["logit_opac"]], "lr": 5e-2},
        {"params": [params["colors"]], "lr": 5e-2},
    ])
    vm, vm_rs = _t(p["viewmats"]), _t(p["viewmats_rs"])
    losses = []
    for _ in range(100):
        rc, _, _ = gs.rasterization(params["means"], params["quats"], torch.exp(params["log_scales"]),
                                    torch.sigmoid(params["logit_opac"]), params["colors"], vm, _t(p["Ks"]), W, H, packed=False,
                                    with_ut=True, with_eval3d=True, camera_model=kind, rolling_shutter=shutter,
                                    viewmats_rs=vm_rs, **co)
        loss = (rc - gt).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(np.isfinite(losses))
    assert losses[-1] < 0.5 * losses[0], (losses[0], losses[-1])
