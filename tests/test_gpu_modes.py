"""GPU tests of the rasterization() configurations beyond classic RGB with SH colours: antialiased compositing (the
compensation backward), the depth render modes, covariance input, pose gradients, batch dimensions,
post-activation colours, orthographic / fisheye cameras and fp16 SH storage.

C1 checks the projection backward kernels with a compensation cotangent against the float32 oracle (and the
reference's golden gradients), C2 runs rasterization() end to end against the float64 oracle chain with the
contract of test_gpu_parity._pipeline_case, C3 checks fp16 SH coefficients on every path.
Run on a GPU machine:  pytest -m gpu
"""
import numpy as np
import pytest
import torch

from oracle import gso
from tests import scene
from tests.test_gpu_parity import _load, _n, _pipeline_case, _t, gs  # noqa: F401  (gs: fixture)

pytestmark = pytest.mark.gpu

W, H = 320, 200  # 200 = 12.5 tiles: a partial tile row


def _rel(a, ref):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    return np.linalg.norm(a - ref) / np.linalg.norm(ref)


# ------------------------------------------------------------------------------------------ C1
def _proj_inputs(model, C, covars):
    g = _load("ref_projection.npz" if model == "pinhole" else f"ref_projection_{model}.npz")
    d = {k: np.ascontiguousarray(g[k][:C]) if k in ("viewmats", "Ks") else g[k] for k in ("means", "quats", "scales", "viewmats", "Ks")}
    d["covars"] = gso.quat_scale_to_covar_preci(d["quats"], d["scales"], True, False, True)[0] if covars else None
    rng = np.random.RandomState(C + 7 * covars)
    cot = {k: rng.standard_normal(g[k][:C].shape).astype(np.float32) for k in ("v_means2d", "v_depths", "v_conics")}
    cot["v_compensations"] = rng.standard_normal(g["v_depths"][:C].shape).astype(np.float32)
    return g, d, int(g["width"]), int(g["height"]), cot


def _proj_oracle(d, W_, H_, model, cot, radii, conics, comps):
    vis = (radii > 0).all(-1)
    m = lambda a: (a * (vis[..., None] if a.ndim > vis.ndim else vis)).astype(np.float32)  # noqa: E731
    return gso.fully_fused_projection_bwd(
        d["means"], d["covars"], None if d["covars"] is not None else d["quats"],
        None if d["covars"] is not None else d["scales"], d["viewmats"], d["Ks"], W_, H_, 0.3, radii, conics, comps,
        m(cot["v_means2d"]), m(cot["v_depths"]), m(cot["v_conics"]), m(cot["v_compensations"]), True, model,
    )


@pytest.mark.parametrize("model", ["pinhole", "ortho", "fisheye"])
@pytest.mark.parametrize("C", [1, 2])
@pytest.mark.parametrize("covars", [False, True])
@pytest.mark.parametrize("layout", ["dense", "packed", "sparse"])
def test_projection_bwd_with_compensation(gs, model, C, covars, layout):
    """Dense and packed projection backward with all four cotangents, v_compensations included, vs the float32
    oracle (rel L2 1e-5 pinhole / ortho, 2e-4 fisheye, 1e-3 v_viewmats -- the bounds of the projection tests)."""
    if layout == "sparse" and C > 1:
        pytest.skip("sparse_grad COO rows are checked with one camera (coalesced)")
    g, d, W_, H_, cot = _proj_inputs(model, C, covars)
    means, vm = _t(d["means"], True), _t(d["viewmats"], True)
    if covars:
        cv, q, s = _t(d["covars"], True), None, None
        params = (means, cv, vm)
    else:
        cv, q, s = None, _t(d["quats"], True), _t(d["scales"], True)
        params = (means, q, s, vm)
    packed = layout != "dense"
    out = gs.fully_fused_projection(
        means, cv, q, s, vm, _t(d["Ks"]), W_, H_, calc_compensations=True, camera_model=model, packed=packed,
        sparse_grad=layout == "sparse",
    )
    radii_d, _, _, con_d, comp_d = gs.fully_fused_projection(
        means, cv, q, s, vm, _t(d["Ks"]), W_, H_, calc_compensations=True, camera_model=model
    )
    vis = (radii_d > 0).all(-1)
    assert int(vis.sum()) > 300
    if packed:
        m2, dep, con, comp = out[5], out[6], out[7], out[8]
        sel = lambda k: _t(cot[k])[vis]  # noqa: E731
    else:
        m2, dep, con, comp = out[1], out[2], out[3], out[4]
        sel = lambda k: _t(cot[k])  # noqa: E731
    loss = (m2 * sel("v_means2d")).sum() + (dep * sel("v_depths")).sum() + (con * sel("v_conics")).sum()
    loss = loss + (comp * sel("v_compensations")).sum()
    grads = torch.autograd.grad(loss, params)
    grads = [x.to_dense() if x.is_sparse else x for x in grads]
    ov = _proj_oracle(d, W_, H_, model, cot, _n(radii_d), _n(con_d), _n(comp_d))
    tol = 2e-4 if model == "fisheye" else 1e-5
    names = ("v_means", "v_covars", "v_viewmats") if covars else ("v_means", "v_quats", "v_scales", "v_viewmats")
    refs = dict(v_means=ov[0], v_covars=ov[1], v_quats=ov[2], v_scales=ov[3], v_viewmats=ov[4])
    for a, name in zip(grads, names):
        rel = _rel(_n(a), refs[name])
        bound = 1e-3 if name == "v_viewmats" else tol
        assert rel < bound, f"{name}: rel L2 error vs f32 oracle {rel:.3e}"


def test_projection_bwd_with_compensation_vs_golden(gs):
    """The reference's own torch autograd gradients, compensation term included (golden cotangents): 2e-2 rel L2 as
    for the `_nc` twins in test_projection_vs_oracle_and_golden."""
    g = _load("ref_projection.npz")
    W_, H_ = int(g["width"]), int(g["height"])
    means, quats, scales, vm = (_t(g[k], True) for k in ("means", "quats", "scales", "viewmats"))
    radii, m2, dep, con, comp = gs.fully_fused_projection(means, None, quats, scales, vm, _t(g["Ks"]), W_, H_,
                                                          calc_compensations=True)
    valid = _t((g["radii"] > 0).all(-1))
    v = {k: _t(g[k].astype(np.float32)) for k in ("v_means2d", "v_depths", "v_conics", "v_compensations")}
    loss = ((m2 * v["v_means2d"]).sum(-1) * valid).sum() + (dep * v["v_depths"] * valid).sum()
    loss = loss + ((con * v["v_conics"]).sum(-1) * valid).sum() + (comp * v["v_compensations"] * valid).sum()
    grads = torch.autograd.grad(loss, (means, quats, scales, vm))
    sel = (g["radii"] > 0).all(-1).any(0)
    for a, name in zip(grads, ("v_means", "v_quats", "v_scales", "v_viewmats")):
        ref = g[name]
        a = _n(a)
        if name != "v_viewmats":
            a, ref = a[sel], ref[sel]
        rel = _rel(a, ref)
        assert rel < 2e-2, f"{name}: relative L2 error vs reference golden (with compensation) {rel:.3e}"


@pytest.mark.parametrize("C", [1, 2])
def test_fused_project_sh_bwd_with_compensation_and_depth(gs, C):
    """fused_project_sh backward (both ONE_CAM instantiations) with v_compensations and v_depths, vs the float32
    oracle projection + SH backward."""
    sc = scene.make_scene(n_max=20000, sh_degree=3)
    Ks = np.ascontiguousarray(scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:C])
    vm = np.ascontiguousarray(sc["viewmats"][:C])
    P = {k: _t(sc[k], True) for k in ("means", "quats", "scales", "sh")}
    radii, m2, dep, con, col, comp = gs.fused_project_sh(
        P["means"], P["quats"], P["scales"], _t(sc["opacities"]), P["sh"], _t(vm), _t(Ks), W, H, 3,
        calc_compensations=True,
    )
    o = gso.fully_fused_projection(sc["means"], None, sc["quats"], sc["scales"], vm, Ks, W, H, 0.3, 0.01, 1e10, 0.0,
                                   True, "pinhole", sc["opacities"])
    assert np.array_equal(_n(radii), o[0])
    vis = (o[0] > 0).all(-1)
    assert vis.sum() > 2000
    rng = np.random.RandomState(C)
    cot = [rng.standard_normal(x.shape).astype(np.float32) * (vis[..., None] if x.ndim == 3 else vis)
           for x in (m2, dep, con, col, comp)]
    loss = sum((x * _t(c)).sum() for x, c in zip((m2, dep, con, col, comp), cot))
    gm, gq, gsc, gsh = torch.autograd.grad(loss, (P["means"], P["quats"], P["scales"], P["sh"]))
    ov = gso.fully_fused_projection_bwd(sc["means"], None, sc["quats"], sc["scales"], vm, Ks, W, H, 0.3, o[0], o[3],
                                        o[4], cot[0], cot[1], cot[2], cot[4])
    raw = gso.spherical_harmonics(3, sc["means"], vm, sc["sh"], vis)
    v_col = (cot[3] * ((raw + np.float32(0.5)) >= 0)).astype(np.float32)
    v_sh, v_m_sh = gso.spherical_harmonics_bwd(3, sc["means"], vm, sc["sh"], vis, v_col)
    for a, ref, name in ((gm, ov[0] + v_m_sh, "v_means"), (gq, ov[2], "v_quats"), (gsc, ov[3], "v_scales"),
                         (gsh, v_sh, "v_sh")):
        rel = _rel(_n(a), ref)
        assert rel < 1e-5, f"{name}: rel L2 error vs f32 oracle {rel:.3e}"


# ------------------------------------------------------------------------------------------ C2
@pytest.fixture(scope="module")
def sc30k():
    sc = scene.make_scene(n_max=30000, sh_degree=3)
    return sc, scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)


_AA = dict(rasterize_mode="antialiased")
CASES = {
    "aa_fused_one_cam": dict(C=1, sh_degree=3, **_AA),
    "aa_fused_backgrounds": dict(C=2, sh_degree=3, backgrounds=True, **_AA),
    "aa_packed_sh2": dict(C=2, sh_degree=2, packed=True, **_AA),
    "rgbd_fused_one_cam": dict(C=1, sh_degree=1, render_mode="RGB+D"),
    "rgbd_fused": dict(C=2, sh_degree=1, render_mode="RGB+D"),
    "depth_only": dict(C=2, sh_degree=None, render_mode="D"),
    "aa_packed_rgb_ed": dict(C=2, sh_degree=1, packed=True, render_mode="RGB+ED", **_AA),
    "pose_dense_sh3": dict(C=2, sh_degree=3, viewmats_grad=True),
    "pose_packed_sh1": dict(C=2, sh_degree=1, packed=True, viewmats_grad=True),
    "batch_dense": dict(C=2, sh_degree=1, batch=2),
    "covars_dense": dict(C=2, sh_degree=1, covars=True),
    "covars_packed": dict(C=2, sh_degree=1, covars=True, packed=True),
    "colors_per_gauss": dict(C=2, sh_degree=None, colors="N"),
    "colors_per_view": dict(C=2, sh_degree=None, colors="CN"),
    "aa_ortho": dict(C=1, sh_degree=1, camera_model="ortho", **_AA),
    # the fisheye projection goes through atan2f and a dual-number Jacobian on the GPU: compared with the float32
    # oracle, render within the tolerance of test_rasterization_camera_models
    "aa_fisheye": dict(C=1, sh_degree=1, camera_model="fisheye", oracle_dtype=np.float32, render_tol=(2e-4, 2e-5), **_AA),
    "clip_planes": dict(C=2, sh_degree=1, near_plane=2.0, radius_clip=1.5, eps2d=0.1),
}


@pytest.mark.parametrize("case", list(CASES))
def test_rasterization_modes_vs_oracle(gs, sc30k, case):
    sc, Ks = sc30k
    cfg = dict(CASES[case])
    C, sh_degree = cfg.pop("C"), cfg.pop("sh_degree")
    if cfg.get("camera_model") == "ortho":
        Ks = Ks.copy()
        Ks[:, 0, 0], Ks[:, 1, 1] = 60.0, 60.0
    if isinstance(cfg.get("colors"), str):
        rng = np.random.RandomState(5)
        cfg["colors"] = rng.random_sample(((C,) if cfg["colors"] == "CN" else ()) + (sc["means"].shape[0], 5))
    rc, ra, meta, fwd = _pipeline_case(gs, sc, W, H, Ks, C, sh_degree, **cfg)
    if cfg.get("batch"):
        assert tuple(rc.shape[:2]) == (cfg["batch"], C) and meta["n_batches"] == cfg["batch"]
    assert meta["isect_offsets"].shape[-2] == 13 and fwd["flatten_ids"].shape[0] > 2000


# ------------------------------------------------------------------------------------------ C3
@pytest.mark.parametrize("path", ["dense_fused", "packed", "dense_pose"])
def test_fp16_sh_storage(gs, sc30k, path):
    """fp16 SH coefficients render exactly like their float32 upcast, and get the float32 gradient back in fp16."""
    sc, Ks = sc30k
    P = {k: _t(sc[k]) for k in ("means", "quats", "scales", "opacities")}
    vm = _t(sc["viewmats"][:2], path == "dense_pose")
    sh16 = _t(sc["sh"]).half()
    kw = dict(sh_degree=3, packed=path == "packed")
    v = None
    outs = []
    for coeffs in (sh16.clone().requires_grad_(True), sh16.float().requires_grad_(True)):
        rc, ra, _ = gs.rasterization(P["means"], P["quats"], P["scales"], P["opacities"], coeffs, vm, _t(Ks[:2]), W, H, **kw)
        if v is None:
            v = torch.randn_like(rc)
        (rc * v).sum().backward()
        outs.append((rc.detach(), ra.detach(), coeffs.grad))
    (rc16, ra16, g16), (rc32, ra32, g32) = outs
    assert torch.equal(rc16, rc32) and torch.equal(ra16, ra32)
    assert g16.dtype == torch.float16
    # the float32 gradient is summed with float atomics: two runs can differ in the last bits, which moves a
    # handful of entries across an fp16 rounding boundary
    exact = (g16 == g32.half()).float().mean().item()
    assert exact > 0.999, f"only {exact * 100:.3f}% of fp16 gradient entries equal the float32 gradient cast to fp16"
    torch.testing.assert_close(g16.float(), g32.half().float(), rtol=2e-3, atol=1e-6)
