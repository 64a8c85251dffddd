"""Self-check of the projection / intersection sweep (tests/projection_edges.py) on the CPU: the float32 oracle, which
follows the reference's projection, must agree with the float64 truth on every decided row of every configuration;
the undecided fraction is bounded per class, so that the GPU file keeps checking most of the sweep; the oracle's tile
lists cover every decided pixel of alpha >= 1/255; and the intended differences are asserted explicitly."""
import math

import numpy as np
import pytest

from oracle import gso
from tests import projection_edges as pe


@pytest.fixture(scope="module")
def sweep():
    return pe.make_sweep()


def _oracle32(rows, cfg):
    vm, Ks = cfg.camera_arrays()
    kw = cfg.kwargs()
    return gso.fully_fused_projection(
        rows["means"], rows["covars"] if cfg.covars else None, rows["quats"], rows["scales"], vm, Ks, kw["width"],
        kw["height"], kw["eps2d"], kw["near_plane"], kw["far_plane"], kw["radius_clip"], cfg.comp, kw["camera_model"],
        rows["opacities"] if cfg.opacities else None,
    )


def test_sweep_covers_the_edges(sweep):
    n = sum(r["means"].shape[0] for r in sweep.values())
    assert 4000 <= n <= 8000, n
    for fam, rows in sweep.items():
        cls = rows["cls"]
        for k in ("depth", "covariance", "covars", "opacity", "opacity*comp", "extend", "ratio_floor", "eps2d=0",
                  "degenerate", "bulk"):
            assert (cls == k).sum() >= 8, (fam, k)
    assert (sweep["pinhole"]["cls"] == "clamp").sum() >= 280
    assert (sweep["pinhole"]["cls"] == "radius_clip").sum() >= 40
    assert (sweep["ortho"]["cls"] == "offscreen").sum() >= 200
    for k in ("fisheye_axis", "fisheye_x=0", "fisheye_theta", "fisheye_wide"):
        assert (sweep["fisheye"]["cls"] == k).sum() >= 50, k
    # the depth rows sit exactly on the float32 planes
    z = sweep["pinhole"]["means"][:, 2]
    assert (z == np.float32(pe.NEAR)).sum() >= 3 and (z == np.float32(pe.FAR)).sum() >= 3


@pytest.mark.parametrize("cfg", pe.CONFIGS, ids=str)
def test_float32_oracle_matches_float64_truth(sweep, cfg):
    rows = sweep[cfg.family]
    tr = pe.truth(rows, cfg)
    # the float64 oracle itself agrees with the numpy restatement of the decisions
    assert (tr.values["radii"][tr.decided] == tr.radii[tr.decided]).all()
    msgs = pe.check_forward(rows, cfg, tr, *_oracle32(rows, cfg), what=f"float32 oracle {cfg}")
    assert not msgs, "\n".join(msgs)
    vis = tr.decided & (tr.radii > 0).all(-1)
    # (ortho rows sized for the perspective cameras are sub-pixel: with compensation, most fall below 1/255)
    assert vis.sum() > 0.3 * vis.size, f"{cfg}: only {vis.mean():.1%} of the rows are decided and visible"


@pytest.mark.parametrize("cfg", pe.GRAD_CONFIGS, ids=str)
def test_float32_oracle_backward_within_budget(sweep, cfg):
    rows = sweep[cfg.family]
    N = rows["means"].shape[0]
    tr = pe.truth(rows, cfg)
    ref, beta, cot = pe.grad_truth(rows, cfg, tr, pe.cotangents(cfg, N))
    vm, Ks = cfg.camera_arrays()
    kw = cfg.kwargs()
    radii, _, _, con, comp = _oracle32(rows, cfg)
    vmn, _, vq, vs, vv = gso.fully_fused_projection_bwd(
        rows["means"], None, rows["quats"], rows["scales"], vm, Ks, pe.W, pe.H, kw["eps2d"], radii, con, comp,
        cot["v_means2d"], cot["v_depths"], cot["v_conics"], None, True, cfg.family,
    )
    msgs = pe.check_grads(rows, tr, dict(v_means=vmn, v_quats=vq, v_scales=vs, v_viewmats=vv), ref, beta,
                          f"float32 oracle backward {cfg}")
    assert not msgs, "\n".join(msgs)
    # the budgets are tight for most gaussians: the median budget is below 1e-4 of the gradient
    seen = (tr.decided & (tr.radii > 0).all(-1)).any(0)
    r = beta["v_means"][seen].max(-1) / np.abs(ref["v_means"][seen]).max(-1).clip(1e-30)
    assert np.median(r) < 1e-4, np.median(r)


def test_decisions_are_exercised(sweep):
    """each culling decision culls some decided rows and keeps decided rows next to it"""
    tr = pe.truth(sweep["pinhole"], pe.Config("pinhole"))
    cls, dec, vis = tr.cls, tr.decided[0], (tr.radii[0] > 0).all(-1)
    z = sweep["pinhole"]["means"][:, 2]
    # z == float32(near) is kept (the kernel compares pc.z < near), one ulp below is culled
    at_near = (z == np.float32(pe.NEAR)) & dec
    assert at_near.sum() >= 3 and vis[at_near].all()
    below = (z == np.nextafter(np.float32(pe.NEAR), np.float32(0))) & dec
    assert below.sum() >= 3 and not vis[below].any()
    at_far = (z == np.float32(pe.FAR)) & dec
    assert at_far.sum() >= 3 and vis[at_far].all()
    for k in ("opacity", "opacity*comp", "offscreen", "clamp", "covariance"):
        sel = (cls == k) & dec
        assert vis[sel].any(), k
    assert (~vis[(cls == "opacity") & dec]).sum() >= 3
    # the ortho border rows: x == -R exactly is culled (m2x + rx <= 0), one ulp inside is kept
    to = pe.truth(sweep["ortho"], pe.Config("ortho"))
    sel = (to.cls == "offscreen") & to.decided[0]
    m2 = sweep["ortho"]["means"][:, :2]
    r = to.radii[0]
    ortho_vis = (r > 0).all(-1)
    edge = sel & np.isin(m2[:, 0], -np.arange(3, 41, dtype=np.float32))
    assert edge.sum() >= 5 and not ortho_vis[edge].any()
    assert (sel & ortho_vis).sum() >= 30 and (sel & ~ortho_vis).sum() >= 30
    # radius_clip = 5 culls the rows whose radii are at most 5 and keeps the others
    tc = pe.truth(sweep["pinhole"], pe.Config("pinhole", radius_clip=pe.RCLIP))
    rc = (tc.cls == "radius_clip") & tc.decided[0]
    t0 = tr.radii[0][rc]
    assert ((t0 <= pe.RCLIP).all(-1)).sum() >= 10 and ((t0 > pe.RCLIP).any(-1)).sum() >= 10
    assert ((tc.radii[0][rc] > 0).all(-1) == (t0 > pe.RCLIP).any(-1)).all()


def test_undecided_fraction_is_bounded(sweep):
    print("\nundecided rows per class:")
    worst = {}
    for cfg in (pe.Config("pinhole", C=2), pe.Config("pinhole", C=2, comp=True), pe.Config("ortho"), pe.Config("fisheye"),
                pe.Config("pinhole", eps2d=0.0)):
        rep = pe.undecided_report(pe.truth(sweep[cfg.family], cfg))
        print(f"  {cfg}: " + ", ".join(f"{k} {v:.1%}" for k, v in rep.items()))
        if cfg.eps2d == 0.0:  # unblurred needles: det_blur itself cancels
            continue
        for k, v in rep.items():
            if cfg.comp and k == "ratio_floor":  # det_orig of a needle thinner than 1e-6 is rounding noise
                continue
            worst[k] = max(worst.get(k, 0.0), v)
    # the classes placed a few ulp from a decision are undecided by design for those rows
    # (radius>=2^31: the orthographic camera, fx = 1, puts these rows between 2^22 and 2^31, where float32 rounds the
    # radius; they are decided on the pinhole and fisheye cameras)
    limits = {"opacity": 0.6, "clamp": 0.4, "covariance": 0.2, "covars": 0.45, "opacity*comp": 0.4, "radius>=2^31": 1.0}
    for k, v in worst.items():
        assert v <= limits.get(k, 0.1), (k, v)


def test_radius_beyond_int32_saturates(sweep):
    """pinhole, fx = 500, z = 2, scales (1e7, 1e7, 1e-3): extend * sqrt(c00) ~ 8e9.  The kernels convert with
    cvt.rzi.s32.f32, which saturates: the row is kept with radius INT32_MAX (a plain C cast gives INT32_MIN on x86 and
    would cull it).  The oracle converts the same way, and its AABB then lists every tile."""
    rows = sweep["pinhole"]
    cfg = pe.Config("pinhole")
    tr = pe.truth(rows, cfg)
    sel = np.nonzero((tr.cls == "radius>=2^31") & tr.decided[0])[0]
    assert len(sel) >= 3
    assert (tr.radii[0, sel] == pe.INT32_MAX).all()
    for dt in (np.float32, np.float64):
        r = _oracle32({k: (v.astype(dt) if v.dtype == np.float32 else v) for k, v in rows.items()}, cfg)[0]
        assert (r[0, sel] == pe.INT32_MAX).all(), dt
    radii, m2, dep, con, _ = _oracle32(rows, cfg)
    tw, th = math.ceil(pe.W / 16), math.ceil(pe.H / 16)
    one = lambda a: np.ascontiguousarray(a[:, sel[:1]])  # noqa: E731
    tpg, _, _ = gso.isect_tiles(one(m2), one(radii), one(dep), 16, tw, th, True)
    assert tpg[0, 0] == tw * th


def test_float32_thresholds_matter(sweep):
    """At z = float32(0.01) the kernels keep the row (they compare with float(near_plane)); a truth that compared with
    the double 0.01 would cull it -- so the truth uses the float32 value of every threshold."""
    rows = sweep["pinhole"]
    sel = rows["means"][:, 2] == np.float32(pe.NEAR)
    cfg = pe.Config("pinhole")
    vm, Ks = cfg.camera_arrays()
    f8 = {k: v.astype(np.float64) for k, v in rows.items() if k != "cls"}
    args = (f8["means"], None, f8["quats"], f8["scales"], vm.astype(np.float64), Ks.astype(np.float64), pe.W, pe.H, 0.3)
    r32 = gso.fully_fused_projection(*args, pe.NEAR, pe.FAR, 0.0, False, "pinhole", f8["opacities"])[0]
    r64 = gso.fully_fused_projection(*args, 0.01, pe.FAR, 0.0, False, "pinhole", f8["opacities"])[0]
    assert (r32[0, sel] > 0).all(-1).sum() >= 3 and not (r64[0, sel] > 0).any()


def test_oracle_tiles_cover_decided_pixels(sweep):
    """AccuTile and the radius AABB of the oracle list every (gaussian, tile) with a decided pixel of alpha >= 1/255:
    on the 2D adversarial sets (247 and 425 tiles) and on the sweep's own projected rows"""
    rows = sweep["pinhole"]
    radii, m2, dep, con, _ = _oracle32(rows, pe.Config("pinhole"))
    sets = [("projected", m2, radii, dep, con, np.ascontiguousarray(rows["opacities"][None]), pe.W, pe.H)]
    for W2, H2 in ((304, 208), (400, 272)):
        a = pe.adversarial_2d(W2, H2)
        sets.append((f"2d {W2}x{H2}", a["means2d"], a["radii"], a["depths"], a["conics"], a["opacities"], W2, H2))
    for name, m2, radii, dep, con, op, W2, H2 in sets:
        tw, th = math.ceil(W2 / 16), math.ceil(H2 / 16)
        bits = gso.bits_for_count(tw * th)
        req = pe.required_tiles(m2, con, op, radii, W2, H2)
        assert len(req) > 100, name
        N = m2.shape[1]
        for accu in (True, False):
            kw = dict(conics=con, opacities=op) if accu else {}
            tpg, ids, fl = gso.isect_tiles(m2, radii, dep, 16, tw, th, True, **kw)
            miss = pe.missing_tiles(req, pe.listed_tiles(ids, fl, N, bits))
            assert not miss, f"{name} {'accu' if accu else 'aabb'}: {len(miss)} gaussians miss tiles, e.g. {miss[:3]}"
            if accu and name != "projected":
                assert (tpg > 64).sum() >= 10, "needles spanning more than 64 tiles take the cooperative emit"
