"""The 2DGS kernels on the adversarial sweep of tests/surfel_edges.py, against its float64 truth.

* Projection forward (C = 1, C = 2, radius_clip = 3): radii exact and means2d / depths / ray transforms / normals within
  their budgets on every decided row; culled rows have zero floats; radii of 2^31 or more are INT32_MAX and go through
  isect_tiles_sorted, whose lists equal the oracle's on the GPU's own projected rows.
* Projection backward (C = 1, C = 2 and a leading batch dim of 2 with N not a multiple of 32) against the float64
  backward within per-surfel entry-wise budgets.
* Compositing at exact ties: g3 == g2 takes the ray-splat kernel (v_ray_transforms twice the oracle's, which splits a
  tie evenly; v_means2d and absgrad zero), the median rule T > 0.5 and the exclusive transmittance stop on their
  float32 ties (median_ids / last_ids exact), and an alpha clamped at 0.99 gives no geometry or opacity gradient.
* Surfels with finite inputs whose float32 ray transform overflows change no pixel of a rendering; surfels whose ray
  transform fits float32 but whose ext = m2^2 - tmp overflows keep the radius of the kernel's float32 evaluation.
* A surfel drawn by the screen-space filter alone gets a zero v_ray_transforms and the oracle's v_means2d and absgrad.
"""
import math

import numpy as np
import pytest
import torch

from oracle import surfel
from tests import surfel_edges as se

pytestmark = pytest.mark.gpu
dev = "cuda"
f64 = torch.float64


@pytest.fixture(scope="module")
def gs():
    import gsplat_b200

    return gsplat_b200


@pytest.fixture(scope="module")
def rows():
    return se.make_rows()


def _t(a, grad=False):
    return torch.tensor(np.ascontiguousarray(a), device=dev).requires_grad_(grad)


def _n(t):
    return t.detach().cpu().double().numpy()


CONFIGS = [(1, 0.0), (2, 0.0), (1, se.RCLIP)]


def _project(gs, rows, C, clip, grad=False):
    vm, Ks = se.camera_arrays(C)
    leaves = [_t(rows[k], grad) for k in ("means", "quats", "scales")] + [_t(vm, grad)]
    out = gs.fully_fused_projection_2dgs(*leaves, _t(Ks), se.W, se.H, near_plane=se.NEAR, far_plane=se.FAR, radius_clip=clip)
    return leaves, out


@pytest.mark.parametrize("C,clip", CONFIGS)
def test_projection_forward_vs_truth(gs, rows, C, clip):
    tr = se.truth(rows, C, clip)
    _, out = _project(gs, rows, C, clip)
    print("\nundecided (rows, undecided pairs, pairs) per class:", se.undecided_report(tr))
    msgs = se.check_projection(rows, tr, *(o.cpu().numpy() for o in out), what=f"GPU C={C} clip={clip}")
    assert not msgs, "\n".join(msgs)


@pytest.mark.parametrize("C,clip", CONFIGS)
def test_projection_backward_vs_truth(gs, rows, C, clip):
    tr = se.truth(rows, C, clip)
    ref, beta, cot = se.grad_truth(rows, tr, clip, se.cotangents((C, rows["means"].shape[0])))
    leaves, out = _project(gs, rows, C, clip, grad=True)
    loss = sum((o * _t(cot[k])).sum() for o, k in zip(out[1:], ("means2d", "depths", "ray_transforms", "normals")))
    g = torch.autograd.grad(loss, leaves)
    got = dict(v_means=_n(g[0]), v_quats=_n(g[1]), v_scales=_n(g[2]), v_viewmats=_n(g[3]))
    assert (got["v_scales"][:, 2] == 0).all()
    msgs = se.check_grads(rows, tr, got, ref, beta, f"GPU C={C} clip={clip}")
    assert not msgs, "\n".join(msgs)


def test_projection_batch_dims_straddling_warps(gs, rows):
    """leading batch [2] with N = 77 rows per element: warps straddle the two elements, and v_viewmats takes the
    per-lane atomics; each element against its own truth"""
    N = 77
    bulk = np.nonzero(np.isin(rows["cls"], ("bulk", "quat_norm", "cosv", "ceil")))[0]
    parts = [se.subset(rows, bulk[(np.arange(N) * k + 3 * k) % len(bulk)]) for k in (1, 7)]
    C = 2
    truths = [se.truth(p, C) for p in parts]
    gts = [se.grad_truth(p, t, 0.0, se.cotangents((C, N), seed=b)) for b, (p, t) in enumerate(zip(parts, truths))]
    st = lambda k: np.stack([p[k] for p in parts])  # noqa: E731
    vm, Ks = se.camera_arrays(C)
    leaves = [_t(st(k), True) for k in ("means", "quats", "scales")] + [_t(np.stack([vm, vm]), True)]
    out = gs.fully_fused_projection_2dgs(*leaves, _t(np.stack([Ks, Ks])), se.W, se.H, near_plane=se.NEAR, far_plane=se.FAR)
    cot = {k: np.stack([g[2][k] for g in gts]) for k in ("means2d", "depths", "ray_transforms", "normals")}
    loss = sum((o * _t(cot[k])).sum() for o, k in zip(out[1:], ("means2d", "depths", "ray_transforms", "normals")))
    g = torch.autograd.grad(loss, leaves)
    for b in range(2):
        msgs = se.check_projection(parts[b], truths[b], *(_n(o[b]) for o in out), what=f"batch {b}")
        got = dict(v_means=_n(g[0])[b], v_quats=_n(g[1])[b], v_scales=_n(g[2])[b], v_viewmats=_n(g[3])[b])
        msgs += se.check_grads(parts[b], truths[b], got, gts[b][0], gts[b][1], f"batch element {b}")
        assert not msgs, "\n".join(msgs)


def test_radius_int32_max_and_tile_lists(gs, rows):
    """radii of 2^31 or more are INT32_MAX and list every tile; isect_tiles_sorted on the GPU's own projected rows
    (C = 2) equals the oracle's radius-box lists bit for bit"""
    C = 2
    _, (radii, m2, dep, _, _) = _project(gs, rows, C, 0.0)
    tr = se.truth(rows, C)
    big = (tr.cls == "radius>=2^31")[None] & tr.decided
    r = radii.cpu().numpy()
    assert big.sum() >= 8 and (r[big] == se.INT32_MAX).all()
    tw, th = math.ceil(se.W / 16), math.ceil(se.H / 16)
    hits = gs.ops.isect_tiles_sorted(m2, radii, dep, 16, tw, th)
    fl, off = surfel.isect(m2.cpu().numpy(), r, dep.cpu().numpy(), 16, tw, th)
    assert np.array_equal(hits.flatten_ids.cpu().numpy(), fl)
    assert np.array_equal(hits.isect_offsets.reshape(C, th, tw).cpu().numpy(), off)
    n_big_tiles = sum(int((np.asarray(fl) == c * r.shape[1] + n).sum()) for c, n in np.argwhere(big))
    assert n_big_tiles == int(big.sum()) * tw * th


# ------------------------------------------------------------------------------------------------------------------
# compositing at exact ties
def _tie_run(gs, D=3):
    ti = se.tie_images(D)
    leaves = {k: _t(ti[k], True) for k in ("means2d", "ray_transforms", "colors", "opacities", "normals")}
    densify = torch.zeros(ti["means2d"].shape, device=dev, requires_grad=True)
    outs = gs.rasterize_to_pixels_2dgs(
        leaves["means2d"], leaves["ray_transforms"], leaves["colors"], leaves["opacities"], leaves["normals"], densify,
        se.IW, se.IH, 16, _t(ti["isect_offsets"]), _t(ti["flatten_ids"]), absgrad=True)
    rng = np.random.RandomState(1)
    cots = [_t(rng.standard_normal(o.shape).astype(np.float32)) for o in outs]
    g = torch.autograd.grad(sum((o * c).sum() for o, c in zip(outs, cots)), list(leaves.values()))
    grads = dict(zip(leaves, (_n(x) for x in g)))
    grads["absgrad"] = _n(leaves["means2d"].absgrad)
    ref = surfel.rasterize_vjp(*(torch.tensor(ti[k], dtype=f64) for k in leaves), se.IW, se.IH, 16, ti["isect_offsets"],
                               ti["flatten_ids"], [c.cpu().double() for c in cots])
    return ti, outs, grads, ref


def _raw_ids(gs, ti, D=3):
    from gsplat_b200._cabi import ptr, stream

    I, N = ti["means2d"].shape[:2]
    o = lambda *s, dt=torch.float32: torch.empty(s, device=dev, dtype=dt)  # noqa: E731
    rc, ra, rn, rd, rm = o(I, se.IH, se.IW, D), o(I, se.IH, se.IW, 1), o(I, se.IH, se.IW, 3), o(I, se.IH, se.IW, 1), o(I, se.IH, se.IW, 1)
    li, mi = o(I, se.IH, se.IW, dt=torch.int32), o(I, se.IH, se.IW, dt=torch.int32)
    t = {k: _t(ti[k]) for k in ("means2d", "ray_transforms", "colors", "opacities", "normals", "isect_offsets", "flatten_ids")}
    rc_ = gs._cabi.lib().gsb200_surfel_raster_fwd(
        I, N, D, ptr(t["means2d"]), ptr(t["ray_transforms"]), ptr(t["colors"]), ptr(t["opacities"]), ptr(t["normals"]),
        None, None, se.IW, se.IH, 16, 3, 3, ptr(t["isect_offsets"]), ptr(t["flatten_ids"]), len(ti["flatten_ids"]), ptr(rc),
        ptr(ra), ptr(rn), ptr(rd), ptr(rm), ptr(li), ptr(mi), stream())
    assert rc_ == 0
    torch.cuda.synchronize()
    return li.cpu().numpy(), mi.cpu().numpy(), rm.cpu().numpy()


def test_kernel_choice_at_g3_equal_g2(gs):
    """every pixel of image 0 ties g3 == g2 exactly: the kernels take the ray-splat kernel (g3 <= g2)"""
    ti, outs, g, ref = _tie_run(gs)
    assert (_n(outs[1])[0] > 0).sum() >= 9
    vrt, ovrt = g["ray_transforms"][0, 0], 2.0 * ref["v_ray_transforms"].numpy()[0, 0]
    assert np.abs(ovrt).max() > 1e-3
    assert np.allclose(vrt, ovrt, rtol=1e-4, atol=1e-5 * np.abs(ovrt).max()), (vrt, ovrt)
    assert (g["means2d"][0, 0] == 0).all() and (g["absgrad"][0, 0] == 0).all(), (g["means2d"][0, 0], g["absgrad"][0, 0])


def test_median_and_stop_at_their_ties(gs):
    """T == 0.5 exactly before the median image's second surfel: the median stays on the first (T > 0.5); the stop
    image's fifth surfel brings next_T to float32(1e-4) exactly: it does not contribute (next_T <= 1e-4 stops)"""
    ti = se.tie_images()
    li, mi, rm = _raw_ids(gs, ti)
    (x1, y1), (x2, y2) = ti["centres"][1], ti["centres"][2]
    start1, start2 = ti["isect_offsets"][1].reshape(-1), ti["isect_offsets"][2].reshape(-1)
    tile1, tile2 = (y1 // 16) * 3 + x1 // 16, (y2 // 16) * 3 + x2 // 16
    assert li[1, y1, x1] == start1[tile1] + 1 and mi[1, y1, x1] == start1[tile1]
    assert rm[1, y1, x1, 0] == ti["colors"][1, 0, -1]
    last, _ = se.stop_chain_float32()
    assert last == 3
    assert li[2, y2, x2] == start2[tile2] + last, (li[2, y2, x2], start2[tile2])


def test_clamped_alpha_has_no_geometry_or_opacity_gradient(gs):
    """image 3: raw alpha > 0.99 on every pixel; the clamp's derivative is zero"""
    ti, outs, g, ref = _tie_run(gs)
    assert (np.abs(_n(outs[1])[3] - se.MAX_ALPHA) < 1e-6).all()
    for k in ("means2d", "ray_transforms", "opacities", "absgrad"):
        assert (g[k][3, 0] == 0).all(), (k, g[k][3, 0])
    assert np.abs(g["colors"][3, 0]).max() > 0
    np.testing.assert_allclose(g["colors"][3, 0], ref["v_colors"].numpy()[3, 0], rtol=1e-4, atol=1e-4)


def test_filter_only_surfel_has_no_ray_transform_gradient(gs):
    """image 4: g2 < g3 at every pixel, so only the screen-space filter draws the surfel"""
    ti, outs, g, ref = _tie_run(gs)
    assert (_n(outs[1])[4] > 0).sum() >= 4
    assert (g["ray_transforms"][4, 0] == 0).all(), g["ray_transforms"][4, 0]
    for k, rk in (("means2d", "v_means2d"), ("absgrad", "absgrad"), ("opacities", "v_opacities")):
        r = ref[rk].numpy()[4, 0]
        assert np.abs(r).max() > 1e-3, k
        np.testing.assert_allclose(g[k][4, 0], r, rtol=1e-4, atol=1e-5 * np.abs(r).max(), err_msg=k)


# ------------------------------------------------------------------------------------------------------------------
# the non-finite hazard
def test_overflowing_surfels_change_no_pixel(gs):
    """surfels with finite inputs whose float32 ray transform overflows (scale 1e37 .. 3e38) must not paint: rendering
    a scene with and without them gives the same image, bit for bit, and the projection culls them"""
    from tests import scene

    W, H = 128, 96
    sc = scene.make_scene(n_max=2000, sh_degree=1, seed=42)
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:1]
    vm = sc["viewmats"][:1]
    ov = se.overflow_rows()
    # the overflow rows are built in camera 0's frame of the sweep; move them into this scene's camera frame
    vm0 = se.CAMS[0][0].astype(np.float64)
    pc = (vm0[:3, :3] @ ov["means"].astype(np.float64).T).T + vm0[:3, 3]
    v64 = vm[0].astype(np.float64)
    means_ov = ((pc - v64[:3, 3]) @ v64[:3, :3]).astype(np.float32)
    quat_ov = ov["quats"]  # orientation is immaterial: every row overflows

    def render(extra):
        cat = lambda a, b: np.concatenate([a, b]) if extra else a  # noqa: E731
        args = dict(means=cat(sc["means"], means_ov), quats=cat(sc["quats"], quat_ov), scales=cat(sc["scales"] * 2, ov["scales"]),
                    opacities=cat(sc["opacities"], np.full(len(means_ov), 0.9, np.float32)),
                    colors=cat(sc["colors"], np.ones((len(means_ov), 3), np.float32)))
        out = gs.rasterization_2dgs(*(_t(args[k]) for k in ("means", "quats", "scales", "opacities", "colors")), _t(vm), _t(Ks),
                                    W, H, render_mode="RGB+ED")
        return out

    a, b = render(False), render(True)
    radii = b[6]["radii"][0, -len(means_ov):].cpu().numpy()
    m2 = b[6]["means2d"][0, -len(means_ov):].detach().cpu().numpy()
    print(f"\noverflow rows: radii {radii.tolist()}, means2d finite {np.isfinite(m2).all(-1).tolist()}")
    assert (radii == 0).all()
    for k, (x, y) in enumerate(zip(a[:6], b[:6])):
        if x is None:
            continue
        changed = (x != y).reshape(-1, x.shape[-1]).any(-1) if x.dim() > 2 else (x != y)
        assert not changed.any(), f"output {k}: {int(changed.sum())} pixels changed by the overflowing surfels"


def test_ext_overflow_radius_is_pinned(gs):
    """the ray transform (fx * scale, scales 1e19 .. 1e21) fits float32 and the screen mean is finite, but ext's squares
    overflow: the kernel keeps the row with the radius of the float32 evaluation (INT32_MAX here, as the float64 radius
    also is), so the surfel stays listed on every tile.  This records the behaviour; a change to it must be deliberate."""
    ov = se.ext_overflow_rows()
    vm, Ks = se.camera_arrays(1)
    radii, m2, dep, rt, _ = gs.fully_fused_projection_2dgs(*(_t(ov[k]) for k in ("means", "quats", "scales")), _t(vm), _t(Ks),
                                                          se.W, se.H, near_plane=se.NEAR, far_plane=se.FAR)
    want, finite = se.radii_float32(ov, 1)
    got = radii.cpu().numpy()
    print(f"\next overflow rows: radii {got[0].tolist()}")
    assert finite.all() and np.isfinite(_n(m2)).all() and np.isfinite(_n(rt)).all()
    assert np.array_equal(got, want), (got.tolist(), want.tolist())
    assert (got > 0).all()
