"""3DGUT operators on the GPU against the float64 oracle (oracle/ut.py): the UT projection, the eval3d compositing and
its gradients, batch dims, backgrounds and masks, determinism, and the full chain on the garden scene."""
import numpy as np
import pytest
import torch

import gsplat_b200 as gs
from oracle import ut as U
from tests import scene

pytestmark = pytest.mark.gpu
DEV = "cuda"
W, H = 96, 64
CAMS = [
    ("pinhole", {}),
    ("pinhole", dict(radial=[0.08, -0.03, 0.005, 0.01, 0.0, 0.0])),
    ("pinhole", dict(tangential=[0.004, -0.003])),
    ("pinhole", dict(thin=[0.002, -0.001, 0.001, 0.0005])),
    ("fisheye", {}),
    ("fisheye", dict(radial=[0.04, -0.01, 0.002, -0.0003])),
]
KEYS = {"radial": "radial_coeffs", "tangential": "tangential_coeffs", "thin": "thin_prism_coeffs"}


def _small(n=400, seed=0):
    sc = scene.make_scene(n_max=n, sh_degree=0, seed=seed)
    K = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:1].copy()
    return sc, sc["viewmats"][:1].copy(), K


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _coeffs(coeffs, C=1):
    return {KEYS[k]: _t(np.tile(np.float32(v), (C, 1))) for k, v in coeffs.items()}


def _scales(sc, f=4.0):
    return sc["scales"] * f  # a few pixels across at 96x64, so that pairs overlap


@pytest.mark.parametrize("kind,coeffs", CAMS)
def test_projection_against_oracle(kind, coeffs):
    sc, vm, K = _small()
    s = _scales(sc)
    r, m2, d, co, cp = gs.fully_fused_projection_with_ut(
        _t(sc["means"]), _t(sc["quats"]), _t(s), _t(sc["opacities"]), _t(vm), _t(K), W, H, calc_compensations=True,
        camera_model=kind, **_coeffs(coeffs),
    )
    cam = U.Camera(kind, K[0], W, H, **coeffs)
    o = U.ut_projection(sc["means"], sc["quats"], s, sc["opacities"], vm[0], cam)
    r = r[0].cpu().numpy()
    ro = o["radii"].numpy()
    # radii are exact except where the unrounded radius sits on an integer, or a cull decision is marginal
    frac = o["radii_unrounded"].numpy()
    on_edge = (np.abs(frac - np.round(frac)) < 1e-3).any(-1)
    diff = (r != ro).any(-1)
    assert (diff & ~on_edge).sum() <= max(2, len(r) // 200), (diff & ~on_edge).sum()
    ok = (r > 0).all(-1) & (ro > 0).all(-1)
    assert ok.sum() > 50
    np.testing.assert_allclose(m2[0].cpu().numpy()[ok], o["means2d"].numpy()[ok], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(d[0].cpu().numpy()[ok], o["depths"].numpy()[ok], rtol=1e-5)
    c, cref = co[0].cpu().numpy()[ok], o["conics"].numpy()[ok]
    np.testing.assert_allclose(c, cref, rtol=2e-3, atol=2e-3 * np.abs(cref).max())
    # the compensation is a ratio of determinants, det_orig being a difference of near-equal float32 products
    np.testing.assert_allclose(cp[0].cpu().numpy()[ok], o["compensations"].numpy()[ok], rtol=1e-2, atol=1e-4)
    culled = ~(r > 0).all(-1)
    assert (m2[0].cpu().numpy()[culled] == 0).all() and (co[0].cpu().numpy()[culled] == 0).all()


def _render(sc, vm, K, kind, coeffs, s, C=1, backgrounds=None, masks=None):
    means, quats, scales = _t(sc["means"]), _t(sc["quats"]), _t(s)
    r, m2, d, co, _ = gs.fully_fused_projection_with_ut(
        means, quats, scales, _t(sc["opacities"]), _t(vm), _t(K), W, H, camera_model=kind, **_coeffs(coeffs, C)
    )
    tw, th = (W + 15) // 16, (H + 15) // 16
    _, isect_ids, flatten_ids = gs.isect_tiles(m2, r, d, 16, tw, th)
    offs = gs.isect_offset_encode(isect_ids, C, tw, th)
    return offs.reshape(C, th, tw), flatten_ids


@pytest.mark.parametrize("kind,coeffs", CAMS)
def test_eval3d_forward_and_gradients_against_oracle(kind, coeffs):
    sc, vm, K = _small()
    s = _scales(sc)
    offs, fl = _render(sc, vm, K, kind, coeffs, s)
    assert fl.numel() > 50
    N = len(s)
    rng = np.random.RandomState(1)
    bg = rng.random_sample((1, 3)).astype(np.float32)
    colors = sc["colors"][None].astype(np.float32)
    opac = sc["opacities"][None].astype(np.float32)
    leaves = [_t(x).requires_grad_(True) for x in (sc["means"], sc["quats"], s, colors, opac, bg)]
    rc, ra = gs.rasterize_to_pixels_eval3d(
        leaves[0], leaves[1], leaves[2], leaves[3], leaves[4], _t(vm), _t(K), W, H, 16, offs, fl, backgrounds=leaves[5],
        camera_model=kind, **_coeffs(coeffs),
    )
    v_rc = rng.standard_normal(rc.shape).astype(np.float32)
    v_ra = rng.standard_normal(ra.shape).astype(np.float32)
    ((rc * _t(v_rc)).sum() + (ra * _t(v_ra)).sum()).backward()

    cam = U.Camera(kind, K[0], W, H, **coeffs)
    f8 = [torch.from_numpy(np.asarray(x, np.float64)).requires_grad_(True) for x in (sc["means"], sc["quats"], s, colors[0], opac[0], bg[0])]
    oc, oa, margin = U.eval3d_render(f8[0], f8[1], f8[2], f8[3], f8[4], vm[0], cam, offs.cpu(), fl.cpu().tolist(), 1, N, 0,
                                     background=f8[5])
    ((oc * torch.from_numpy(v_rc[0].astype(np.float64))).sum() + (oa * torch.from_numpy(v_ra[0].astype(np.float64))).sum()).backward()
    # pixels whose decisions all sit clear of a threshold must agree to float32 accuracy; the rest are counted and bounded
    clear = (margin > 1e-3).numpy()
    err = np.abs(rc[0].detach().cpu().numpy() - oc.detach().numpy()).max(-1)
    bad = err > 2e-4
    assert (bad & clear).sum() <= max(1, clear.size // 1000), (bad & clear).sum()
    assert (bad & ~clear).sum() <= max(8, clear.size // 50), (bad & ~clear).sum()
    aerr = np.abs(ra[0, ..., 0].detach().cpu().numpy() - oa[..., 0].detach().numpy())
    assert ((aerr > 2e-4) & clear).sum() <= max(1, clear.size // 1000)
    for name, a, b in zip(("means", "quats", "scales", "colors", "opacities", "backgrounds"), leaves, f8):
        g, gr = a.grad.detach().cpu().numpy().reshape(-1), b.grad.numpy().reshape(-1)
        rel = np.linalg.norm(g - gr) / max(np.linalg.norm(gr), 1e-12)
        assert rel < 2e-2, (name, rel)


def test_eval3d_bit_identical_batch_masks_and_empty():
    sc, vm, K = _small(n=300)
    s = _scales(sc)
    kind, coeffs = CAMS[1]
    vm2 = np.stack([vm[0], vm[0]])[None].repeat(2, 0)  # [B=2, C=2, 4, 4]
    K2 = np.stack([K[0], K[0]])[None].repeat(2, 0)
    means = np.stack([sc["means"], sc["means"] + 0.01])
    quats, scales = np.stack([sc["quats"]] * 2), np.stack([s] * 2)
    opac = np.stack([sc["opacities"]] * 2)
    co = {KEYS[k]: _t(np.tile(np.float32(v), (2, 2, 1))) for k, v in coeffs.items()}
    r, m2, d, _, _ = gs.fully_fused_projection_with_ut(_t(means), _t(quats), _t(scales), _t(opac), _t(vm2), _t(K2), W, H,
                                                      camera_model=kind, **co)
    tw, th = (W + 15) // 16, (H + 15) // 16
    _, ii, fl = gs.isect_tiles(m2, r, d, 16, tw, th)
    offs = gs.isect_offset_encode(ii, 4, tw, th).reshape(2, 2, th, tw)
    colors = _t(np.stack([np.stack([sc["colors"]] * 2)] * 2).astype(np.float32))
    opac_c = _t(np.stack([np.stack([sc["opacities"]] * 2)] * 2))
    bg = torch.rand(2, 2, 3, device=DEV)
    masks = torch.ones(2, 2, th, tw, dtype=torch.bool, device=DEV)
    masks[1, 0, 0, 0] = False
    args = (_t(means), _t(quats), _t(scales), colors, opac_c, _t(vm2), _t(K2), W, H, 16, offs, fl)
    a = gs.rasterize_to_pixels_eval3d(*args, backgrounds=bg, masks=masks, camera_model=kind, **co)
    b = gs.rasterize_to_pixels_eval3d(*args, backgrounds=bg, masks=masks, camera_model=kind, **co)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert a[0].shape == (2, 2, H, W, 3) and a[1].shape == (2, 2, H, W, 1)
    # a masked tile is the background
    assert torch.equal(a[0][1, 0, :16, :16], bg[1, 0].expand(16, 16, 3)) and (a[1][1, 0, :16, :16] == 0).all()
    assert (a[1][0, 0] > 0).any()
    # a batch entry equals the single-image render of its inputs, with that image's own lists
    b_, c_ = 1, 1
    r1, m1, d1, _, _ = gs.fully_fused_projection_with_ut(_t(means[b_]), _t(quats[b_]), _t(scales[b_]), _t(opac[b_]), _t(vm2[b_, c_:c_ + 1]),
                                                        _t(K2[b_, c_:c_ + 1]), W, H, camera_model=kind,
                                                        **{k: v[b_, c_:c_ + 1] for k, v in co.items()})
    _, i1, f1 = gs.isect_tiles(m1, r1, d1, 16, tw, th)
    o1 = gs.isect_offset_encode(i1, 1, tw, th).reshape(1, th, tw)
    one = gs.rasterize_to_pixels_eval3d(_t(means[b_]), _t(quats[b_]), _t(scales[b_]), colors[b_, c_:c_ + 1], opac_c[b_, c_:c_ + 1],
                                        _t(vm2[b_, c_:c_ + 1]), _t(K2[b_, c_:c_ + 1]), W, H, 16, o1, f1, backgrounds=bg[b_, c_:c_ + 1],
                                        camera_model=kind, **{k: v[b_, c_:c_ + 1] for k, v in co.items()})
    assert torch.equal(one[0][0], a[0][b_, c_]) and torch.equal(one[1][0], a[1][b_, c_])
    # empty lists: the background, no launch
    e = gs.rasterize_to_pixels_eval3d(*args[:10], torch.zeros_like(offs), fl[:0], backgrounds=bg, camera_model=kind, **co)
    assert torch.equal(e[0], bg[..., None, None, :].expand(2, 2, H, W, 3)) and (e[1] == 0).all()


@pytest.mark.parametrize("kind,coeffs", [CAMS[1], CAMS[5]])
def test_end_to_end_chain_on_garden(kind, coeffs):
    sc = scene.make_scene(n_max=60000, sh_degree=0)
    Wf, Hf = 320, 208
    K = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], Wf, Hf)[:2].copy()
    vm = sc["viewmats"][:2].copy()
    leaves = [_t(x).requires_grad_(True) for x in (sc["means"], sc["quats"], sc["scales"])]
    co = _coeffs(coeffs, 2)
    r, m2, d, _, _ = gs.fully_fused_projection_with_ut(*[x.detach() for x in leaves], _t(sc["opacities"]), _t(vm), _t(K),
                                                      Wf, Hf, camera_model=kind, **co)
    tw, th = (Wf + 15) // 16, (Hf + 15) // 16
    _, ii, fl = gs.isect_tiles(m2, r, d, 16, tw, th)
    offs = gs.isect_offset_encode(ii, 2, tw, th)
    colors = _t(np.stack([sc["colors"]] * 2).astype(np.float32)).requires_grad_(True)
    opac = _t(np.stack([sc["opacities"]] * 2)).requires_grad_(True)
    rc, ra = gs.rasterize_to_pixels_eval3d(*leaves, colors, opac, _t(vm), _t(K), Wf, Hf, 16, offs, fl, camera_model=kind, **co)
    assert fl.numel() > 0 and (ra > 0).any()
    (rc.square().sum() + ra.sum()).backward()
    for t in leaves + [colors, opac]:
        assert torch.isfinite(t.grad).all()
    assert torch.isfinite(rc).all() and torch.isfinite(ra).all()


# ---- the kernels against the reference's own outputs (tests/golden/ref_ut.npz, make_ref_ut_golden.py)
import os  # noqa: E402

from tests.test_ut_cpu import REF_CAMERAS, REF_NPZ, ref_case  # noqa: E402


@pytest.mark.parametrize("name", REF_CAMERAS)
def test_kernels_against_reference(name):
    z = np.load(REF_NPZ)
    Wr, Hr = int(z["width"]), int(z["height"])
    model, coeffs = ref_case(z, name)
    co = {KEYS[k]: _t(np.float32([v])) for k, v in coeffs.items()}
    r, m2, d, cn, cp = gs.fully_fused_projection_with_ut(
        _t(z["means"]), _t(z["quats"]), _t(z["scales"]), _t(z["opacities"]), _t(z["viewmats"]), _t(z["Ks"]), Wr, Hr,
        calc_compensations=True, camera_model=model, **co,
    )
    cam = U.Camera(model, z["Ks"][0], Wr, Hr, **coeffs)
    o = U.ut_projection(z["means"], z["quats"], z["scales"], z["opacities"], z["viewmats"][0], cam)
    frac = o["radii_unrounded"].numpy()
    on_edge = (np.abs(frac - np.round(frac)) < 1e-3).any(-1)
    r, rr = r[0].cpu().numpy(), z[f"{name}/radii"][0]
    diff = (r != rr).any(-1)
    # radii are exact except on integer boundaries, where two float32 evaluations may round apart
    assert (diff & ~on_edge).sum() == 0 and diff.sum() <= max(2, len(r) // 100), (diff.sum(), (diff & ~on_edge).sum())
    ok = (r > 0).all(-1) & (rr > 0).all(-1)
    np.testing.assert_allclose(m2[0].cpu().numpy()[ok], z[f"{name}/means2d"][0][ok], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(d[0].cpu().numpy()[ok], z[f"{name}/depths"][0][ok], rtol=1e-5)
    cref = z[f"{name}/conics"][0][ok]
    np.testing.assert_allclose(cn[0].cpu().numpy()[ok], cref, rtol=2e-3, atol=2e-3 * np.abs(cref).max())
    np.testing.assert_allclose(cp[0].cpu().numpy()[ok], z[f"{name}/compensations"][0][ok], rtol=1e-2, atol=1e-4)

    leaves = [_t(z[k]).requires_grad_(True) for k in ("means", "quats", "scales")]
    leaves += [_t(z["colors"][None]).requires_grad_(True), _t(z["opacities"][None]).requires_grad_(True),
               _t(z["backgrounds"]).requires_grad_(True)]
    offs, fl = _t(z[f"{name}/isect_offsets"]), _t(z[f"{name}/flatten_ids"])
    rc, ra = gs.rasterize_to_pixels_eval3d(*leaves[:5], _t(z["viewmats"]), _t(z["Ks"]), Wr, Hr, 16, offs, fl,
                                           backgrounds=leaves[5], camera_model=model, **co)
    ((rc * _t(z["v_render_colors"])).sum() + (ra * _t(z["v_render_alphas"])).sum()).backward()
    # the float64 oracle's margins mark the pixels with a decision near a threshold; only those may differ
    N = len(z["means"])
    f8 = [torch.from_numpy(np.asarray(z[k], np.float64)) for k in ("means", "quats", "scales", "colors", "opacities")]
    _, _, margin = U.eval3d_render(*f8, z["viewmats"][0], cam, offs.cpu(), fl.cpu().tolist(), 1, N, 0,
                                   background=torch.from_numpy(z["backgrounds"][0].astype(np.float64)))
    clear = (margin > 1e-3).numpy()
    err = np.abs(rc[0].detach().cpu().numpy() - z[f"{name}/render_colors"][0]).max(-1)
    aerr = np.abs(ra[0, ..., 0].detach().cpu().numpy() - z[f"{name}/render_alphas"][0][..., 0])
    assert ((err > 2e-4) & clear).sum() == 0 and ((aerr > 2e-4) & clear).sum() == 0, ((err > 2e-4) & clear).sum()
    assert ((err > 2e-4) & ~clear).sum() <= max(4, clear.size // 100)
    for k, leaf in zip(("means", "quats", "scales", "colors", "opacities", "backgrounds"), leaves):
        g, gr = leaf.grad.detach().cpu().numpy().reshape(-1), z[f"{name}/v_{k}"].reshape(-1)
        rel = np.linalg.norm(g - gr) / max(np.linalg.norm(gr), 1e-12)
        assert rel < 2e-2, (k, rel)
