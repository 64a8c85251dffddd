"""rasterize_to_pixels_eval3d_sparse on the GPU.

The sparse result at a requested pixel inside the image is defined as the dense eval3d rendering there, so it is
compared with the dense ops of this library on the same UT rows: the lists of isect_tiles_sparse with
isect_tiles_sorted restricted to the active tiles, the forward bit for bit with rasterize_to_pixels_eval3d gathered at
the in-image pixels, the backward with the dense backward of the same cotangents scattered into zero images, and both
with the float64 oracle (oracle/ut.py).  A requested pixel in the margin of a partial tile has no dense counterpart: it
must come out as the background with alpha 0 and pass no gradient to the gaussians.  Scene: a garden crop at 320 x 200
(the last tile row is half outside the image), one and two cameras and a batch dimension, a distorted pinhole, a
fisheye, an FTheta camera and a rolling shutter; the pixel sets are those of tests/test_sparse_raster_gpu.py.
"""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ut as U
from tests import scene
from tests.test_sparse_raster_gpu import KINDS, TH, TW, H, W, _pixel_set

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_ref_ut_ftheta_golden import ftheta_K  # noqa: E402
from make_ref_ut_rs_golden import end_poses  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CHANNELS = (1, 2, 3, 4, 5, 8, 16, 32)
# layouts of the images: (batch B, cameras C); the images are the B * C flattened (b, c)
LAYOUTS = {"1cam": (0, 1), "2cam": (0, 2), "batch": (2, 2)}
# camera: (camera_model, coefficients, FTheta calibration, rolling shutter)
CAMS = {
    "pinhole": ("pinhole", dict(radial=[0.08, -0.03, 0.005, 0.01, 0.0, 0.0], tangential=[0.004, -0.003],
                                thin=[0.002, -0.001, 0.001, 0.0005]), None, False),
    "fisheye": ("fisheye", dict(radial=[0.04, -0.01, 0.002, -0.0003]), None, False),
    # the forward polynomial as the reference: pixels whose Newton inversion does not converge composite nothing
    "ftheta": ("ftheta", {}, "cross_left_120fov", False),
    "rolling": ("pinhole", dict(radial=[0.08, -0.03, 0.005, 0.01, 0.0, 0.0], tangential=[0.004, -0.003]), None, True),
}
KEYS = {"radial": "radial_coeffs", "tangential": "tangential_coeffs", "thin": "thin_prism_coeffs"}
GRADS = ("means", "quats", "scales", "colors", "opacities")


@pytest.fixture(scope="module")
def gs():
    import gsplat_b200

    assert torch.cuda.is_available(), "needs a GPU"
    return gsplat_b200


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _camera(gs, cam, lead, vm, Ks, width, height):
    """(Ks, the camera keyword arguments of both ops, a description for the float64 oracle of image 0)."""
    model, coeffs, cal, rolling = CAMS[cam]
    C = lead[-1]
    kw = dict(camera_model=model)
    for k, v in coeffs.items():
        kw[KEYS[k]] = _t(np.broadcast_to(np.float32(v), lead + (len(v),)))
    ftheta = None
    if cal is not None:
        params, pp, _ = scene.scaled(scene.calibrations()[cal], width)
        ftheta = dict(params, reference_poly=1)
        kw["ftheta_coeffs"] = gs.FThetaCameraDistortionParameters(**ftheta)
        Ks = np.broadcast_to(ftheta_K((pp[0] - 0.5, pp[1] - 0.5), C), lead + (3, 3)).copy()
    vm_rs = None
    if rolling:
        vm_rs = end_poses(vm.reshape(-1, 4, 4)).reshape(vm.shape).astype(np.float32)
        kw.update(rolling_shutter=gs.RollingShutterType.ROLLING_TOP_TO_BOTTOM, viewmats_rs=_t(vm_rs))
    return Ks, kw, (model, coeffs, ftheta, vm_rs)


def _rows(gs, B, C, D, cam="pinhole", n=20000, seed=0):
    """The UT rows of a garden crop seen by C cameras (and B batch entries), D random colour channels."""
    sc = scene.make_scene(n_max=n, sh_degree=0, seed=42 + seed)
    lead = (B, C) if B else (C,)
    vm = sc["viewmats"][:C].astype(np.float32)
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:C].astype(np.float32)
    means, quats, scales = sc["means"], sc["quats"], sc["scales"]
    if B:
        rng = np.random.RandomState(seed)
        means = means[None] + (rng.standard_normal((B,) + means.shape) * 0.01).astype(np.float32) * (np.arange(B) > 0)[:, None, None]
        quats, scales = np.broadcast_to(quats, (B,) + quats.shape), np.broadcast_to(scales, (B,) + scales.shape)
        vm, Ks = np.broadcast_to(vm, (B,) + vm.shape).copy(), np.broadcast_to(Ks, (B,) + Ks.shape).copy()
    Ks, kw, _ = _camera(gs, cam, lead, vm, Ks, W, H)
    means, quats, scales, vm, Ks = (_t(np.asarray(x, np.float32)) for x in (means, quats, scales, vm, Ks))
    op = _t(np.broadcast_to(sc["opacities"], lead[:-1] + sc["opacities"].shape))
    with torch.no_grad():
        radii, m2, dep, _, _ = gs.fully_fused_projection_with_ut(means, quats, scales, op, vm, Ks, W, H, **kw)
    N = means.shape[-2]
    g = torch.Generator(device=DEV).manual_seed(seed)
    colors = torch.rand(lead + (N, D), device=DEV, generator=g)
    opac = torch.broadcast_to(op[..., None, :], lead + (N,)).contiguous()
    return dict(means=means, quats=quats, scales=scales, colors=colors, opacities=opac, viewmats=vm, Ks=Ks, kw=kw,
                radii=radii, means2d=m2, depths=dep, lead=lead)


def _n_images(rows):
    return int(np.prod(rows["lead"]))


def _dense_lists(gs, rows):
    hits = gs.ops.isect_tiles_sorted(rows["means2d"], rows["radii"], rows["depths"], 16, TW, TH)
    return hits.isect_offsets.reshape(rows["lead"] + (TH, TW)), hits.flatten_ids


def _sparse_pipeline(gs, rows, pixels, image_ids):
    I, N = _n_images(rows), rows["means"].shape[-2]
    layout = gs.build_sparse_tile_layout(pixels, image_ids, I, 16, TW, TH)
    tile_offsets, flatten_ids = gs.isect_tiles_sparse(
        rows["means2d"].reshape(I, N, 2), rows["radii"].reshape(I, N, 2), rows["depths"].reshape(I, N), layout[1],
        layout[0], I, 16, TW, TH,
    )
    return layout, tile_offsets, flatten_ids


def _render_both(gs, rows, pixels, image_ids, bg=None, masks=None, seed=0, cots=None):
    """Sparse and dense forward + backward with the same random cotangents (the dense side gets those of the in-image
    pixels, scattered into zero images).  Returns ({mode: (outputs, gradients)}, inside [P] bool, cotangents, lists);
    gradients are v_means, v_quats, v_scales, v_colors, v_opacities, then v_backgrounds where present."""
    lead, D = rows["lead"], rows["colors"].shape[-1]
    layout, tile_offsets, flatten_ids = _sparse_pipeline(gs, rows, pixels, image_ids)
    offsets, fl = _dense_lists(gs, rows)
    P = pixels.shape[0]
    if cots is None:
        g = torch.Generator(device=DEV).manual_seed(seed + 1)
        cots = [torch.randn((P, k), device=DEV, generator=g) for k in (D, 1)]
    p, ids = pixels.long(), image_ids.long()
    inside = p[:, 0] < H
    out = {}
    for mode in ("sparse", "dense"):
        ins = [rows[k].detach().clone().requires_grad_(True) for k in GRADS]
        tbg = bg.detach().clone().requires_grad_(True) if bg is not None else None
        if mode == "sparse":
            active, _, words, cumsum, pmap = layout
            outs = gs.rasterize_to_pixels_eval3d_sparse(
                *ins, rows["viewmats"], rows["Ks"], image_ids, active, tile_offsets, flatten_ids, words, cumsum, pmap, W,
                H, 16, TW, TH, backgrounds=tbg, masks=masks, **rows["kw"],
            )
            loss = sum((o * c).sum() for o, c in zip(outs, cots))
        else:
            dbg = tbg.reshape(lead + (D,)) if tbg is not None else None
            dm = masks.reshape(lead + (TH, TW)) if masks is not None else None
            imgs = gs.rasterize_to_pixels_eval3d(*ins, rows["viewmats"], rows["Ks"], W, H, 16, offsets, fl, backgrounds=dbg,
                                                 masks=dm, **rows["kw"])
            flat = [x.reshape((-1, H, W, x.shape[-1])) for x in imgs]
            outs = [torch.zeros((P, x.shape[-1]), device=DEV) for x in flat]
            loss = 0.0
            for o, x, c in zip(outs, flat, cots):
                o[inside] = x[ids[inside], p[inside, 0], p[inside, 1]].detach()
                v = torch.zeros_like(x)
                v[ids[inside], p[inside, 0], p[inside, 1]] = c[inside]
                loss = loss + (x * v).sum()
        targets = ins + ([tbg] if tbg is not None else [])
        grads = list(torch.autograd.grad(loss, targets, allow_unused=True)) if P > 0 else [None] * len(targets)
        grads = [torch.zeros_like(x) if gr is None else gr for x, gr in zip(targets, grads)]
        out[mode] = ([o.detach() for o in outs], grads)
    return out, inside, cots, (layout, tile_offsets, flatten_ids, offsets, fl)


def _rel(a, b):
    nb = torch.linalg.norm(b.double())
    return float(torch.linalg.norm(a.double() - b.double()) / max(float(nb), 1e-30))


def _check_equal_to_dense(out, inside, image_ids, cots, bg=None):
    (so, sg), (do, dg) = out["sparse"], out["dense"]
    # in-image pixels: bit for bit; margin pixels: the background (or 0) and alpha 0
    for name, a, b in zip(("colors", "alphas"), so, do):
        assert torch.equal(a[inside], b[inside]), name
    rc, ra = so
    margin = ~inside
    want = bg[image_ids.long()[margin]] if bg is not None else torch.zeros_like(rc[margin])
    assert torch.equal(rc[margin], want) and torch.equal(ra[margin], torch.zeros_like(ra[margin]))
    assert len(sg) == len(dg)
    for i, (a, b) in enumerate(zip(sg, dg)):
        if i == 5:
            # v_backgrounds: the margin pixels show the background, so their colour cotangents reach it, which the dense
            # image (it has no such pixels) cannot give; a float32 sum in another order than the dense one: 1e-5, as in
            # tests/test_sparse_2dgs_gpu.py
            b = b.clone().index_add_(0, image_ids.long()[margin], cots[0][margin])
            tol = 1e-5
        else:
            tol = 1e-6
        assert _rel(a, b) <= tol, f"gradient {i}: rel-L2 {_rel(a, b):.3e}"


@pytest.mark.parametrize("cam", list(CAMS))
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("kind", KINDS)
def test_lists_match_dense(gs, kind, layout, cam):
    B, C = LAYOUTS[layout]
    rows = _rows(gs, B, C, 3, cam)
    I = _n_images(rows)
    pixels, image_ids = _pixel_set(kind, I, np.random.RandomState(10 * KINDS.index(kind) + I))
    (active, *_), tile_offsets, flatten_ids = _sparse_pipeline(gs, rows, pixels, image_ids)
    offsets, fl = _dense_lists(gs, rows)
    off = np.concatenate([offsets.cpu().numpy().reshape(-1), [fl.shape[0]]])
    fl = fl.cpu().numpy()
    exp_ids = [fl[off[t] : off[t + 1]] for t in active.cpu().numpy()]
    exp_off = np.concatenate([[0], np.cumsum([len(x) for x in exp_ids])]).astype(np.int32)
    assert np.array_equal(tile_offsets.cpu().numpy(), exp_off)
    exp_fl = np.concatenate(exp_ids) if exp_ids else np.zeros(0, np.int32)
    assert np.array_equal(flatten_ids.cpu().numpy(), exp_fl)
    if kind not in ("empty", "one"):
        assert flatten_ids.numel() > 1000


@pytest.mark.parametrize("cam", list(CAMS))
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("kind", KINDS)
def test_matches_dense(gs, kind, layout, cam):
    B, C = LAYOUTS[layout]
    rows = _rows(gs, B, C, 3, cam)
    I = _n_images(rows)
    pixels, image_ids = _pixel_set(kind, I, np.random.RandomState(100 + 10 * KINDS.index(kind) + I))
    out, inside, cots, _ = _render_both(gs, rows, pixels, image_ids, seed=KINDS.index(kind))
    P = pixels.shape[0]
    assert [tuple(o.shape) for o in out["sparse"][0]] == [(P, 3), (P, 1)]
    if kind in ("random", "patches", "all"):
        assert (out["sparse"][0][1] > 0).any()
    _check_equal_to_dense(out, inside, image_ids, cots)


@pytest.mark.parametrize("cam", list(CAMS))
def test_margin_pixels_pass_no_gradient(gs, cam):
    """Cotangents on the margin pixels alone: every gaussian gradient is exactly zero; the background's is their sum."""
    rows = _rows(gs, 0, 2, 3, cam)
    pixels, image_ids = _pixel_set("margin", 2, np.random.RandomState(11))
    inside = (pixels[:, 0] < H)[:, None]
    assert inside.any() and not inside.all()
    g = torch.Generator(device=DEV).manual_seed(12)
    # Cotangents on a 2^-10 grid within [-8, 8]: an image's 856 margin pixels then sum below 2^14, so every partial sum
    # is a float32 and the background's gradient is exact in whatever order index_add_'s atomics add it up.
    cots = [
        (torch.randn((pixels.shape[0], k), device=DEV, generator=g) * 1024).round().clamp(-8192, 8192) / 1024 * ~inside
        for k in (3, 1)
    ]
    bg = torch.rand((2, 3), device=DEV, generator=g)
    out, inside, _, _ = _render_both(gs, rows, pixels, image_ids, bg=bg, cots=cots)
    (rc, ra), grads = out["sparse"]
    assert torch.equal(rc[~inside], bg[image_ids.long()[~inside]]) and (ra[~inside] == 0).all()
    for i, x in enumerate(grads[:5]):
        assert torch.equal(x, torch.zeros_like(x)), GRADS[i]
    want = torch.zeros_like(bg).index_add_(0, image_ids.long(), cots[0])
    assert torch.equal(grads[5], want)


@pytest.mark.parametrize("D", CHANNELS)
@pytest.mark.parametrize("extras", ["plain", "bg+masks"])
def test_channels_backgrounds_masks(gs, D, extras):
    rows = _rows(gs, 0, 2, D, seed=D)
    pixels, image_ids = _pixel_set("patches", 2, np.random.RandomState(D))
    bg = masks = None
    if extras != "plain":
        bg = torch.rand((2, D), device=DEV, generator=torch.Generator(device=DEV).manual_seed(D))
        masks = torch.from_numpy(np.random.RandomState(3).random_sample((2, TH, TW)) > 0.3).to(DEV)
    out, inside, cots, (layout, *_rest) = _render_both(gs, rows, pixels, image_ids, bg=bg, masks=masks, seed=D)
    if masks is not None:  # some requested tiles are masked off: they show the background
        assert not masks.reshape(-1)[layout[0].long()].all()
    _check_equal_to_dense(out, inside, image_ids, cots, bg)
    assert len(out["sparse"][1]) == 5 + (bg is not None)


@pytest.mark.parametrize("cam", list(CAMS))
def test_cameras_backgrounds_masks(gs, cam):
    rows = _rows(gs, 2, 2, 4, cam, seed=5)
    pixels, image_ids = _pixel_set("margin", 4, np.random.RandomState(6))
    bg = torch.rand((4, 4), device=DEV, generator=torch.Generator(device=DEV).manual_seed(6))
    masks = torch.from_numpy(np.random.RandomState(7).random_sample((4, TH, TW)) > 0.3).to(DEV)
    out, inside, cots, _ = _render_both(gs, rows, pixels, image_ids, bg=bg, masks=masks, seed=6)
    _check_equal_to_dense(out, inside, image_ids, cots, bg)


def test_active_tile_with_empty_list(gs):
    """A requested tile no gaussian reaches renders the background and has an empty range."""
    rows = _rows(gs, 0, 1, 3)
    t = 5 * TW + 7  # tile (7, 5): drop every gaussian whose box reaches it
    offsets, fl = _dense_lists(gs, rows)
    off = np.concatenate([offsets.cpu().numpy().reshape(-1), [fl.shape[0]]])
    hit = torch.from_numpy(fl.cpu().numpy()[off[t] : off[t + 1]].astype(np.int64)).to(DEV)
    assert hit.numel() > 0
    radii = rows["radii"].clone()
    radii.view(-1, 2)[hit] = 0
    rows = dict(rows, radii=radii)
    pixels = torch.tensor([[5 * 16 + 3, 7 * 16 + 9], [5 * 16 + 15, 7 * 16], [10, 10]], device=DEV, dtype=torch.int32)
    image_ids = torch.zeros(3, device=DEV, dtype=torch.int32)
    bg = torch.tensor([[0.25, 0.5, 0.75]], device=DEV)
    out, inside, cots, (layout, tile_offsets, *_rest) = _render_both(gs, rows, pixels, image_ids, bg=bg)
    a = int(np.nonzero(layout[0].cpu().numpy() == t)[0][0])
    assert tile_offsets[a] == tile_offsets[a + 1]
    rc, ra = out["sparse"][0]
    assert torch.equal(rc[:2], bg.expand(2, 3)) and torch.equal(ra[:2], torch.zeros_like(ra[:2]))
    _check_equal_to_dense(out, inside, image_ids, cots, bg)


def test_no_lists_at_all(gs):
    """Nothing listed in any active tile: the background at every requested pixel, zero gradients but v_backgrounds."""
    rows = _rows(gs, 0, 2, 3, n=2000)
    rows = dict(rows, radii=torch.zeros_like(rows["radii"]))
    pixels, image_ids = _pixel_set("margin", 2, np.random.RandomState(4))
    bg = torch.rand((2, 3), device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    out, inside, cots, (_, _, flatten_ids, *_rest) = _render_both(gs, rows, pixels, image_ids, bg=bg)
    assert flatten_ids.numel() == 0
    (rc, ra), grads = out["sparse"]
    assert torch.equal(rc, bg[image_ids.long()]) and torch.equal(ra, torch.zeros_like(ra))
    for x, like in zip(grads[:5], (rows[k] for k in GRADS)):
        assert x.shape == like.shape and torch.equal(x, torch.zeros_like(x))
    _check_equal_to_dense(out, inside, image_ids, cots, bg)


def test_no_pixels(gs):
    rows = _rows(gs, 0, 1, 3, n=2000)
    pixels, image_ids = _pixel_set("empty", 1, np.random.RandomState(0))
    (active, _, words, cumsum, pmap), tile_offsets, flatten_ids = _sparse_pipeline(gs, rows, pixels, image_ids)
    ins = [rows[k].detach().clone().requires_grad_(True) for k in GRADS]
    bg = torch.ones((1, 3), device=DEV, requires_grad=True)
    rc, ra = gs.rasterize_to_pixels_eval3d_sparse(
        *ins, rows["viewmats"], rows["Ks"], image_ids, active, tile_offsets, flatten_ids, words, cumsum, pmap, W, H, 16,
        TW, TH, backgrounds=bg, **rows["kw"],
    )
    assert tuple(rc.shape) == (0, 3) and tuple(ra.shape) == (0, 1)
    (rc.sum() + ra.sum()).backward()
    for x in ins + [bg]:
        assert x.grad.shape == x.shape and torch.equal(x.grad, torch.zeros_like(x))


def test_forward_deterministic(gs):
    rows = _rows(gs, 0, 2, 4, "rolling")
    pixels, image_ids = _pixel_set("random", 2, np.random.RandomState(7))
    (active, _, words, cumsum, pmap), tile_offsets, flatten_ids = _sparse_pipeline(gs, rows, pixels, image_ids)

    def run():
        return gs.rasterize_to_pixels_eval3d_sparse(
            *(rows[k] for k in GRADS), rows["viewmats"], rows["Ks"], image_ids, active, tile_offsets, flatten_ids, words,
            cumsum, pmap, W, H, 16, TW, TH, **rows["kw"],
        )

    for x, y in zip(run(), run()):
        assert torch.equal(x, y)


# ---- against the float64 oracle, on the small scene of tests/test_ut_gpu.py
WS, HS = 96, 64


@pytest.mark.parametrize("cam", list(CAMS))
def test_against_float64_oracle(gs, cam):
    """Forward and gradients at a quarter of the pixels against oracle/ut.py's eval3d_render on the same lists, with the
    margin-based tolerances of tests/test_ut_gpu.py (pixels with a decision near a threshold are counted and bounded)."""
    sc = scene.make_scene(n_max=400, sh_degree=0, seed=0)
    vm = sc["viewmats"][:1].astype(np.float32)
    K = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], WS, HS)[:1].astype(np.float32)
    K, kw, (model, coeffs, ftheta, vm_rs) = _camera(gs, cam, (1,), vm, K, WS, HS)
    s = (sc["scales"] * 4.0).astype(np.float32)
    N = len(s)
    with torch.no_grad():
        r, m2, d, _, _ = gs.fully_fused_projection_with_ut(_t(sc["means"]), _t(sc["quats"]), _t(s), _t(sc["opacities"]),
                                                          _t(vm), _t(K), WS, HS, **kw)
    tw, th = WS // 16, HS // 16
    hits = gs.ops.isect_tiles_sorted(m2, r, d, 16, tw, th)
    offs, fl = hits.isect_offsets.reshape(1, th, tw), hits.flatten_ids
    assert fl.numel() > 50
    rng = np.random.RandomState(1)
    flat = np.sort(rng.choice(WS * HS, WS * HS // 4, replace=False))
    px = np.stack([flat // WS, flat % WS], -1)
    pixels, image_ids = _t(px.astype(np.int32)), torch.zeros(len(px), device=DEV, dtype=torch.int32)
    active, amask, words, cumsum, pmap = gs.build_sparse_tile_layout(pixels, image_ids, 1, 16, tw, th)
    toff, sfl = gs.isect_tiles_sparse(m2, r, d, amask, active, 1, 16, tw, th)
    bg = rng.random_sample((1, 3)).astype(np.float32)
    colors, opac = sc["colors"][None].astype(np.float32), sc["opacities"][None].astype(np.float32)
    leaves = [_t(x).requires_grad_(True) for x in (sc["means"], sc["quats"], s, colors, opac, bg)]
    rc, ra = gs.rasterize_to_pixels_eval3d_sparse(
        *leaves[:5], _t(vm), _t(K), image_ids, active, toff, sfl, words, cumsum, pmap, WS, HS, 16, tw, th,
        backgrounds=leaves[5], **kw,
    )
    v_rc = rng.standard_normal(rc.shape).astype(np.float32)
    v_ra = rng.standard_normal(ra.shape).astype(np.float32)
    ((rc * _t(v_rc)).sum() + (ra * _t(v_ra)).sum()).backward()

    if ftheta is not None:
        ocam = U.FThetaCamera(ftheta, K[0], WS, HS)
    else:
        ocam = U.Camera(model, K[0], WS, HS, **coeffs)
    pose = vm[0] if vm_rs is None else U.ShutterPoses(vm[0], vm_rs[0], 0)
    f8 = [torch.from_numpy(np.asarray(x, np.float64)).requires_grad_(True) for x in (sc["means"], sc["quats"], s, colors[0], opac[0], bg[0])]
    oc, oa, margin = U.eval3d_render(*f8[:5], pose, ocam, offs.cpu(), fl.cpu().tolist(), 1, N, 0, background=f8[5])
    sel = (torch.from_numpy(px[:, 0]), torch.from_numpy(px[:, 1]))
    ((oc[sel] * torch.from_numpy(v_rc.astype(np.float64))).sum() + (oa[sel] * torch.from_numpy(v_ra.astype(np.float64))).sum()).backward()
    clear = (margin[sel] > 1e-3).numpy()
    if ftheta is not None:  # a Newton step near the 1e-6 convergence threshold may converge in one precision only
        step = ocam.last_step.reshape(HS, WS).numpy()[px[:, 0], px[:, 1]]
        clear &= ~((step > 1e-7) & (step < 1e-5))
    err = np.abs(rc.detach().cpu().numpy() - oc[sel].detach().numpy()).max(-1)
    bad = err > 2e-4
    assert (bad & clear).sum() <= max(1, clear.size // 1000), (bad & clear).sum()
    assert (bad & ~clear).sum() <= max(8, clear.size // 50), (bad & ~clear).sum()
    aerr = np.abs(ra[:, 0].detach().cpu().numpy() - oa[sel][:, 0].detach().numpy())
    assert ((aerr > 2e-4) & clear).sum() <= max(1, clear.size // 1000)
    assert (ra > 0).any()
    for name, a, b in zip(GRADS + ("backgrounds",), leaves, f8):
        g, gr = a.grad.detach().cpu().numpy().reshape(-1), b.grad.numpy().reshape(-1)
        rel = np.linalg.norm(g - gr) / max(np.linalg.norm(gr), 1e-12)
        assert rel < 2e-2, (name, rel)
