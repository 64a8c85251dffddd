"""2DGS on the H100 against the float64 oracle (oracle/surfel.py), on garden crops from tests/scene.py.

* projection: radii exact except counted ceil / screen-edge flips; floats and every gradient by relative L2;
* compositing: colours, alphas, normals, distortion, median depth at rtol 1e-4 / atol 1e-5 on the pixels whose
  threshold decisions (alpha, stop, median, parallel ray) are not marginal, a bounded share of marginal pixels,
  last_ids / median_ids exact there; every gradient, v_densify and absgrad included, by relative L2;
* rasterization_2dgs: render modes x distloss x depth_mode, backgrounds, masks, edge tiles, C = 2, a batch dimension,
  channel counts, SH and precomputed colours, viewmats.requires_grad, the empty scene, ~30k gaussians end to end, and
  bit-identical forward outputs of two runs.

The compositing oracle always runs on the tile lists of the GPU intersection (the radius box), so that a radius flip
only moves which tiles list a gaussian whose alpha there is below the threshold anyway.
"""
import math

import numpy as np
import pytest
import torch

from oracle import surfel
from tests import scene

pytestmark = pytest.mark.gpu
dev = "cuda"
f64 = torch.float64
REL_PROJ = 2e-4  # floats / gradients of the projection (tests/test_gpu_parity.py: 2e-4 pinhole, 1e-3 v_viewmats)
REL_GRAD = 1e-3  # compositing gradients (tests/test_gpu_parity.py: 1e-3)
# v_ray_transforms: h_u = px * M2 - M0 cancels (both terms grow with the pixel coordinate), so its float32 value carries
# a relative error a few times larger than the other gradients'
REL_RT = 5e-3
REL_VIEWMATS = 3e-3  # v_viewmats through rasterization_2dgs also collects the depth-normal and world-normal rotations


@pytest.fixture(scope="module")
def gs():
    import gsplat_b200

    return gsplat_b200


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    nb = np.linalg.norm(b)
    return np.linalg.norm(a - b) / max(nb, 1e-30)


def _n(t):
    return t.detach().cpu().double().numpy()


def _scene(n, W, H, C=1, B=0, seed=0, scale_mul=2.0):
    sc = scene.make_scene(n_max=n, sh_degree=1, seed=42 + seed)
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:C]
    vm = sc["viewmats"][:C]
    d = dict(means=sc["means"], quats=sc["quats"], scales=sc["scales"] * scale_mul, opacities=sc["opacities"], sh=sc["sh"],
             colors=sc["colors"], viewmats=vm, Ks=Ks)
    if B:
        rng = np.random.RandomState(seed)
        d = {k: np.stack([v] + [v + (rng.standard_normal(v.shape) * 0.01 if k == "means" else 0) for _ in range(B - 1)]).astype(np.float32)
             if k not in ("sh",) else v for k, v in d.items()}
    return d


# ------------------------------------------------------------------ projection
@pytest.mark.parametrize("C,B,vm_grad,clip", [(1, 0, False, 0.0), (2, 0, True, 0.0), (2, 2, True, 0.0), (1, 0, False, 3.0)])
def test_projection_vs_oracle(gs, C, B, vm_grad, clip):
    W, H = 256, 168
    d = _scene(3000, W, H, C=C, B=B)
    t = {k: torch.tensor(d[k], device=dev).requires_grad_(True) for k in ("means", "quats", "scales", "viewmats")}
    t["viewmats"].requires_grad_(vm_grad)
    Ks = torch.tensor(d["Ks"], device=dev)
    radii, m2, dep, rt, nrm = gs.fully_fused_projection_2dgs(t["means"], t["quats"], t["scales"], t["viewmats"], Ks, W, H, radius_clip=clip)
    o = {k: torch.tensor(d[k], dtype=f64).requires_grad_(True) for k in ("means", "quats", "scales", "viewmats")}
    oK = torch.tensor(d["Ks"], dtype=f64)
    orad, om2, odep, ort, onrm = surfel.project(o["means"], o["quats"], o["scales"], o["viewmats"], oK, W, H, radius_clip=clip)
    ceil_m, screen_m, _ = surfel.project_margins(o["means"].detach(), o["quats"].detach(), o["scales"].detach(), o["viewmats"].detach(), oK, W, H)
    marginal = (ceil_m < 4.0) | (screen_m < 5e-2)
    gr, orr = radii.cpu().numpy(), orad.numpy()
    diff = (gr != orr).any(-1)
    assert not (diff & ~marginal.numpy()).any(), f"{int((diff & ~marginal.numpy()).sum())} radii differ away from a ceil / edge boundary"
    assert diff.mean() < 5e-3, f"{diff.sum()} ceil-boundary flips"
    both = ((gr > 0).all(-1) & (orr > 0).all(-1))
    assert both.sum() > 100
    for name, a, b in (("means2d", m2, om2), ("depths", dep, odep), ("ray_transforms", rt, ort), ("normals", nrm, onrm)):
        rel = _rel(_n(a)[both], _n(b)[both])
        assert rel < REL_PROJ, f"{name}: rel L2 {rel:.3e}"
    # culled rows: zero floats
    culled = (gr == 0).all(-1)
    assert (_n(m2)[culled] == 0).all() and (_n(rt)[culled] == 0).all()
    rng = np.random.RandomState(1)
    mask = torch.tensor(both)
    cots = [torch.tensor(rng.standard_normal(x.shape)) * mask.reshape(mask.shape + (1,) * (x.dim() - mask.dim())) for x in (m2, dep, rt, nrm)]
    loss = sum((a * c.float().to(dev)).sum() for a, c in zip((m2, dep, rt, nrm), cots))
    keys = ["means", "quats", "scales"] + (["viewmats"] if vm_grad else [])
    g = torch.autograd.grad(loss, [t[k] for k in keys])
    og = torch.autograd.grad(sum((a * c).sum() for a, c in zip((om2, odep, ort, onrm), cots)), [o[k] for k in keys])
    for k, a, b in zip(keys, g, og):
        rel = _rel(_n(a), _n(b))
        assert rel < (1e-3 if k == "viewmats" else REL_PROJ), f"v_{k}: rel L2 {rel:.3e}"
    assert (_n(g[2])[..., 2] == 0).all()


# ------------------------------------------------------------------ compositing
def _raster_inputs(gs, n, W, H, D, C=1, B=0, seed=0):
    d = _scene(n, W, H, C=C, B=B, seed=seed)
    with torch.no_grad():
        radii, m2, dep, rt, nrm = gs.fully_fused_projection_2dgs(
            *(torch.tensor(d[k], device=dev) for k in ("means", "quats", "scales", "viewmats", "Ks")), W, H
        )
    rng = np.random.RandomState(seed)
    lead = tuple(m2.shape[:-1])
    col = torch.tensor(rng.random_sample(lead + (D,)).astype(np.float32), device=dev)
    col[..., -1] = dep  # the depth channel
    op = torch.broadcast_to(torch.tensor(d["opacities"], device=dev)[..., None, :], lead).contiguous()
    th, tw = math.ceil(H / 16), math.ceil(W / 16)
    hits = gs.ops.isect_tiles_sorted(m2, radii, dep, 16, tw, th)
    off = hits.isect_offsets.reshape(lead[:-1] + (th, tw))
    return dict(means2d=m2, ray_transforms=rt, colors=col, opacities=op, normals=nrm, isect_offsets=off, flatten_ids=hits.flatten_ids)


def _raster_case(gs, inp, W, H, bg=None, masks=None, absgrad=False, seed=0, cot_keys=(0, 1, 2, 3, 4), max_marginal=0.02):
    lead = tuple(inp["means2d"].shape[:-1])
    leaves = {k: inp[k].clone().requires_grad_(True) for k in ("means2d", "ray_transforms", "colors", "opacities", "normals")}
    densify = torch.zeros(lead + (2,), device=dev, requires_grad=True)
    outs = gs.rasterize_to_pixels_2dgs(
        leaves["means2d"], leaves["ray_transforms"], leaves["colors"], leaves["opacities"], leaves["normals"], densify, W, H, 16,
        inp["isect_offsets"], inp["flatten_ids"], backgrounds=bg, masks=masks, absgrad=absgrad,
    )
    rng = np.random.RandomState(seed + 7)
    cots = [torch.tensor(rng.standard_normal(o.shape).astype(np.float32), device=dev) if i in cot_keys else None for i, o in enumerate(outs)]
    loss = sum((o * c).sum() for o, c in zip(outs, cots) if c is not None)
    keys = ("means2d", "ray_transforms", "colors", "opacities", "normals")
    g = dict(zip(keys, torch.autograd.grad(loss, [leaves[k] for k in keys] + [densify], retain_graph=False)[:5]))
    # densify: a second backward so that .grad is filled the way a strategy reads it
    outs2 = gs.rasterize_to_pixels_2dgs(
        leaves["means2d"], leaves["ray_transforms"], leaves["colors"], leaves["opacities"], leaves["normals"], densify, W, H, 16,
        inp["isect_offsets"], inp["flatten_ids"], backgrounds=bg, masks=masks, absgrad=absgrad,
    )
    sum((o * c).sum() for o, c in zip(outs2, cots) if c is not None).backward()
    torch.cuda.synchronize()
    o64 = {k: inp[k].detach().cpu().double() for k in keys}
    ref = surfel.rasterize_vjp(
        o64["means2d"], o64["ray_transforms"], o64["colors"], o64["opacities"], o64["normals"], W, H, 16,
        inp["isect_offsets"].cpu().numpy(), inp["flatten_ids"].cpu().numpy(), [None if c is None else c.cpu().double() for c in cots],
        backgrounds=None if bg is None else bg.cpu().double(), masks=None if masks is None else masks.cpu().numpy(),
    )
    ok = ref["margins"] > 1e-3
    assert (~ok).mean() < max_marginal, f"{(~ok).mean() * 100:.2f}% marginal pixels"
    for name, o in zip(surfel._OUT_NAMES, outs):
        a, b = _n(o)[ok], ref[name].numpy()[ok]
        bad = np.abs(a - b) > 1e-4 * np.abs(b) + 1e-5
        assert bad.mean() < 1e-3, f"{name}: {bad.mean() * 100:.3f}% of non-marginal pixels out of tolerance, max err {np.abs(a - b).max():.2e}"
    for k in keys:
        rel = _rel(_n(g[k]), ref["v_" + k].numpy())
        assert rel < (REL_RT if k == "ray_transforms" else REL_GRAD), f"v_{k}: rel L2 {rel:.3e}"
    rel = _rel(_n(densify.grad), ref["v_densify"].numpy())
    assert rel < REL_RT, f"v_densify: rel L2 {rel:.3e}"  # a column of v_ray_transforms, scaled
    if absgrad:
        rel = _rel(_n(leaves["means2d"].absgrad), ref["absgrad"].numpy())
        assert rel < REL_GRAD, f"absgrad: rel L2 {rel:.3e}"
    return outs, ref, ok


@pytest.mark.parametrize("D", [1, 3, 4, 32])
def test_compositing_channels(gs, D):
    W, H = 200, 136  # edge tiles: neither is a multiple of 16
    inp = _raster_inputs(gs, 6000, W, H, D)
    outs, ref, ok = _raster_case(gs, inp, W, H)
    # render side outputs held by the op for its backward: last / median ids exact away from marginal pixels
    assert inp["flatten_ids"].numel() > 1000


def test_compositing_ids_exact(gs):
    W, H = 160, 112
    inp = _raster_inputs(gs, 4000, W, H, 4)
    lib = gs._cabi.lib()
    from gsplat_b200._cabi import ptr, stream

    I = 1
    th, tw = inp["isect_offsets"].shape[-2:]
    o = lambda *s, dt=torch.float32: torch.empty(s, device=dev, dtype=dt)  # noqa: E731
    rc, ra, rn, rd, rm = o(1, H, W, 4), o(1, H, W, 1), o(1, H, W, 3), o(1, H, W, 1), o(1, H, W, 1)
    li, mi = o(1, H, W, dt=torch.int32), o(1, H, W, dt=torch.int32)
    fl = inp["flatten_ids"]
    rc_ = lib.gsb200_surfel_raster_fwd(
        I, inp["means2d"].shape[-2], 4, ptr(inp["means2d"]), ptr(inp["ray_transforms"]), ptr(inp["colors"]), ptr(inp["opacities"]),
        ptr(inp["normals"]), None, None, W, H, 16, tw, th, ptr(inp["isect_offsets"]), ptr(fl), fl.numel(), ptr(rc), ptr(ra), ptr(rn),
        ptr(rd), ptr(rm), ptr(li), ptr(mi), stream(),
    )
    assert rc_ == 0
    torch.cuda.synchronize()
    ref = surfel.rasterize(*(inp[k].cpu().double() for k in ("means2d", "ray_transforms", "colors", "opacities", "normals")), W, H, 16,
                           inp["isect_offsets"].cpu().numpy(), fl.cpu().numpy())
    ok = ref["margins"] > 1e-3
    np.testing.assert_array_equal(li.cpu().numpy()[ok], ref["last_ids"][ok])
    np.testing.assert_array_equal(mi.cpu().numpy()[ok], ref["median_ids"][ok])


def test_compositing_backgrounds_masks_absgrad(gs):
    W, H = 184, 120
    inp = _raster_inputs(gs, 5000, W, H, 4, C=2)
    rng = np.random.RandomState(3)
    bg = torch.tensor(rng.random_sample((2, 4)).astype(np.float32), device=dev)
    th, tw = inp["isect_offsets"].shape[-2:]
    masks = torch.tensor(rng.random_sample((2, th, tw)) > 0.3, device=dev)
    _raster_case(gs, inp, W, H, bg=bg, masks=masks, absgrad=True)


def test_compositing_batch_dims(gs):
    W, H = 128, 96
    inp = _raster_inputs(gs, 3000, W, H, 3, C=2, B=2)
    assert inp["means2d"].dim() == 4
    _raster_case(gs, inp, W, H, absgrad=True)


# ------------------------------------------------------------------ rasterization_2dgs against the oracle chain
def _oracle_chain(d, W, H, fl, off, render_mode, depth_mode, bg, colors_f64, cots):
    """Float64 forward and gradients of rasterization_2dgs on the GPU's tile lists.  colors_f64 are post-activation
    colours [..., N, D] (None for depth-only modes).  Returns outputs and the gradients of sum(out * cot)."""
    leaves = {k: torch.tensor(d[k], dtype=f64, requires_grad=True) for k in ("means", "quats", "scales", "opacities", "viewmats")}
    col = None if colors_f64 is None else colors_f64.clone().requires_grad_(True)
    Ks = torch.tensor(d["Ks"], dtype=f64)
    radii, m2, dep, rt, nrm = surfel.project(leaves["means"], leaves["quats"], leaves["scales"], leaves["viewmats"], Ks, W, H)
    C, N = m2.shape[-3], m2.shape[-2]
    has_depth = render_mode in ("D", "ED", "RGB+D", "RGB+ED")
    feat = None
    if col is not None:
        feat = torch.broadcast_to(col[..., None, :, :], col.shape[:-2] + (C,) + col.shape[-2:])
    if has_depth:
        feat = dep[..., None] if feat is None else torch.cat([feat, dep[..., None]], -1)
        if bg is not None and col is not None:
            bg = torch.cat([bg, torch.zeros_like(bg[..., :1])], -1)
    op = torch.broadcast_to(leaves["opacities"][..., None, :], m2.shape[:-1])
    raw_in = [m2, rt, feat, op, nrm]
    det = [x.detach() for x in raw_in]
    raw = surfel.rasterize(*det, W, H, 16, off, fl, backgrounds=None if bg is None else bg.detach())
    raw_leaf = [raw[n].detach().requires_grad_(True) for n in surfel._OUT_NAMES]
    rc, ra, rn, rd, rm = raw_leaf
    if render_mode in ("ED", "RGB+ED"):
        rc = torch.cat([rc[..., :-1], rc[..., -1:] / ra.clamp(min=1e-10)], -1)
    c2w = torch.linalg.inv(leaves["viewmats"])
    surf = None
    if has_depth and col is not None:
        surf = surfel.depth_to_normal(rm if depth_mode == "median" else rc[..., -1:], c2w, Ks).squeeze(0)
    rn_w = torch.einsum("...ij,...hwj->...hwi", c2w[..., :3, :3], rn)
    outs = [rc, ra, rn_w, surf, rd, rm]
    loss = sum((o * c).sum() for o, c in zip(outs, cots) if o is not None and c is not None)
    post = torch.autograd.grad(loss, raw_leaf + [leaves["viewmats"]], allow_unused=True)
    vj = surfel.rasterize_vjp(*det, W, H, 16, off, fl, [p for p in post[:5]], backgrounds=None if bg is None else bg.detach())
    grads_raw = [vj["v_means2d"], vj["v_ray_transforms"], vj["v_colors"], vj["v_opacities"], vj["v_normals"]]
    targets = [(x, gx) for x, gx in zip(raw_in, grads_raw) if x.requires_grad]
    keys = ["means", "quats", "scales", "opacities", "viewmats"]
    inputs = [leaves[k] for k in keys] + ([col] if col is not None else [])
    g = torch.autograd.grad([x for x, _ in targets], inputs, [gx for _, gx in targets], allow_unused=True)
    g = [torch.zeros_like(x) if gx is None else gx for x, gx in zip(inputs, g)]
    if post[5] is not None:
        g[4] = g[4] + post[5]
    names = keys + (["colors"] if col is not None else [])
    return [None if o is None else o.detach() for o in outs], dict(zip(names, g)), raw


def _run_2dgs(gs, d, W, H, render_mode="RGB", depth_mode="expected", distloss=False, bg=None, sh=False, vm_grad=True, seed=0,
              ops=("means", "quats", "scales", "opacities", "viewmats", "colors"), rel_grad=REL_GRAD, surf_cot=True, max_marginal=0.02):
    t = {k: torch.tensor(d[k], device=dev).requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "viewmats")}
    t["viewmats"].requires_grad_(vm_grad)
    Ks = torch.tensor(d["Ks"], device=dev)
    colors_in = torch.tensor(d["colors"], device=dev).requires_grad_(True)
    bg_t = None if bg is None else torch.tensor(bg, device=dev)
    out = gs.rasterization_2dgs(
        t["means"], t["quats"], t["scales"], t["opacities"], colors_in, t["viewmats"], Ks, W, H, render_mode=render_mode,
        depth_mode=depth_mode, distloss=distloss, backgrounds=bg_t, absgrad=True,
    )
    rc, ra, rn, surf, rd, rm, meta = out
    rng = np.random.RandomState(seed + 11)
    outs = [rc, ra, rn, surf, rd, rm]
    cots = [None if o is None else torch.tensor(rng.standard_normal(o.shape).astype(np.float32), device=dev) for o in outs]
    if surf is not None:
        # depth normals only where the 3 x 3 neighbourhood is well covered: next to empty pixels the cross product of
        # the point differences vanishes and its normalisation amplifies float32 rounding without bound
        a = torch.nn.functional.pad(ra.detach()[..., 0], (1, 1, 1, 1))
        a = a.reshape(-1, 1, H + 2, W + 2)
        cover = (-torch.nn.functional.max_pool2d(-a, 3, stride=1)).reshape(ra.shape[:-1]) > 0.9
        cots[3] = cots[3] * cover[..., None].reshape(cots[3].shape[:-1] + (1,)) * float(surf_cot)
    # no cotangent on pixels with a marginal threshold decision (from the float64 compositing of the projected rows): a
    # decision that flips there moves a gradient discontinuously
    fl = meta["flatten_ids"].cpu().numpy()
    off = meta["isect_offsets"].cpu().numpy()
    pre = surfel.rasterize(*(meta[k].detach().cpu().double() for k in ("means2d", "ray_transforms")),
                           torch.zeros(meta["means2d"].shape[:-1] + (1,), dtype=f64),
                           *(meta[k].detach().cpu().double() for k in ("opacities", "normals")), W, H, 16, off, fl)
    keep = torch.tensor(pre["margins"] > 1e-3, device=dev)[..., None]
    cots = [None if c is None else c * keep for c in cots]
    loss = sum((o * c).sum() for o, c in zip(outs, cots) if o is not None)
    loss.backward()
    torch.cuda.synchronize()
    has_color = render_mode in ("RGB", "RGB+D", "RGB+ED")
    col64 = torch.tensor(d["colors"], dtype=f64) if has_color else None
    ref_outs, ref_g, raw = _oracle_chain(
        d, W, H, fl, off, render_mode, depth_mode, None if bg is None else torch.tensor(bg, dtype=f64), col64,
        [None if c is None else c.cpu().double() for c in cots],
    )
    ok = raw["margins"] > 1e-3
    assert (~ok).mean() < max_marginal, f"{(~ok).mean() * 100:.2f}% marginal pixels"
    for name, a, b in zip(("colors", "alphas", "normals", "surf_normals", "distort", "median"), outs, ref_outs):
        if b is None:
            assert a is None, name
            continue
        a, b = _n(a), b.numpy()
        okb = np.broadcast_to(ok.reshape(ok.shape + (1,)), a.shape) if name != "surf_normals" else None
        if name == "surf_normals":
            m = cover.reshape(a.shape[:-1]).cpu().numpy()
            rel = _rel(a[m], b[m])
            assert rel < 1e-3, f"surf_normals rel L2 {rel:.3e}"
            continue
        err = np.abs(a - b) - (1e-4 * np.abs(b) + 1e-5)
        bad = (err > 0) & okb
        assert bad.mean() < 1e-3, f"{name}: {bad.mean() * 100:.3f}% out of tolerance, max err {np.abs(a - b)[okb].max():.2e}"
    got = {k: t[k].grad for k in ("means", "quats", "scales", "opacities", "viewmats")}
    got["colors"] = colors_in.grad
    for k in ops:
        if k not in ref_g or (k == "viewmats" and not vm_grad):
            continue
        rel = _rel(_n(got[k]), ref_g[k].numpy())
        assert rel < (REL_VIEWMATS if k == "viewmats" else rel_grad), f"v_{k}: rel L2 {rel:.3e}"
    assert meta["gradient_2dgs"].grad is not None and meta["gradient_2dgs"].grad.shape == meta["means2d"].shape
    assert meta["means2d"].absgrad.shape == meta["means2d"].shape
    return out


@pytest.mark.parametrize("render_mode", ["RGB", "D", "ED", "RGB+D", "RGB+ED"])
@pytest.mark.parametrize("distloss", [False, True])
@pytest.mark.parametrize("depth_mode", ["expected", "median"])
def test_rasterization_2dgs_modes(gs, render_mode, distloss, depth_mode):
    if distloss and render_mode == "RGB":
        pytest.skip("distloss needs a depth channel (ValueError, checked on the CPU)")
    W, H = 152, 104
    d = _scene(2500, W, H)
    _run_2dgs(gs, d, W, H, render_mode=render_mode, depth_mode=depth_mode, distloss=distloss)


def test_rasterization_2dgs_backgrounds_two_cameras(gs):
    W, H = 136, 88
    d = _scene(2500, W, H, C=2)
    bg = np.random.RandomState(5).random_sample((2, 3)).astype(np.float32)
    _run_2dgs(gs, d, W, H, render_mode="RGB+ED", bg=bg)


def test_rasterization_2dgs_batch_dims(gs):
    W, H = 120, 80
    d = _scene(1500, W, H, C=2, B=2)
    _run_2dgs(gs, d, W, H, render_mode="RGB+D", depth_mode="median", distloss=True)


def test_rasterization_2dgs_sh_matches_precomputed_colors(gs):
    W, H = 128, 96
    d = _scene(2000, W, H)
    sh = torch.tensor(d["sh"], device=dev).requires_grad_(True)
    args = [torch.tensor(d[k], device=dev) for k in ("means", "quats", "scales", "opacities")]
    vm, Ks = torch.tensor(d["viewmats"], device=dev), torch.tensor(d["Ks"], device=dev)
    out_sh = gs.rasterization_2dgs(*args, sh, vm, Ks, W, H, sh_degree=1, render_mode="RGB+D")
    rng = np.random.RandomState(0)
    cot = torch.tensor(rng.standard_normal(out_sh[0].shape).astype(np.float32), device=dev)
    (out_sh[0] * cot).sum().backward()
    sh2 = torch.tensor(d["sh"], device=dev).requires_grad_(True)
    radii = out_sh[6]["radii"]
    col = torch.clamp_min(gs.spherical_harmonics(1, args[0], vm, sh2, masks=(radii > 0).all(-1)) + 0.5, 0.0)
    out_pc = gs.rasterization_2dgs(*args, col, vm, Ks, W, H, render_mode="RGB+D")
    (out_pc[0] * cot).sum().backward()
    torch.testing.assert_close(out_sh[0], out_pc[0], rtol=0, atol=0)
    rel = float((sh.grad - sh2.grad).norm() / sh2.grad.norm())
    assert rel < 1e-6, rel


def test_rasterization_2dgs_empty_scene(gs):
    W, H = 64, 48
    d = _scene(200, W, H)
    means = torch.tensor(d["means"], device=dev)
    means = (means - means.mean(0)) * 0 + torch.tensor([0.0, 0.0, -50.0], device=dev)  # everything behind the cameras
    means.requires_grad_(True)
    op = torch.tensor(d["opacities"], device=dev).requires_grad_(True)
    col = torch.tensor(d["colors"], device=dev).requires_grad_(True)
    vm = torch.eye(4, device=dev)[None]
    bg = torch.tensor([[0.1, 0.2, 0.3]], device=dev)
    rc, ra, rn, surf, rd, rm, meta = gs.rasterization_2dgs(
        means, torch.tensor(d["quats"], device=dev), torch.tensor(d["scales"], device=dev), op, col, vm,
        torch.tensor(d["Ks"], device=dev), W, H, backgrounds=bg, render_mode="RGB+D",
    )
    assert meta["flatten_ids"].numel() == 0
    assert torch.equal(rc[..., :3], bg[:, None, None, :].expand(1, H, W, 3)) and (rc[..., 3] == 0).all()
    assert (ra == 0).all() and (rn == 0).all() and (rd == 0).all() and (rm == 0).all()
    (rc.sum() + ra.sum() + rd.sum() + rm.sum()).backward()
    assert (means.grad == 0).all() and (op.grad == 0).all() and (col.grad == 0).all()


def test_rasterization_2dgs_end_to_end_30k(gs):
    W, H = 320, 200
    d = _scene(30000, W, H)
    # no cotangent on the depth normals here: with 30k small surfels the neighbouring depths differ by little, and the
    # normal of their differences turns float32 depth rounding into gradient noise (the mode tests cover that path)
    # a denser scene takes more threshold decisions per pixel: more of its pixels are marginal.  The gaussian gradients sum
    # colour, depth-channel, distortion and expected-depth paths that partly cancel: in float32 the sum lands at about
    # 3e-3 relative L2 at this size (tests/test_gpu_parity.py allows 2e-3 for the 3DGS colour-only pipeline)
    _run_2dgs(gs, d, W, H, render_mode="RGB+ED", distloss=True, vm_grad=False, surf_cot=False, max_marginal=0.05, rel_grad=5e-3)


def test_rasterization_2dgs_forward_deterministic(gs):
    W, H = 200, 136
    d = _scene(8000, W, H, C=2)
    args = [torch.tensor(d[k], device=dev) for k in ("means", "quats", "scales", "opacities", "colors", "viewmats", "Ks")]
    a = gs.rasterization_2dgs(*args, W, H, render_mode="RGB+ED", distloss=True)
    b = gs.rasterization_2dgs(*args, W, H, render_mode="RGB+ED", distloss=True)
    for x, y in zip(a[:6], b[:6]):
        assert torch.equal(x, y)
