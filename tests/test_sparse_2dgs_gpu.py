"""rasterize_to_pixels_2dgs_sparse on the GPU.

The sparse result is defined as the dense 2DGS rendering at each requested pixel, so it is compared with the dense ops
of this library on the same surfel rows: the lists of isect_tiles_sparse with isect_tiles_sorted restricted to the
active tiles, all five forward outputs bit for bit with rasterize_to_pixels_2dgs gathered at the pixels, the backward
with the dense backward of the same cotangents scattered into zero images, and both with the float64 oracle
(oracle/surfel.py).  Scene: garden surfels at 320 x 200 (the last tile row is half outside the image, and the dense side
renders the full 208-row tile grid so that margin pixels exist), one and two cameras and a batch dimension; the pixel
sets are those of tests/test_sparse_raster_gpu.py.
"""
import numpy as np
import pytest
import torch

from oracle import surfel
from tests import scene
from tests.test_sparse_raster_gpu import GRID_H, KINDS, TH, TW, H, W, _pixel_set

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CHANNELS = (1, 2, 3, 4, 5, 8, 16, 32)
# layouts of the surfel rows: (batch B, cameras C); the images are the B * C leading rows
LAYOUTS = {"1cam": (0, 1), "2cam": (0, 2), "batch": (2, 2)}
REL_GRAD = 1e-3  # compositing gradients against float64 (tests/test_2dgs_gpu.py)
REL_RT = 5e-3  # v_ray_transforms and v_densify against float64 (tests/test_2dgs_gpu.py)


@pytest.fixture(scope="module")
def gs():
    import gsplat_b200

    assert torch.cuda.is_available(), "needs a GPU"
    return gsplat_b200


def _rows(gs, B, C, D, n=20000, seed=0):
    """Projected surfel rows [*lead, N, ...] (lead = (B, C) or (C,)), D channels whose last is the depth."""
    sc = scene.make_scene(n_max=n, sh_degree=0, seed=42 + seed)
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:C]
    vm = sc["viewmats"][:C]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    means, quats, scales, op = t(sc["means"]), t(sc["quats"]), t(sc["scales"] * 2.0), t(sc["opacities"])
    vm, Ks = t(vm), t(Ks)
    if B:
        rng = np.random.RandomState(seed)
        shift = torch.from_numpy(rng.standard_normal((B,) + tuple(means.shape)).astype(np.float32) * 0.01).to(DEV)
        shift[0] = 0
        means = means[None] + shift
        quats, scales = quats.expand(B, *quats.shape).contiguous(), scales.expand(B, *scales.shape).contiguous()
        vm, Ks = vm.expand(B, *vm.shape).contiguous(), Ks.expand(B, *Ks.shape).contiguous()
    with torch.no_grad():
        radii, m2, dep, rt, nrm = gs.fully_fused_projection_2dgs(means, quats, scales, vm, Ks, W, H)
    lead = tuple(m2.shape[:-1])
    g = torch.Generator(device=DEV).manual_seed(seed)
    col = torch.rand(lead + (D,), device=DEV, generator=g)
    col[..., -1] = dep  # the depth channel
    opac = torch.broadcast_to(op, lead).contiguous()
    return dict(means2d=m2, ray_transforms=rt, colors=col, opacities=opac, normals=nrm, radii=radii, depths=dep)


def _n_images(rows):
    return int(np.prod(rows["means2d"].shape[:-2]))


def _dense_lists(gs, rows):
    lead = tuple(rows["means2d"].shape[:-2])
    hits = gs.ops.isect_tiles_sorted(rows["means2d"], rows["radii"], rows["depths"], 16, TW, TH)
    return hits.isect_offsets.reshape(lead + (TH, TW)), hits.flatten_ids


def _sparse_pipeline(gs, rows, pixels, image_ids):
    I = _n_images(rows)
    N = rows["means2d"].shape[-2]
    layout = gs.build_sparse_tile_layout(pixels, image_ids, I, 16, TW, TH)
    tile_offsets, flatten_ids = gs.isect_tiles_sparse(
        rows["means2d"].reshape(I, N, 2), rows["radii"].reshape(I, N, 2), rows["depths"].reshape(I, N), layout[1], layout[0],
        I, 16, TW, TH,
    )
    return layout, tile_offsets, flatten_ids


def _gather(img, pixels, image_ids):
    """[*lead, GRID_H, W, k] at the requested pixels -> [P, k]"""
    p = pixels.long()
    return img.reshape((-1,) + tuple(img.shape[-3:]))[image_ids.long(), p[:, 0], p[:, 1]]


def _scatter(vals, pixels, image_ids, lead):
    out = torch.zeros((int(np.prod(lead)), GRID_H, W, vals.shape[-1]), device=DEV, dtype=vals.dtype)
    p = pixels.long()
    out[image_ids.long(), p[:, 0], p[:, 1]] = vals
    return out.reshape(tuple(lead) + (GRID_H, W, vals.shape[-1]))


KEYS = ("means2d", "ray_transforms", "colors", "opacities", "normals")


def _render_both(gs, rows, pixels, image_ids, bg=None, masks=None, absgrad=False, seed=0, cots=None):
    """Sparse and dense forward + backward with the same random cotangents on all five outputs.  Returns
    {mode: (outputs, gradients)}; gradients are v_means2d, v_ray_transforms, v_colors, v_opacities, v_normals,
    v_densify, then v_backgrounds and absgrad where present."""
    lead = tuple(rows["means2d"].shape[:-2])
    layout, tile_offsets, flatten_ids = _sparse_pipeline(gs, rows, pixels, image_ids)
    offsets, fl = _dense_lists(gs, rows)
    P, D = pixels.shape[0], rows["colors"].shape[-1]
    if cots is None:
        g = torch.Generator(device=DEV).manual_seed(seed + 1)
        cots = [torch.randn((P, k), device=DEV, generator=g) for k in (D, 1, 3, 1, 1)]
    out = {}
    for mode in ("sparse", "dense"):
        ins = [rows[k].detach().clone().requires_grad_(True) for k in KEYS]
        densify = torch.zeros(tuple(rows["means2d"].shape), device=DEV, requires_grad=True)
        tbg = bg.detach().clone().requires_grad_(True) if bg is not None else None
        if mode == "sparse":
            active, _, words, cumsum, pmap = layout
            outs = gs.rasterize_to_pixels_2dgs_sparse(
                *ins, densify, image_ids, active, tile_offsets, flatten_ids, words, cumsum, pmap, W, H, 16, TW, TH,
                backgrounds=tbg, masks=masks, absgrad=absgrad, distloss=True,
            )
            loss = sum((o * c).sum() for o, c in zip(outs, cots))
        else:
            dbg = tbg.reshape(lead + (D,)) if tbg is not None else None
            dm = masks.reshape(lead + (TH, TW)) if masks is not None else None
            imgs = gs.rasterize_to_pixels_2dgs(
                *ins, densify, W, GRID_H, 16, offsets, fl, backgrounds=dbg, masks=dm, absgrad=absgrad, distloss=True
            )
            outs = [_gather(o, pixels, image_ids) for o in imgs]
            loss = sum((o * _scatter(c, pixels, image_ids, lead)).sum() for o, c in zip(imgs, cots))
        targets = ins + [densify] + ([tbg] if tbg is not None else [])
        grads = list(torch.autograd.grad(loss, targets)) if P > 0 else [torch.zeros_like(x) for x in targets]
        if absgrad:
            grads.append(ins[0].absgrad if P > 0 else torch.zeros_like(ins[0]))
        out[mode] = ([o.detach() for o in outs], grads)
    return out, (layout, tile_offsets, flatten_ids, offsets, fl, cots)


def _rel(a, b):
    nb = torch.linalg.norm(b.double())
    return float(torch.linalg.norm(a.double() - b.double()) / max(float(nb), 1e-30))


def _check_equal_to_dense(out, has_bg=False):
    (so, sg), (do, dg) = out["sparse"], out["dense"]
    for name, a, b in zip(surfel._OUT_NAMES, so, do):
        assert a.shape == b.shape and torch.equal(a, b), name
    assert len(sg) == len(dg)
    for i, (a, b) in enumerate(zip(sg, dg)):
        # v_backgrounds (i == 6) is a float32 sum over the requested pixels, taken in another order than the dense
        # backward's sum over the image (with cancellation between pixels): 1e-5, as in tests/test_sparse_raster_gpu.py;
        # the kernel gradients 1e-6
        tol = 1e-5 if has_bg and i == 6 else 1e-6
        assert _rel(a, b) <= tol, f"gradient {i}: rel-L2 {_rel(a, b):.3e}"


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("kind", KINDS)
def test_lists_match_dense(gs, kind, layout):
    B, C = LAYOUTS[layout]
    rows = _rows(gs, B, C, 3)
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


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("kind", KINDS)
def test_matches_dense(gs, kind, layout):
    B, C = LAYOUTS[layout]
    rows = _rows(gs, B, C, 4)
    I = _n_images(rows)
    pixels, image_ids = _pixel_set(kind, I, np.random.RandomState(100 + 10 * KINDS.index(kind) + I))
    out, _ = _render_both(gs, rows, pixels, image_ids, absgrad=True, seed=KINDS.index(kind))
    P = pixels.shape[0]
    assert [tuple(o.shape) for o in out["sparse"][0]] == [(P, 4), (P, 1), (P, 3), (P, 1), (P, 1)]
    _check_equal_to_dense(out)


@pytest.mark.parametrize("D", CHANNELS)
@pytest.mark.parametrize("extras", ["plain", "bg+masks+absgrad"])
def test_channels_backgrounds_masks(gs, D, extras):
    rows = _rows(gs, 0, 2, D, seed=D)
    pixels, image_ids = _pixel_set("patches", 2, np.random.RandomState(D))
    bg = masks = None
    absgrad = extras != "plain"
    if absgrad:
        bg = torch.rand((2, D), device=DEV, generator=torch.Generator(device=DEV).manual_seed(D))
        masks = torch.from_numpy(np.random.RandomState(3).random_sample((2, TH, TW)) > 0.3).to(DEV)
    out, (layout, *_rest) = _render_both(gs, rows, pixels, image_ids, bg=bg, masks=masks, absgrad=absgrad, seed=D)
    if masks is not None:  # some requested tiles are masked off: they show the background
        assert not masks.reshape(-1)[layout[0].long()].all()
    _check_equal_to_dense(out, has_bg=bg is not None)
    assert len(out["sparse"][1]) == 6 + (bg is not None) + absgrad


def test_active_tile_with_empty_list(gs):
    """A requested tile no surfel reaches renders the background and zeros and has an empty range."""
    rows = _rows(gs, 0, 1, 3)
    t = 5 * TW + 7  # tile (7, 5): drop every surfel whose box reaches it
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
    out, (layout, tile_offsets, *_rest) = _render_both(gs, rows, pixels, image_ids, bg=bg, absgrad=True)
    a = int(np.nonzero(layout[0].cpu().numpy() == t)[0][0])
    assert tile_offsets[a] == tile_offsets[a + 1]
    rc, ra, rn, rd, rm = out["sparse"][0]
    assert torch.equal(rc[:2], bg.expand(2, 3))
    for x in (ra, rn, rd, rm):
        assert torch.equal(x[:2], torch.zeros_like(x[:2]))
    _check_equal_to_dense(out, has_bg=True)


def test_no_lists_at_all(gs):
    """Nothing listed in any active tile: the background at every requested pixel, zero gradients but v_backgrounds."""
    rows = _rows(gs, 0, 2, 3, n=2000)
    rows = dict(rows, radii=torch.zeros_like(rows["radii"]))
    pixels, image_ids = _pixel_set("random", 2, np.random.RandomState(4))
    bg = torch.rand((2, 3), device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    out, (_, _, flatten_ids, *_rest) = _render_both(gs, rows, pixels, image_ids, bg=bg, absgrad=True)
    assert flatten_ids.numel() == 0
    rc, ra, rn, rd, rm = out["sparse"][0]
    assert torch.equal(rc, bg[image_ids.long()])
    assert all(torch.equal(x, torch.zeros_like(x)) for x in (ra, rn, rd, rm))
    grads = out["sparse"][1]
    assert all(torch.equal(x, torch.zeros_like(x)) for i, x in enumerate(grads) if i != 6)
    _check_equal_to_dense(out, has_bg=True)


def test_no_pixels(gs):
    rows = _rows(gs, 0, 1, 3, n=2000)
    pixels, image_ids = _pixel_set("empty", 1, np.random.RandomState(0))
    layout, tile_offsets, flatten_ids = _sparse_pipeline(gs, rows, pixels, image_ids)
    active, _, words, cumsum, pmap = layout
    ins = [rows[k].detach().clone().requires_grad_(True) for k in KEYS]
    densify = torch.zeros(tuple(rows["means2d"].shape), device=DEV, requires_grad=True)
    outs = gs.rasterize_to_pixels_2dgs_sparse(
        *ins, densify, image_ids, active, tile_offsets, flatten_ids, words, cumsum, pmap, W, H, 16, TW, TH,
        backgrounds=torch.ones((1, 3), device=DEV),
    )
    assert [tuple(o.shape) for o in outs] == [(0, 3), (0, 1), (0, 3), (0, 1), (0, 1)]
    sum(o.sum() for o in outs).backward()
    assert all(torch.equal(x.grad, torch.zeros_like(x)) for x in ins + [densify])


@pytest.mark.parametrize("kind", ["random", "margin"])
def test_against_float64_oracle(gs, kind):
    """Forward and backward at the requested pixels against the float64 oracle compositing on the same lists, with the
    tolerances of tests/test_2dgs_gpu.py; requested pixels whose threshold decisions are marginal get no cotangent."""
    rows = _rows(gs, 0, 1, 4, n=4000, seed=1)
    pixels, image_ids = _pixel_set(kind, 1, np.random.RandomState(5))
    bg = torch.tensor([[0.1, 0.2, 0.3, 0.0]], device=DEV)
    offsets, fl = _dense_lists(gs, rows)
    o64 = {k: rows[k].detach().cpu().double() for k in KEYS}
    off_np, fl_np = offsets.cpu().numpy(), fl.cpu().numpy()
    pre = surfel.rasterize(*(o64[k] for k in KEYS), W, GRID_H, 16, off_np, fl_np, backgrounds=bg.cpu().double())
    px, ids = pixels.cpu().numpy().astype(np.int64), image_ids.cpu().numpy().astype(np.int64)
    ok = pre["margins"][ids, px[:, 0], px[:, 1]] > 1e-3
    assert ok.mean() > 0.97
    P = pixels.shape[0]
    g = torch.Generator(device=DEV).manual_seed(9)
    keep = torch.from_numpy(ok).to(DEV)[:, None]
    cots = [torch.randn((P, k), device=DEV, generator=g) * keep for k in (4, 1, 3, 1, 1)]
    out, _ = _render_both(gs, rows, pixels, image_ids, bg=bg, absgrad=True, cots=cots)
    outs, grads = out["sparse"]
    lead = tuple(rows["means2d"].shape[:-2])
    ref = surfel.rasterize_vjp(
        *(o64[k] for k in KEYS), W, GRID_H, 16, off_np, fl_np,
        [_scatter(c, pixels, image_ids, lead).cpu().double() for c in cots], backgrounds=bg.cpu().double(),
    )
    for name, a in zip(surfel._OUT_NAMES, outs):
        b = ref[name].numpy()[ids, px[:, 0], px[:, 1]][ok]
        a = a.double().cpu().numpy()[ok]
        bad = np.abs(a - b) > 1e-4 * np.abs(b) + 1e-5
        assert bad.mean() < 1e-3, f"{name}: {bad.mean() * 100:.3f}% of non-marginal pixels out of tolerance"
    for k, a in zip(KEYS, grads):
        rel = _rel(a.cpu(), ref["v_" + k])
        assert rel < (REL_RT if k == "ray_transforms" else REL_GRAD), f"v_{k}: rel L2 {rel:.3e}"
    rel = _rel(grads[5].cpu(), ref["v_densify"])
    assert rel < REL_RT, f"v_densify: rel L2 {rel:.3e}"
    rel = _rel(grads[6].cpu(), ref["v_backgrounds"])
    assert rel < REL_GRAD, f"v_backgrounds: rel L2 {rel:.3e}"
    rel = _rel(grads[7].cpu(), ref["absgrad"])
    assert rel < REL_GRAD, f"absgrad: rel L2 {rel:.3e}"


def test_forward_deterministic(gs):
    rows = _rows(gs, 0, 2, 4)
    pixels, image_ids = _pixel_set("random", 2, np.random.RandomState(7))
    (active, _, words, cumsum, pmap), tile_offsets, flatten_ids = _sparse_pipeline(gs, rows, pixels, image_ids)
    densify = torch.zeros(tuple(rows["means2d"].shape), device=DEV)
    run = lambda: gs.rasterize_to_pixels_2dgs_sparse(  # noqa: E731
        *(rows[k] for k in KEYS), densify, image_ids, active, tile_offsets, flatten_ids, words, cumsum, pmap, W, H, 16, TW, TH
    )
    for x, y in zip(run(), run()):
        assert torch.equal(x, y)
