"""Sparse-pixel rendering (build_sparse_tile_layout, isect_tiles_sparse, rasterize_to_pixels_sparse) on the GPU.

The sparse result is defined as the dense rendering at each requested pixel, so every output is compared with the dense
ops of this library on the same inputs: the layout with a numpy model of its definition, the intersections with
isect_tiles(conics=None) + isect_offset_encode restricted to the active tiles, the forward bit for bit with
rasterize_to_pixels gathered at the pixels, the backward with the dense backward of the same cotangents scattered into
a zero image, and both with the float64 oracle.  Scene: a garden crop at 320 x 200 (the last tile row is half outside
the image), one and two cameras, dense and packed projections.
"""
import numpy as np
import pytest
import torch

from oracle import gso
from tests import scene

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
W, H = 320, 200
TW, TH = (W + 15) // 16, (H + 15) // 16
GRID_H = TH * 16  # 208: dense renders at the full tile grid also hold the margin pixels of the partial tile row


@pytest.fixture(scope="module")
def gs():
    import gsplat_b200

    assert torch.cuda.is_available(), "needs a GPU"
    return gsplat_b200


@pytest.fixture(scope="module")
def garden():
    sc = scene.make_scene(n_max=30000, sh_degree=0)
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)
    return sc, Ks


def _project(gs, garden, C, packed):
    """Projected rows: dict of means2d / conics / colors / opacities / radii / depths (+ image_ids when packed)."""
    sc, Ks = garden
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    means, quats, scales = t(sc["means"]), t(sc["quats"]), t(sc["scales"])
    opac, cols = t(sc["opacities"]), t(sc["colors"])
    vm, K = t(sc["viewmats"][:C]), t(Ks[:C])
    if packed:
        b, cam, gid, _, radii, m2, depths, conics, _ = gs.fully_fused_projection(means, None, quats, scales, vm, K, W, H, packed=True)
        return dict(means2d=m2, conics=conics, colors=cols[gid], opacities=opac[gid], radii=radii, depths=depths, image_ids=cam)
    radii, m2, depths, conics, _ = gs.fully_fused_projection(means, None, quats, scales, vm, K, W, H)
    N = means.shape[0]
    return dict(
        means2d=m2, conics=conics, colors=cols[None].expand(C, N, 3).contiguous(), opacities=opac[None].expand(C, N).contiguous(),
        radii=radii, depths=depths, image_ids=None,
    )


def _dense_lists(gs, rows, C, tw=TW, th=TH):
    packed = rows["image_ids"] is not None
    _, isect_ids, flatten_ids = gs.isect_tiles(
        rows["means2d"], rows["radii"], rows["depths"], 16, tw, th, packed=packed, n_images=C if packed else None,
        image_ids=rows["image_ids"],
    )
    return gs.isect_offset_encode(isect_ids, C, tw, th), flatten_ids


def _assert_active_lists(gs, rows, C, active, tile_offsets, flatten_ids, tw=TW, th=TH):
    """the sparse lists are the dense pipeline's lists of the active tiles, in its order"""
    offsets, fl = _dense_lists(gs, rows, C, tw, th)
    off = np.concatenate([offsets.cpu().numpy().reshape(-1), [fl.shape[0]]])
    fl = fl.cpu().numpy()
    exp_ids = [fl[off[t] : off[t + 1]] for t in active]
    exp_off = np.concatenate([[0], np.cumsum([len(x) for x in exp_ids])]).astype(np.int32)
    assert tile_offsets.dtype == torch.int32 and np.array_equal(tile_offsets.cpu().numpy(), exp_off)
    exp_fl = np.concatenate(exp_ids) if exp_ids else np.zeros(0, np.int32)
    assert np.array_equal(flatten_ids.cpu().numpy(), exp_fl)


def _pixel_set(kind, C, rng):
    """(pixels int32 [P, 2] (row, col), image_ids int32 [P])"""
    if kind == "random":
        per = []
        for i in range(C):
            flat = rng.choice(W * H, W * H // 100, replace=False)
            per.append(np.stack([flat // W, flat % W, np.full_like(flat, i)], -1))
        a = np.concatenate(per)
        a = a[rng.permutation(len(a))]
    elif kind == "patches":
        corners = [(0, 0), (40, 100), (150, 240), (168, 288)]  # the last one reaches the image's bottom-right corner
        a = np.array([(y0 + y, x0 + x, i) for i in range(C) for (y0, x0) in corners for y in range(32) for x in range(32)
                      if y0 + y < H and x0 + x < W])
    elif kind == "all":
        yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        a = np.concatenate([np.stack([yy.ravel(), xx.ravel(), np.full(H * W, i)], -1) for i in range(C)])
    elif kind == "one":
        a = np.array([[77, 131, C - 1]])
    elif kind == "empty":
        a = np.zeros((0, 3), np.int64)
    elif kind == "margin":
        # rows 200..207 of the half-outside last tile row, plus in-image pixels of the same tiles
        a = np.array([(y, x, i) for i in range(C) for y in range(192, GRID_H) for x in range(0, W, 3)])
        a = a[rng.permutation(len(a))]
    else:
        raise AssertionError(kind)
    a = np.asarray(a, np.int64).reshape(-1, 3)
    assert len(np.unique(a, axis=0)) == len(a), "requested pixels must not repeat"
    return torch.from_numpy(a[:, :2].astype(np.int32)).to(DEV), torch.from_numpy(a[:, 2].astype(np.int32)).to(DEV)


def _layout_model(pixels, image_ids, n_images):
    """numpy model of the layout's definition"""
    px, ids = pixels.cpu().numpy().astype(np.int64), image_ids.cpu().numpy().astype(np.int64)
    P = len(px)
    tile = (ids * TH + px[:, 0] // 16) * TW + px[:, 1] // 16
    pos = (px[:, 0] % 16) * 16 + px[:, 1] % 16
    pixel_map = np.argsort(tile * 256 + pos, kind="stable")
    active, counts = np.unique(tile, return_counts=True)
    mask = np.zeros(n_images * TH * TW, bool)
    mask[active] = True
    words = np.zeros((len(active), 4), np.uint64)
    r = np.searchsorted(active, tile)
    np.bitwise_or.at(words, (r, pos // 64), np.left_shift(np.uint64(1), (pos % 64).astype(np.uint64)))
    cumsum = np.cumsum(counts) if P else np.zeros(1, np.int64)
    return active.astype(np.int32), mask.reshape(n_images, TH, TW), words.view(np.int64), cumsum.astype(np.int64), pixel_map


def _gather(img, pixels, image_ids):
    p = pixels.long()
    return img[image_ids.long(), p[:, 0], p[:, 1]]


def _scatter(vals, pixels, image_ids, C, D):
    out = torch.zeros((C, GRID_H, W, D), device=DEV, dtype=vals.dtype)
    p = pixels.long()
    out[image_ids.long(), p[:, 0], p[:, 1]] = vals
    return out


def _sparse_pipeline(gs, rows, pixels, image_ids, C):
    layout = gs.build_sparse_tile_layout(pixels, image_ids, C, 16, TW, TH)
    active, amask = layout[0], layout[1]
    tile_offsets, flatten_ids = gs.isect_tiles_sparse(
        rows["means2d"], rows["radii"], rows["depths"], amask, active, C, 16, TW, TH, image_ids=rows["image_ids"]
    )
    return layout, tile_offsets, flatten_ids


KINDS = ["random", "patches", "all", "one", "empty", "margin"]


@pytest.mark.parametrize("packed", [False, True], ids=["dense", "packed"])
@pytest.mark.parametrize("C", [1, 2])
@pytest.mark.parametrize("kind", KINDS)
def test_layout_and_intersections(gs, garden, kind, C, packed):
    rng = np.random.RandomState(10 * KINDS.index(kind) + C)
    pixels, image_ids = _pixel_set(kind, C, rng)
    rows = _project(gs, garden, C, packed)
    (active, amask, words, cumsum, pmap), tile_offsets, flatten_ids = _sparse_pipeline(gs, rows, pixels, image_ids, C)
    m_active, m_mask, m_words, m_cumsum, m_pmap = _layout_model(pixels, image_ids, C)
    assert active.dtype == torch.int32 and np.array_equal(active.cpu().numpy(), m_active)
    assert amask.dtype == torch.bool and np.array_equal(amask.cpu().numpy(), m_mask)
    assert words.dtype == torch.uint64 and tuple(words.shape) == (len(m_active), 4)
    assert np.array_equal(words.view(torch.int64).cpu().numpy(), m_words)
    assert cumsum.dtype == torch.int64 and np.array_equal(cumsum.cpu().numpy(), m_cumsum)
    assert pmap.dtype == torch.int64 and np.array_equal(pmap.cpu().numpy(), m_pmap)
    # the intersections of the active tiles, in the dense pipeline's order
    _assert_active_lists(gs, rows, C, m_active, tile_offsets, flatten_ids)


@pytest.mark.parametrize("packed", [False, True], ids=["dense", "packed"])
def test_intersections_wide_tile_ids(gs, packed):
    """One image on a 300 x 256 tile grid: more than 65536 tiles, so the masked lists are sorted on 4-byte tile ids (the
    grid of the other tests fits 2-byte ids)."""
    tw, th, n = 300, 256, 4000
    rng = np.random.RandomState(5)
    m2 = rng.uniform(-40.0, [tw * 16 + 40.0, th * 16 + 40.0], (n, 2)).astype(np.float32)
    radii = rng.randint(1, 90, (n, 2)).astype(np.int32)
    radii[rng.rand(n) < 0.3] = 0  # culled rows
    depths = rng.choice(np.linspace(1.0, 40.0, 300), n).astype(np.float32)  # many equal depths: the row index decides
    t = lambda a: torch.from_numpy(a).to(DEV)  # noqa: E731
    if packed:
        rows = dict(means2d=t(m2), radii=t(radii), depths=t(depths), image_ids=torch.zeros(n, device=DEV, dtype=torch.int64))
    else:
        rows = dict(means2d=t(m2[None]), radii=t(radii[None]), depths=t(depths[None]), image_ids=None)
    flat = rng.choice(tw * 16 * th * 16, 20000, replace=False)
    pixels = t(np.stack([flat // (tw * 16), flat % (tw * 16)], -1).astype(np.int32))
    active, amask = gs.build_sparse_tile_layout(pixels, torch.zeros(len(flat), device=DEV, dtype=torch.int32), 1, 16, tw, th)[:2]
    tile_offsets, flatten_ids = gs.isect_tiles_sparse(
        rows["means2d"], rows["radii"], rows["depths"], amask, active, 1, 16, tw, th, image_ids=rows["image_ids"]
    )
    assert flatten_ids.shape[0] > 0
    _assert_active_lists(gs, rows, 1, active.cpu().numpy(), tile_offsets, flatten_ids, tw, th)


def _features(rows, D, seed):
    """D-channel features per row: the RGB colours, then seeded extra channels"""
    base = rows["colors"]
    if D <= 3:
        return base[..., :D].contiguous()
    g = torch.Generator(device=DEV).manual_seed(seed)
    extra = torch.rand(base.shape[:-1] + (D - 3,), device=DEV, generator=g)
    return torch.cat([base, extra], -1)


def _render_both(gs, rows, pixels, image_ids, C, D, bg, masks, absgrad, seed=0):
    """sparse and dense forward + backward with the same cotangents; returns the outputs and the gradients"""
    packed = rows["image_ids"] is not None
    layout, tile_offsets, flatten_ids = _sparse_pipeline(gs, rows, pixels, image_ids, C)
    offsets, fl = _dense_lists(gs, rows, C)
    feats = _features(rows, D, seed)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    P = pixels.shape[0]
    v_rc = torch.randn((P, D), device=DEV, generator=g)
    v_ra = torch.randn((P, 1), device=DEV, generator=g)
    out = {}
    for mode in ("sparse", "dense"):
        ins = [rows["means2d"].detach().clone().requires_grad_(True), rows["conics"].detach().clone().requires_grad_(True),
               feats.detach().clone().requires_grad_(True), rows["opacities"].detach().clone().requires_grad_(True)]
        tbg = bg.detach().clone().requires_grad_(True) if bg is not None else None
        if mode == "sparse":
            active, _, words, cumsum, pmap = layout
            rc, ra = gs.rasterize_to_pixels_sparse(
                *ins, image_ids, active, tile_offsets, flatten_ids, words, cumsum, pmap, W, H, 16, TW, TH, backgrounds=tbg,
                masks=masks, packed=packed, absgrad=absgrad,
            )
            loss = (rc * v_rc).sum() + (ra * v_ra).sum()
        else:
            rci, rai = gs.rasterize_to_pixels(*ins, W, GRID_H, 16, offsets, fl, backgrounds=tbg, masks=masks, packed=packed, absgrad=absgrad)
            rc, ra = _gather(rci, pixels, image_ids), _gather(rai, pixels, image_ids)
            loss = (rci * _scatter(v_rc, pixels, image_ids, C, D)).sum() + (rai * _scatter(v_ra, pixels, image_ids, C, 1)).sum()
        targets = ins + ([tbg] if tbg is not None else [])
        grads = torch.autograd.grad(loss, targets) if P > 0 else [torch.zeros_like(x) for x in targets]
        if absgrad and P > 0:
            grads = list(grads) + [ins[0].absgrad]
        out[mode] = (rc.detach(), ra.detach(), grads)
    return out, (layout, tile_offsets, flatten_ids, offsets, fl, feats, v_rc, v_ra)


def _rel(a, b):
    nb = torch.linalg.norm(b.double())
    return float(torch.linalg.norm(a.double() - b.double()) / max(float(nb), 1e-30))


@pytest.mark.parametrize("packed", [False, True], ids=["dense", "packed"])
@pytest.mark.parametrize("C", [1, 2])
@pytest.mark.parametrize("kind", KINDS)
def test_matches_dense(gs, garden, kind, C, packed):
    rng = np.random.RandomState(100 + 10 * KINDS.index(kind) + C)
    pixels, image_ids = _pixel_set(kind, C, rng)
    rows = _project(gs, garden, C, packed)
    out, _ = _render_both(gs, rows, pixels, image_ids, C, 3, None, None, False)
    (rc, ra, gs_), (drc, dra, dgs) = out["sparse"], out["dense"]
    assert rc.shape == (pixels.shape[0], 3) and ra.shape == (pixels.shape[0], 1)
    assert torch.equal(rc, drc) and torch.equal(ra, dra)
    for a, b in zip(gs_, dgs):
        assert _rel(a, b) <= 1e-6


@pytest.mark.parametrize("D", [1, 3, 6, 32])
@pytest.mark.parametrize("extras", ["plain", "bg", "bg+masks+absgrad"])
def test_channels_backgrounds_masks(gs, garden, D, extras):
    C = 2
    rng = np.random.RandomState(D)
    pixels, image_ids = _pixel_set("patches", C, rng)
    rows = _project(gs, garden, C, False)
    bg = torch.rand((C, D), device=DEV, generator=torch.Generator(device=DEV).manual_seed(D)) if extras != "plain" else None
    masks = None
    absgrad = extras == "bg+masks+absgrad"
    if absgrad:
        masks = torch.from_numpy(np.random.RandomState(3).random_sample((C, TH, TW)) > 0.3).to(DEV)
    out, _ = _render_both(gs, rows, pixels, image_ids, C, D, bg, masks, absgrad, seed=D)
    (rc, ra, g_s), (drc, dra, g_d) = out["sparse"], out["dense"]
    assert rc.shape == (pixels.shape[0], D)
    assert torch.equal(rc, drc) and torch.equal(ra, dra)
    assert len(g_s) == len(g_d) == 4 + (bg is not None) + absgrad
    for i, (a, b) in enumerate(zip(g_s, g_d)):
        # v_backgrounds (i == 4) is a float32 sum over all requested pixels, taken in another order than the dense
        # backward's sum over the image (with cancellation between pixels): 1e-5; the kernel gradients 1e-6
        tol = 1e-5 if i == 4 else 1e-6
        assert _rel(a, b) <= tol, f"gradient {i}: rel-L2 {_rel(a, b):.3e}"


def test_active_tile_with_empty_list(gs, garden):
    """A requested tile no gaussian reaches renders background / alpha 0 and gets an empty range."""
    C = 1
    rows = _project(gs, garden, C, False)
    t = 5 * TW + 7  # tile (7, 5): drop every gaussian whose box reaches it
    offsets, fl = _dense_lists(gs, rows, C)
    off = np.concatenate([offsets.cpu().numpy().reshape(-1), [fl.shape[0]]])
    hit = torch.from_numpy(fl.cpu().numpy()[off[t] : off[t + 1]].astype(np.int64)).to(DEV)
    radii = rows["radii"].clone()
    radii.view(-1, 2)[hit] = 0
    rows = dict(rows, radii=radii)
    pixels = torch.tensor([[5 * 16 + 3, 7 * 16 + 9], [5 * 16 + 15, 7 * 16], [10, 10]], device=DEV, dtype=torch.int32)
    image_ids = torch.zeros(3, device=DEV, dtype=torch.int32)
    bg = torch.tensor([[0.25, 0.5, 0.75]], device=DEV)
    out, (layout, tile_offsets, *_rest) = _render_both(gs, rows, pixels, image_ids, C, 3, bg, None, False)
    active = layout[0].cpu().numpy()
    a = int(np.nonzero(active == t)[0][0])
    assert tile_offsets[a] == tile_offsets[a + 1]
    rc, ra, g_s = out["sparse"]
    assert torch.equal(rc[:2], bg.expand(2, 3)) and torch.equal(ra[:2], torch.zeros_like(ra[:2]))
    assert torch.equal(rc, out["dense"][0]) and torch.equal(ra, out["dense"][1])
    for x, y in zip(g_s, out["dense"][2]):
        assert _rel(x, y) <= 1e-6


def test_matches_rasterization_image(gs, garden):
    """The sparse ops on rasterization()'s own projected rows reproduce its image at the requested pixels."""
    sc, Ks = garden
    C = 2
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    cols = t(sc["colors"])
    img, alpha, meta = gs.rasterization(
        t(sc["means"]), t(sc["quats"]), t(sc["scales"]), t(sc["opacities"]), cols, t(sc["viewmats"][:C]), t(Ks[:C]), W, H,
        packed=False,
    )
    N = cols.shape[0]
    rows = dict(
        means2d=meta["means2d"], conics=meta["conics"], colors=cols[None].expand(C, N, 3).contiguous(),
        opacities=meta["opacities"].expand(C, N).contiguous(), radii=meta["radii"], depths=meta["depths"], image_ids=None,
    )
    pixels, image_ids = _pixel_set("random", C, np.random.RandomState(11))
    (active, _, words, cumsum, pmap), tile_offsets, flatten_ids = _sparse_pipeline(gs, rows, pixels, image_ids, C)
    rc, ra = gs.rasterize_to_pixels_sparse(
        rows["means2d"], rows["conics"], rows["colors"], rows["opacities"], image_ids, active, tile_offsets, flatten_ids, words,
        cumsum, pmap, W, H, 16, TW, TH,
    )
    # the AABB lists are a superset of rasterization()'s lists; the extra pairs never reach alpha 1/255 in the tile
    exp_c, exp_a = _gather(img, pixels, image_ids), _gather(alpha, pixels, image_ids)
    assert (rc - exp_c).abs().max().item() <= 1e-6 and (ra - exp_a).abs().max().item() <= 1e-6
    assert torch.equal(rc, exp_c) and torch.equal(ra, exp_a)


@pytest.mark.parametrize("kind", ["random", "margin"])
def test_against_float64_oracle(gs, garden, kind):
    """Forward and backward against the float64 oracle compositing on the same lists, gathered at the pixels; pixels
    within 1e-4 of a compositing threshold and the gaussians of their tiles are left out of the strict checks."""
    C = 1
    rng = np.random.RandomState(5)
    pixels, image_ids = _pixel_set(kind, C, rng)
    rows = _project(gs, garden, C, False)
    bg = torch.tensor([[0.1, 0.2, 0.3]], device=DEV)
    out, (layout, _, _, offsets, fl, feats, v_rc, v_ra) = _render_both(gs, rows, pixels, image_ids, C, 3, bg, None, True)
    rc, ra, g_s = out["sparse"]
    n = lambda x: x.detach().cpu().numpy().astype(np.float64)  # noqa: E731
    m2, con, col, op = n(rows["means2d"]), n(rows["conics"]), n(feats), n(rows["opacities"])
    off, fln = offsets.cpu().numpy(), fl.cpu().numpy()
    orc, ora, oli, omg = gso.rasterize_to_pixels(m2, con, col, op, W, GRID_H, 16, off, fln, n(bg), None, True)
    px, ids = pixels.cpu().numpy().astype(np.int64), image_ids.cpu().numpy().astype(np.int64)
    ok = omg[ids, px[:, 0], px[:, 1]] > 1e-4
    assert ok.mean() > 0.99
    err_c = np.abs(n(rc) - orc[ids, px[:, 0], px[:, 1]])[ok]
    assert (err_c <= 1e-4 * np.abs(orc[ids, px[:, 0], px[:, 1]][ok]) + 1e-5).all()
    err_a = np.abs(n(ra) - ora[ids, px[:, 0], px[:, 1]])[ok]
    assert (err_a <= 1e-4 * np.abs(ora[ids, px[:, 0], px[:, 1]][ok]) + 1e-5).all()
    V = np.zeros(orc.shape)
    V[ids, px[:, 0], px[:, 1]] = n(v_rc)
    VA = np.zeros(ora.shape)
    VA[ids, px[:, 0], px[:, 1]] = n(v_ra)
    og = gso.rasterize_to_pixels_bwd(m2, con, col, op, W, GRID_H, 16, off, fln, ora, oli, V, VA, n(bg), None, True)
    # gaussians listed in a tile that holds a marginal requested pixel are excluded from the strict bound
    offf = np.concatenate([off.reshape(-1), [len(fln)]])
    tainted = np.zeros(m2.shape[0] * m2.shape[1], bool)
    for k in np.nonzero(~ok)[0]:
        tt = (ids[k] * TH + px[k, 0] // 16) * TW + px[k, 1] // 16
        tainted[fln[offf[tt] : offf[tt + 1]]] = True
    good = ~tainted.reshape(m2.shape[:-1])
    for a, key, mi in ((g_s[0], "v_means2d", 0), (g_s[1], "v_conics", 1), (g_s[3], "v_opacities", 2), (g_s[2], "v_colors", 3)):
        ref = og[key]
        m = og["mag"][..., mi]
        m = m[..., None] if ref.ndim > m.ndim else m
        diff = np.abs(n(a) - ref)
        g3 = np.broadcast_to(good[..., None] if ref.ndim > good.ndim else good, diff.shape)
        assert ((diff <= 1e-4 * m + 1e-5) | ~g3).mean() >= 0.999, key
        assert ((diff <= 1e-3 * m + 1e-4) | ~g3).all(), key
        assert np.linalg.norm(n(a) - ref) / max(np.linalg.norm(ref), 1e-30) < 1e-3, key
    vb = (V * (1.0 - ora)).sum(axis=(-3, -2))
    assert np.allclose(n(g_s[4]), vb, rtol=1e-3, atol=1e-2)
    rel = np.linalg.norm(n(g_s[5]) - og["v_means2d_abs"]) / np.linalg.norm(og["v_means2d_abs"])
    assert rel < 1e-4


def test_errors_before_launch(gs):
    px = torch.tensor([[0, 0], [5, 7]], device=DEV, dtype=torch.int32)
    ids = torch.zeros(2, device=DEV, dtype=torch.int32)
    with pytest.raises(ValueError, match="tile grid"):
        gs.build_sparse_tile_layout(torch.tensor([[0, 0], [TH * 16, 3]], device=DEV, dtype=torch.int32), ids, 1, 16, TW, TH)
    with pytest.raises(ValueError, match="tile grid"):
        gs.build_sparse_tile_layout(torch.tensor([[0, -1], [2, 3]], device=DEV, dtype=torch.int32), ids, 1, 16, TW, TH)
    with pytest.raises(ValueError, match="image id"):
        gs.build_sparse_tile_layout(px, torch.tensor([0, 1], device=DEV, dtype=torch.int32), 1, 16, TW, TH)
    with pytest.raises(ValueError, match="tile_size"):
        gs.build_sparse_tile_layout(px, ids, 1, 8, TW * 2, TH * 2)
    # a valid call on the same tensors still works afterwards
    active = gs.build_sparse_tile_layout(px, ids, 1, 16, TW, TH)[0]
    assert active.tolist() == [0]
