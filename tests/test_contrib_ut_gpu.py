"""The 3DGUT pair query and per-pixel contributor queries on the GPU.  Every output is the eval3d walk's, so each is
checked against rasterize_to_indices_in_range_eval3d(0, inf, T = 1), rasterize_to_pixels_eval3d and rasterization()
on the same inputs, and against a float64 pair walk (tests/ut_pairs.py, on oracle/ut.py's rays and responses).

* Counts equal the per-pixel pair counts; ids are the pairs in order; alphas equal render_alphas bit for bit, also
  those of rasterization(with_ut=True, with_eval3d=True) fed its meta.
* The weights sum to the alphas and reproduce render_colors when accumulated in float64.
* Counts that are too small keep each pixel's first K pairs; top-K equals the model of the reference's rule
  (tests/test_contrib_gpu.py) at K = 1, 8 and the bound; bound + 1 raises ValueError.
* Batch ranges [0, b) and [b, inf) add up to the full range; given transmittances, counts match the float64 walk.
* The sparse forms equal the dense queries gathered at the pixels (random pixels, 64 x 64 patches, margin pixels, an
  active tile with an empty list).
* FTheta pixels whose unprojection does not converge composite nothing.  Empty inputs; two runs are identical.

Scenes: garden crops at 320 x 200 (tests/scene.py) seen by one camera, two cameras and a batch of two; the distorted
pinhole, the fisheye, an FTheta calibration (tests/golden/ftheta_calibrations.json) and a top-to-bottom rolling shutter
(tests/test_ut_sparse_gpu.py's cameras).
"""
import numpy as np
import pytest
import torch

from oracle import ut as U
from tests import scene
from tests.test_contrib_gpu import top_model
from tests.ut_pairs import eval3d_pairs
from tests.test_sparse_raster_gpu import TH, TW, H, W, _pixel_set
from tests.test_ut_sparse_gpu import CAMS, LAYOUTS, _camera, _dense_lists, _rows, _sparse_pipeline, _t

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
BOUND = "gsb200_eval3d_contrib_max_samples"


@pytest.fixture(scope="module")
def gs():
    import gsplat_b200

    assert torch.cuda.is_available(), "needs a GPU"
    return gsplat_b200


def _n(t):
    return t.detach().cpu().numpy()


def _geom(rows):
    return tuple(rows[k] for k in ("means", "quats", "scales", "opacities", "viewmats", "Ks"))


def _pairs(gs, rows, offsets, fl, T=None, r0=0, r1=10**10):
    """the pair query: (gaussian ids, flat pixel index over the images, rank in the pixel)"""
    dims = rows["lead"]
    T = torch.ones(dims + (H, W), device=DEV) if T is None else T
    g, p, i = (_n(x) for x in gs.rasterize_to_indices_in_range_eval3d(r0, r1, T, *_geom(rows), W, H, 16, offsets, fl,
                                                                         **rows["kw"]))
    lin = i.astype(np.int64) * H * W + p
    first = np.r_[True, lin[1:] != lin[:-1]] if len(lin) else np.zeros(0, bool)
    start = np.maximum.accumulate(np.where(first, np.arange(len(lin)), 0)) if len(lin) else lin
    return g, lin, np.arange(len(lin)) - start


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("cam", list(CAMS))
def test_dense_queries(gs, cam, layout):
    B, C = LAYOUTS[layout]
    rows = _rows(gs, B, C, 3, cam, seed=3)
    offsets, fl = _dense_lists(gs, rows)
    args = _geom(rows) + (offsets, fl, W, H, 16)
    dims = rows["lead"]
    P = int(np.prod(dims)) * H * W
    g, lin, rank = _pairs(gs, rows, offsets, fl)
    assert len(g) > 1000
    # counts and alphas: the pairs, and the forward's render_alphas bit for bit
    counts, alphas = gs.rasterize_num_contributing_gaussians_eval3d(*args, **rows["kw"])
    assert counts.dtype == torch.int32 and counts.shape == dims + (H, W) and alphas.shape == dims + (H, W)
    assert np.array_equal(_n(counts).reshape(-1), np.bincount(lin, minlength=P))
    with torch.no_grad():
        rc, ra = gs.rasterize_to_pixels_eval3d(rows["means"], rows["quats"], rows["scales"], rows["colors"],
                                               rows["opacities"], rows["viewmats"], rows["Ks"], W, H, 16, offsets, fl,
                                               **rows["kw"])
    assert torch.equal(alphas, ra[..., 0]), int((alphas != ra[..., 0]).sum())
    # ids: the pairs in order, then -1 / 0
    ids, w = gs.rasterize_contributing_gaussian_ids_eval3d(*args, counts, **rows["kw"])
    K = int(counts.max())
    assert ids.shape == dims + (H, W, K) and w.dtype == torch.float32
    want = np.full((P, K), -1, np.int32)
    want[lin, rank] = g
    ids2, w2 = _n(ids).reshape(P, K), _n(w).reshape(P, K)
    assert np.array_equal(ids2, want)
    assert (w2[want < 0] == 0).all() and (w2[want >= 0] > 0).all()
    # the weights sum to the alphas and reproduce the render in float64
    N = rows["means"].shape[-2]
    wp = w2[lin, rank].astype(np.float64)
    col = _n(rows["colors"]).reshape(-1, 3).astype(np.float64)[g + (lin // (H * W)) * N]
    a64 = np.bincount(lin, wp, minlength=P)
    c64 = np.stack([np.bincount(lin, wp * col[:, k], minlength=P) for k in range(3)], -1)
    assert np.abs(a64 - _n(ra).reshape(-1)).max() < 1e-5
    assert np.abs(c64 - _n(rc).reshape(P, 3)).max() < 1e-4
    # counts too small keep each pixel's first pairs
    for cap in (1, max(K // 3, 1)):
        short = torch.clamp(counts, max=cap)
        short.view(-1)[0] = cap
        ids_s, w_s = gs.rasterize_contributing_gaussian_ids_eval3d(*args, short, **rows["kw"])
        assert torch.equal(ids_s, ids[..., :cap]) and torch.equal(w_s, w[..., :cap])
    # top-K against the model of the reference's rule, at 1, 8 and the bound
    bound = gs.ops._max_depth_samples(torch.device(DEV), BOUND)
    assert bound >= 8
    sel = np.sort(np.random.RandomState(0).choice(P, min(P, 20000), replace=False))
    for k in (1, 8, bound):
        top_i, top_w = gs.rasterize_top_contributing_gaussian_ids_eval3d(*args, k, **rows["kw"])
        assert top_i.shape == dims + (H, W, k)
        mi, mw = top_model(ids2[sel], w2[sel], k)
        assert np.array_equal(_n(top_i).reshape(P, k)[sel], mi) and np.array_equal(_n(top_w).reshape(P, k)[sel], mw)
    with pytest.raises(ValueError, match="exceeds"):
        gs.rasterize_top_contributing_gaussian_ids_eval3d(*args, bound + 1, **rows["kw"])
    # two runs are identical
    again = gs.rasterize_contributing_gaussian_ids_eval3d(*args, counts, **rows["kw"])
    assert torch.equal(again[0], ids) and torch.equal(again[1], w)


def test_rasterization_meta(gs):
    """fed rasterization()'s meta, the count query returns its render_alphas bit for bit"""
    rows = _rows(gs, 0, 2, 3, "rolling", seed=5)
    kw = rows["kw"]
    op = rows["opacities"][0]
    rc, ra, meta = gs.rasterization(rows["means"], rows["quats"], rows["scales"], op, rows["colors"], rows["viewmats"],
                                    rows["Ks"], W, H, packed=False, with_ut=True, with_eval3d=True, **kw)
    counts, alphas = gs.rasterize_num_contributing_gaussians_eval3d(
        rows["means"], rows["quats"], rows["scales"], meta["opacities"], rows["viewmats"], rows["Ks"],
        meta["isect_offsets"], meta["flatten_ids"], W, H, 16, **kw)
    assert torch.equal(alphas, ra[..., 0]) and int(counts.max()) > 0


@pytest.mark.parametrize("cam", ["pinhole", "rolling"])
def test_batch_ranges_add_up(gs, cam):
    """on a scene that never saturates, the pairs of [0, b) and [b, inf) from T = 1 are the full range's"""
    rows = _rows(gs, 0, 2, 3, cam, seed=7)
    rows["opacities"] = rows["opacities"] * 0.05
    offsets, fl = _dense_lists(gs, rows)
    full = _pairs(gs, rows, offsets, fl)
    _, alphas = gs.rasterize_num_contributing_gaussians_eval3d(*_geom(rows), offsets, fl, W, H, 16, **rows["kw"])
    assert float(alphas.max()) < 0.99  # T stays above 0.01: no walk stops, whatever batch it starts from
    for b in (1, 2):
        a, c = _pairs(gs, rows, offsets, fl, r1=b), _pairs(gs, rows, offsets, fl, r0=b)
        assert len(a[0]) > 0 and len(c[0]) > 0
        lin = np.concatenate([a[1], c[1]])
        order = np.argsort(lin, kind="stable")
        assert np.array_equal(lin[order], full[1]) and np.array_equal(np.concatenate([a[0], c[0]])[order], full[0])
    assert all(len(x) == 0 for x in _pairs(gs, rows, offsets, fl, r0=3, r1=3))


# ---- against the float64 pair walk (tests/ut_pairs.py), on a small scene
WS, HS = 96, 64


@pytest.mark.parametrize("cam", list(CAMS))
def test_against_float64_walk(gs, cam):
    """weights within the float32 budget and ids equal at pixels whose decisions are not marginal; with given
    transmittances, the counts of the pair query against the float64 walk's"""
    sc = scene.make_scene(n_max=400, sh_degree=0, seed=0)
    vm = sc["viewmats"][:1].astype(np.float32)
    K = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], WS, HS)[:1].astype(np.float32)
    K, kw, (model, coeffs, ftheta, vm_rs) = _camera(gs, cam, (1,), vm, K, WS, HS)
    s = (sc["scales"] * 4.0).astype(np.float32)
    N = len(s)
    geo = [_t(x) for x in (sc["means"], sc["quats"], s, sc["opacities"][None].astype(np.float32), vm, K)]
    with torch.no_grad():
        r, m2, d, _, _ = gs.fully_fused_projection_with_ut(*geo[:3], geo[3][0], geo[4], geo[5], WS, HS, **kw)
    tw, th = WS // 16, HS // 16
    hits = gs.ops.isect_tiles_sorted(m2, r, d, 16, tw, th)
    offs, fl = hits.isect_offsets.reshape(1, th, tw), hits.flatten_ids
    ocam = U.FThetaCamera(ftheta, K[0], WS, HS) if ftheta is not None else U.Camera(model, K[0], WS, HS, **coeffs)
    pose = vm[0] if vm_rs is None else U.ShutterPoses(vm[0], vm_rs[0], 0)
    f8 = [torch.from_numpy(np.asarray(x, np.float64)) for x in (sc["means"], sc["quats"], s, sc["opacities"])]
    T0 = np.random.RandomState(2).uniform(1e-3, 1.0, (1, HS, WS)).astype(np.float32)
    for T in (None, T0):
        o = eval3d_pairs(*f8, pose, ocam, offs.cpu(), fl.cpu().tolist(), 1, N, 0, transmittances=None if T is None else T[0])
        clear = (o["margins"] > 1e-3).numpy()
        if ftheta is not None:  # a Newton step near the 1e-6 convergence threshold may converge in one precision only
            step = ocam.last_step.reshape(-1).numpy()
            clear &= ~((step > 1e-7) & (step < 1e-5))
        if T is None:
            counts, _ = gs.rasterize_num_contributing_gaussians_eval3d(*geo, offs, fl, WS, HS, 16, **kw)
            ids, w = gs.rasterize_contributing_gaussian_ids_eval3d(*geo, offs, fl, WS, HS, 16, counts, **kw)
            ids, w, cnt = _n(ids).reshape(WS * HS, -1), _n(w).reshape(WS * HS, -1), _n(counts).reshape(-1)
            L = min(ids.shape[1], o["ids"].shape[1])
            oid = o["ids"].numpy()[:, :L]
            assert np.array_equal(cnt[clear], o["count"].numpy()[clear])
            assert np.array_equal(ids[clear, :L], np.where(oid >= 0, oid % N, -1)[clear])
            err = np.abs(w[:, :L] - o["weights"].numpy()[:, :L]).max(-1)
            assert ((err > 2e-4) & clear).sum() <= max(1, clear.size // 1000), ((err > 2e-4) & clear).sum()
            assert clear.mean() > 0.5 and cnt.max() > 0
        else:
            g, p, _ = (_n(x) for x in gs.rasterize_to_indices_in_range_eval3d(0, 10**10, _t(T), *geo, WS, HS, 16, offs,
                                                                                  fl, **kw))
            cnt = np.bincount(p, minlength=WS * HS)
            assert np.array_equal(cnt[clear], o["count"].numpy()[clear])


# ---- sparse forms against the dense queries gathered at the pixels
def _empty_first_tile(tile_offsets):
    """the same layout with the first active tile's list emptied"""
    t = tile_offsets.clone()
    t[0] = t[1]
    return t


@pytest.mark.parametrize("kind", ["random", "patches", "margin", "empty_tile"])
@pytest.mark.parametrize("cam", list(CAMS))
def test_sparse_equals_dense(gs, cam, kind):
    B, C = LAYOUTS["2cam"] if kind != "patches" else LAYOUTS["batch"]
    rows = _rows(gs, B, C, 3, cam, seed=11)
    I = int(np.prod(rows["lead"]))
    rng = np.random.RandomState(3)
    if kind == "patches":  # 64 x 64 patches
        a = np.array([(y0 + y, x0 + x, i) for i in range(I) for (y0, x0) in ((0, 0), (72, 100), (136, 256))
                      for y in range(64) for x in range(64)])
        assert len(np.unique(a, axis=0)) == len(a) and (a[:, 0] < H).all() and (a[:, 1] < W).all()
        pixels, image_ids = _t(a[:, :2].astype(np.int32)), _t(a[:, 2].astype(np.int32))
    else:
        pixels, image_ids = _pixel_set("random" if kind == "empty_tile" else kind, I, rng)
    (active, _, words, cumsum, pmap), tile_offsets, sfl = _sparse_pipeline(gs, rows, pixels, image_ids)
    if kind == "empty_tile":
        tile_offsets = _empty_first_tile(tile_offsets)
    offsets, fl = _dense_lists(gs, rows)
    dense = _geom(rows) + (offsets, fl, W, H, 16)
    sparse = _geom(rows) + (active, tile_offsets, sfl, words, cumsum, pmap)
    grid = (W, H, 16, TW, TH)
    kw = rows["kw"]
    p, ids_ = pixels.long(), image_ids.long()
    inside = p[:, 0] < H
    sel = (ids_[inside], p[inside, 0], p[inside, 1])
    lead_sel = lambda t: t.reshape((I, H, W) + t.shape[len(rows["lead"]) + 2:])[sel]
    # pixels of the emptied tile composite nothing
    keep = torch.ones(len(p), dtype=torch.bool, device=DEV)
    if kind == "empty_tile":
        tile = (ids_ * TH + p[:, 0] // 16) * TW + p[:, 1] // 16
        keep = tile != active[0].long()
        assert bool((~keep).any())
    dc, da = gs.rasterize_num_contributing_gaussians_eval3d(*dense, **kw)
    sc_, sa = gs.rasterize_num_contributing_gaussians_eval3d_sparse(*sparse, *grid, **kw)
    assert sc_.shape == (len(p),) and sa.shape == (len(p),)
    k_in = keep[inside]
    assert torch.equal(sc_[inside][k_in], lead_sel(dc)[k_in]) and torch.equal(sa[inside][k_in], lead_sel(da)[k_in])
    dead = ~inside | ~keep
    assert bool((sc_[dead] == 0).all()) and bool((sa[dead] == 0).all())
    di, dw = gs.rasterize_contributing_gaussian_ids_eval3d(*dense, dc, **kw)
    si, sw = gs.rasterize_contributing_gaussian_ids_eval3d_sparse(*sparse, sc_, *grid, **kw)
    Ks = si.shape[-1]
    assert torch.equal(si[inside][k_in], lead_sel(di)[k_in][:, :Ks]) and torch.equal(sw[inside][k_in], lead_sel(dw)[k_in][:, :Ks])
    assert bool((si[dead] == -1).all()) and bool((sw[dead] == 0).all())
    for k in (1, 8):
        ti, tw_ = gs.rasterize_top_contributing_gaussian_ids_eval3d(*dense, k, **kw)
        si, sw = gs.rasterize_top_contributing_gaussian_ids_eval3d_sparse(*sparse, *grid, k, **kw)
        assert torch.equal(si[inside][k_in], lead_sel(ti)[k_in]) and torch.equal(sw[inside][k_in], lead_sel(tw_)[k_in])
        assert bool((si[dead] == -1).all()) and bool((sw[dead] == 0).all())
    if kind == "margin":
        assert bool((~inside).any()) and int(sc_[inside].max()) > 0


def test_ftheta_pixels_that_do_not_converge(gs):
    """a forward polynomial that turns over: the pixels beyond its largest radius have no ray and composite nothing"""
    ft = dict(reference_poly=1, pixeldist_to_angle_poly=[0.0, 0.01, 0.0, 0.0, 0.0, 0.0],
              angle_to_pixeldist_poly=[0.0, 160.0, 0.0, -60.0, 0.0, 0.0], max_angle=1.5, linear_cde=[1.0, 0.0, 0.0])
    rows = _rows(gs, 0, 1, 3, "pinhole", seed=13)
    Kf = np.array([[[1.0, 0.0, W / 2 - 0.5], [0.0, 1.0, H / 2 - 0.5], [0.0, 0.0, 1.0]]], np.float32)
    kw = dict(camera_model="ftheta", ftheta_coeffs=gs.FThetaCameraDistortionParameters(**ft))
    rows["Ks"], rows["kw"] = _t(Kf), kw
    with torch.no_grad():
        r, m2, d, _, _ = gs.fully_fused_projection_with_ut(rows["means"], rows["quats"], rows["scales"],
                                                          rows["opacities"][0], rows["viewmats"], rows["Ks"], W, H, **kw)
    rows.update(radii=r, means2d=m2, depths=d)
    offsets, fl = _dense_lists(gs, rows)
    counts, alphas = gs.rasterize_num_contributing_gaussians_eval3d(*_geom(rows), offsets, fl, W, H, 16, **kw)
    ocam = U.FThetaCamera(ft, Kf[0], W, H)
    _, _, ok = U.pixel_rays(_n(rows["viewmats"])[0], ocam)
    step = ocam.last_step.reshape(-1).numpy()
    lost = (~ok).numpy() & (step > 1e-5)
    assert lost.sum() > 1000 and (ok.numpy() & (step < 1e-7)).sum() > 100
    c, a = _n(counts).reshape(-1), _n(alphas).reshape(-1)
    assert (c[lost] == 0).all() and (a[lost] == 0).all() and c[ok.numpy()].max() > 0
    ids, w = gs.rasterize_top_contributing_gaussian_ids_eval3d(*_geom(rows), offsets, fl, W, H, 16, 4, **kw)
    assert (_n(ids).reshape(-1, 4)[lost] == -1).all() and (_n(w).reshape(-1, 4)[lost] == 0).all()


def test_empty_inputs(gs):
    rows = _rows(gs, 0, 2, 3, "pinhole", seed=17)
    offsets = torch.zeros((2, TH, TW), device=DEV, dtype=torch.int32)
    fl = torch.zeros(0, device=DEV, dtype=torch.int32)
    args = _geom(rows) + (offsets, fl, W, H, 16)
    counts, alphas = gs.rasterize_num_contributing_gaussians_eval3d(*args, **rows["kw"])
    assert counts.shape == (2, H, W) and int(counts.abs().sum()) == 0 and float(alphas.abs().sum()) == 0
    ids, w = gs.rasterize_contributing_gaussian_ids_eval3d(*args, counts, **rows["kw"])
    assert ids.shape == (2, H, W, 0) and w.shape == (2, H, W, 0)
    ti, tw_ = gs.rasterize_top_contributing_gaussian_ids_eval3d(*args, 3, **rows["kw"])
    assert bool((ti == -1).all()) and bool((tw_ == 0).all())
    assert all(len(x) == 0 for x in _pairs(gs, rows, offsets, fl))
    # a sparse layout without pixels
    z32, z64 = torch.zeros(0, device=DEV, dtype=torch.int32), torch.zeros(0, device=DEV, dtype=torch.int64)
    sparse = _geom(rows) + (z32, torch.zeros(1, device=DEV, dtype=torch.int32), fl, torch.zeros((0, 4), device=DEV, dtype=torch.int64),
                            torch.zeros(1, device=DEV, dtype=torch.int64), z64)
    sc_, sa = gs.rasterize_num_contributing_gaussians_eval3d_sparse(*sparse, W, H, 16, TW, TH, **rows["kw"])
    assert sc_.shape == (0,) and sa.shape == (0,)
    si, sw = gs.rasterize_top_contributing_gaussian_ids_eval3d_sparse(*sparse, W, H, 16, TW, TH, 2, **rows["kw"])
    assert si.shape == (0, 2) and sw.shape == (0, 2)
