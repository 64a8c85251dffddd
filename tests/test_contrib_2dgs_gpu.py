"""The 2DGS per-pixel contributor queries on the GPU.  Every output is the surfel walk's, so each is checked against
rasterize_to_indices_in_range_2dgs(0, inf, T = 1) and rasterize_to_pixels_2dgs on the same inputs.

* Counts equal the per-pixel pair counts and alphas equal render_alphas bit for bit (garden surfels at 320 x 200, a
  height that is not a multiple of 16, with one camera, two cameras and a batch dimension; the tie images of
  tests/surfel_edges.py).
* Padded ids are the pairs in order, -1 / 0 after them; the weights sum to the alphas, and a float64 accumulate of
  weights x colours reproduces render_colors.
* Each weight is the float64 alpha * T of oracle/surfel.py, within the compositing tolerance plus its float32 budget,
  at pixels whose threshold decisions are not marginal.
* Counts that are too small keep the first K pairs of every pixel.
* Top-K equals the numpy model of the reference's rule (tests/test_contrib_gpu.py) applied to the padded lists, at
  K = 1, 8 and the surfel walk's bound; one more than the bound is a ValueError.
* The _2dgs_sparse forms equal the dense queries gathered at the pixels: random pixels and 64 x 64 patches, margin
  pixels of the partial tile row, one and two cameras, and an active tile with an empty list.
* Empty inputs, and two runs give identical outputs.
"""
import numpy as np
import pytest
import torch

from oracle import surfel
from tests import surfel_edges as se
from tests import test_sparse_2dgs_gpu as s2
from tests.test_contrib_gpu import top_model
from tests.test_indices_gpu import _n, _pixel, _t
from tests.test_sparse_raster_gpu import GRID_H, TH, TW, H, W, _pixel_set

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SURFEL_BOUND = "gsb200_surfel_contrib_max_samples"
RTOL, ATOL = 1e-4, 1e-5  # the 2DGS compositing tolerance against float64 (tests/test_2dgs_gpu.py)
MARGIN = 1e-3  # pixels whose threshold decisions lie closer than this (relative) are marginal
ULP = 2.0**-24


@pytest.fixture(scope="module")
def gs():
    import gsplat_b200

    assert torch.cuda.is_available(), "needs a GPU"
    return gsplat_b200


def _view(gs, B, C, n=20000, seed=0):
    """garden surfel rows at W x H with their dense lists: dict of tensors with image dims (C,) or (B, C)"""
    rows = s2._rows(gs, B, C, 3, n=n, seed=seed)
    off, fl = s2._dense_lists(gs, rows)
    return dict(rows, isect_offsets=off, flatten_ids=fl, W=W, H=H)


def _args(v):
    return (v["means2d"], v["ray_transforms"], v["opacities"], v["isect_offsets"], v["flatten_ids"], v["W"], v["H"], 16)


def _lists(gs, v):
    """the pairs of rasterize_to_indices_in_range_2dgs(0, inf, T = 1): (surfel ids, flat pixel index, rank in the pixel)"""
    Wv, Hv = v["W"], v["H"]
    dims = tuple(v["isect_offsets"].shape[:-2])
    ones = torch.ones(dims + (Hv, Wv), device=DEV)
    ids = gs.rasterize_to_indices_in_range_2dgs(0, 10**10, ones, v["means2d"], v["ray_transforms"], v["opacities"], Wv, Hv,
                                                16, v["isect_offsets"], v["flatten_ids"])
    g, lin = _pixel(ids, Hv, Wv)
    first = np.r_[True, lin[1:] != lin[:-1]] if len(lin) else np.zeros(0, bool)
    start = np.maximum.accumulate(np.where(first, np.arange(len(lin)), 0)) if len(lin) else lin
    return g, lin, np.arange(len(lin)) - start


def _check_view(gs, v, top_ks, n_model=None, seed=0):
    """counts, alphas, padded ids, weights, short counts and top-K on one dense view; returns (largest count, ids,
    weights)"""
    Wv, Hv = v["W"], v["H"]
    dims = tuple(v["isect_offsets"].shape[:-2])
    P = int(np.prod(dims)) * Hv * Wv
    g, lin, rank = _lists(gs, v)
    g_t, lin_t, rank_t = (torch.from_numpy(x).to(DEV) for x in (g, lin, rank))
    # counts and alphas
    counts, alphas = gs.rasterize_num_contributing_gaussians_2dgs(*_args(v))
    assert counts.dtype == torch.int32 and alphas.dtype == torch.float32
    assert counts.shape == dims + (Hv, Wv) and alphas.shape == dims + (Hv, Wv)
    assert np.array_equal(_n(counts).reshape(-1), np.bincount(lin, minlength=P)), "counts differ from the pair counts"
    colors = v["colors"]
    rc, ra, *_ = gs.rasterize_to_pixels_2dgs(v["means2d"], v["ray_transforms"], colors, v["opacities"], v["normals"],
                                             torch.zeros_like(v["means2d"]), Wv, Hv, 16, v["isect_offsets"],
                                             v["flatten_ids"])
    bad = int((alphas != ra[..., 0]).sum())
    assert bad == 0, f"{bad} alphas differ from render_alphas"
    # padded ids: the pairs in order, then -1 / 0
    ids, w = gs.rasterize_contributing_gaussian_ids_2dgs(*_args(v), counts)
    K = int(counts.max()) if P else 0
    assert ids.dtype == torch.int32 and w.dtype == torch.float32 and ids.shape == dims + (Hv, Wv, K)
    want = torch.full((P, K), -1, device=DEV, dtype=torch.int32)
    want[lin_t, rank_t] = g_t.to(torch.int32)
    ids2, w2 = ids.reshape(P, K), w.reshape(P, K)
    assert torch.equal(ids2, want), f"{int((ids2 != want).sum())} ids differ from the pairs"
    assert bool((w2[want < 0] == 0).all()) and bool((w2[want >= 0] > 0).all())
    # the weights sum to the alphas, and weights x colours reproduce the render
    N = v["means2d"].shape[-2]
    rows = g_t + (lin_t // (Hv * Wv)) * N
    wp = w2[lin_t, rank_t].double()
    col = colors.reshape(-1, colors.shape[-1]).double()[rows]
    c64 = torch.zeros((P, col.shape[1]), device=DEV, dtype=torch.float64).index_add_(0, lin_t, wp[:, None] * col)
    a64 = w2.double().sum(1)
    torch.testing.assert_close(a64, alphas.reshape(-1).double(), rtol=RTOL, atol=ATOL)
    torch.testing.assert_close(c64, rc.reshape(P, -1).double(), rtol=RTOL, atol=ATOL)
    # counts too small: every pixel keeps its first pairs, nothing lands outside its row
    for cap in (1, max(K // 3, 1)):
        short = torch.clamp(counts, max=cap)
        short.view(-1)[0] = cap
        ids_s, w_s = gs.rasterize_contributing_gaussian_ids_2dgs(*_args(v), short)
        assert torch.equal(ids_s, ids[..., :cap]) and torch.equal(w_s, w[..., :cap])
    # top-K against the model of the reference's rule
    rng = np.random.RandomState(seed)
    sel = np.arange(P) if n_model is None or n_model >= P else np.sort(rng.choice(P, n_model, replace=False))
    sel_t = torch.from_numpy(sel).to(DEV)
    ids_n, w_n = _n(ids2[sel_t]), _n(w2[sel_t])
    for k in top_ks:
        top_i, top_w = gs.rasterize_top_contributing_gaussian_ids_2dgs(*_args(v), k)
        assert top_i.shape == dims + (Hv, Wv, k) and top_w.shape == dims + (Hv, Wv, k)
        mi, mw = top_model(ids_n, w_n, k)
        ti, tw = _n(top_i.reshape(P, k)[sel_t]), _n(top_w.reshape(P, k)[sel_t])
        assert np.array_equal(ti, mi) and np.array_equal(tw, mw), f"K = {k}: {int((ti != mi).any(1).sum())} pixels differ from the model"
        if k >= K:
            pad = (0, k - K)
            assert torch.equal(top_i.reshape(P, k), torch.nn.functional.pad(ids2, pad, value=-1))
            assert torch.equal(top_w.reshape(P, k), torch.nn.functional.pad(w2, pad))
    return K, ids, w


def _check_oracle_weights(v, ids, w, min_checked):
    """every weight against the float64 alpha * T of the oracle's compositing of the same lists, at the pixels whose
    threshold decisions (alpha cull, stop, median) are not marginal: within the compositing tolerance plus the weight's
    float32 budget"""
    f64 = torch.float64
    dims = tuple(v["isect_offsets"].shape[:-2])
    I, N = int(np.prod(dims)), v["means2d"].shape[-2]
    Wv, Hv = v["W"], v["H"]
    m2 = torch.tensor(_n(v["means2d"]).reshape(I * N, 2), dtype=f64)
    rt = torch.tensor(_n(v["ray_transforms"]).reshape(I * N, 3, 3), dtype=f64)
    op = torch.tensor(_n(v["opacities"]).reshape(I * N), dtype=f64)
    col = torch.tensor(_n(v["colors"]).reshape(I * N, -1), dtype=f64)
    nrm = torch.tensor(_n(v["normals"]).reshape(I * N, 3), dtype=f64)
    off, fl = _n(v["isect_offsets"]).reshape(I, *v["isect_offsets"].shape[-2:]), _n(v["flatten_ids"]).astype(np.int64)
    ids_n, w_n = _n(ids).reshape(I, Hv, Wv, -1), _n(w).reshape(I, Hv, Wv, -1)
    checked = total = 0
    for _, img, ys, xs, s0, s1 in surfel._tiles(Wv, Hv, 16, off, fl):
        total += len(ys)
        px, py = torch.as_tensor(xs, dtype=f64) + 0.5, torch.as_tensor(ys, dtype=f64) + 0.5
        lst = torch.as_tensor(fl[s0:s1])
        res = surfel._tile(px, py, m2[lst], rt[lst], op[lst], col[lst], nrm[lst], None)
        keep = res[7].numpy() > MARGIN
        if s1 == s0:
            assert (ids_n[img, ys, xs] == -1).all()
            checked += int(keep.sum())
            continue
        a = res[9][0]  # alpha of each (pixel, listed surfel), 0 where culled
        T_after = torch.cumprod(1.0 - a, dim=1)
        T_before = torch.cat([torch.ones_like(T_after[:, :1]), T_after[:, :-1]], dim=1)
        alive = torch.cumsum(((a > 0) & (T_after <= surfel.TRANSMITTANCE_THRESHOLD)).to(torch.int64), 1) == 0
        use = (a > 0) & alive
        w64 = torch.where(use, a * T_before, torch.zeros_like(a))
        # float32 budget of each weight: the relative error of alpha, i.e. the absolute error of sigma, plus that of T
        # before the pair.  Ray-splat kernel: hu = px * M2 - M0 and hv cancel, and so do the cross products that u, v
        # divide.  Screen-space kernel: dx = mean - px cancels.  Then fast_exp, and two roundings per factor of T.
        R, mean = rt[lst][None], m2[lst][None]
        pxy = torch.stack([px, py], -1)[:, None]
        hu = px[:, None, None] * R[..., 2, :] - R[..., 0, :]
        hv = py[:, None, None] * R[..., 2, :] - R[..., 1, :]
        nrm3 = lambda x: torch.linalg.norm(x, dim=-1)  # noqa: E731
        big = (nrm3(px[:, None, None] * R[..., 2, :]) + nrm3(R[..., 0, :]) + nrm3(hu)) * \
              (nrm3(py[:, None, None] * R[..., 2, :]) + nrm3(R[..., 1, :]) + nrm3(hv))
        s = torch.linalg.cross(hu, hv, dim=-1)
        uv = (s[..., 0].abs() + s[..., 1].abs()) / s[..., 2].abs()  # |u| + |v|; inf only where culled
        g3 = (s[..., 0] ** 2 + s[..., 1] ** 2) / s[..., 2] ** 2
        d = mean - pxy
        g2 = surfel.FILTER_INV_SQUARE * (d * d).sum(-1)
        b3 = 4.0 * ULP * big / s[..., 2].abs() * (1.0 + uv) * uv
        b2 = 4.0 * ULP * surfel.FILTER_INV_SQUARE * (d.abs() * (mean.abs() + pxy.abs())).sum(-1)
        sigma = 0.5 * torch.minimum(g3, g2)
        rel_a = torch.where(use, torch.where(g3 < g2, b3, b2) + (4.0 + 1.2 * sigma) * ULP, torch.zeros_like(a))
        rel_1ma = torch.where(use, a * rel_a / (1.0 - a) + 2.0 * ULP, torch.zeros_like(a))  # of each factor 1 - alpha
        rel_T = torch.cumsum(rel_1ma, 1) - rel_1ma
        tol = (w64 * (rel_a + rel_T)).numpy()
        w64 = w64.numpy()
        use = use.numpy() & keep[:, None]
        cnt = use.sum(1)
        kk = ids_n.shape[-1]
        assert (cnt[keep] <= kk).all()
        # the oracle's pairs of a kept pixel are ours, in order, with their weights
        p_i, k_i = np.nonzero(use)
        r = (np.cumsum(use, 1) - 1)[p_i, k_i]
        got_id, got_w = ids_n[img, ys[p_i], xs[p_i], r], w_n[img, ys[p_i], xs[p_i], r]
        assert np.array_equal(got_id, fl[s0 + k_i] % N), "pairs differ from the float64 oracle"
        err = np.abs(got_w - w64[p_i, k_i]) - tol[p_i, k_i]
        assert (err <= ATOL + RTOL * w64[p_i, k_i]).all(), f"weights beyond their float32 budget by up to {err.max():.3g}"
        # and nothing after them
        full = np.concatenate([ids_n[img, ys, xs], np.full((len(ys), 1), -1, ids_n.dtype)], 1)
        assert (full[keep, cnt[keep]] == -1).all()
        checked += int(keep.sum())
    assert checked >= min_checked * total, f"only {checked} of {total} pixels are away from a threshold decision"
    return checked


LAYOUTS = {"1cam": (0, 1), "2cam": (0, 2), "batch": (2, 2)}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_garden_surfels(gs, layout):
    v = _view(gs, *LAYOUTS[layout])
    bound = gs.ops._max_depth_samples(torch.device(DEV), SURFEL_BOUND)
    assert bound >= 32
    K, ids, w = _check_view(gs, v, (1, 8, bound), n_model=20000)
    assert K > 8
    with pytest.raises(ValueError, match=f"exceeds {bound}"):
        gs.rasterize_top_contributing_gaussian_ids_2dgs(*_args(v), bound + 1)
    with pytest.raises(ValueError, match=f"exceeds {bound}"):
        active = torch.zeros(1, device=DEV, dtype=torch.int32)
        z64 = torch.zeros((1, 4), device=DEV, dtype=torch.int64)
        gs.rasterize_top_contributing_gaussian_ids_2dgs_sparse(
            v["means2d"], v["ray_transforms"], v["opacities"], active, torch.zeros(2, device=DEV, dtype=torch.int32),
            v["flatten_ids"][:0], z64, z64[:, 0], z64[:0, 0], W, H, 16, TW, TH, bound + 1)
    if layout == "1cam":
        _check_oracle_weights(v, ids, w, min_checked=0.9)
    print(f"\n{layout}: largest count {K}, surfel top-K bound {bound}")


def test_surfel_tie_images(gs):
    ti = se.tie_images()
    v = {k: _t(ti[k]) for k in ("means2d", "ray_transforms", "colors", "opacities", "normals", "isect_offsets",
                                "flatten_ids")}
    v.update(W=se.IW, H=se.IH)
    bound = gs.ops._max_depth_samples(torch.device(DEV), SURFEL_BOUND)
    K, ids, w = _check_view(gs, v, (1, 3, bound))
    assert K == 5
    # the stop image: the fifth surfel brings next_T to 1e-4 exactly at the centre pixel and is not a pair there
    counts, _ = gs.rasterize_num_contributing_gaussians_2dgs(*_args(v))
    x, y = ti["centres"][2]
    last, _ = se.stop_chain_float32()
    assert int(counts[2, y, x]) == last + 1
    _check_oracle_weights(v, ids, w, min_checked=0.5)


def test_two_runs_identical(gs):
    v = _view(gs, 0, 2, n=10000, seed=1)
    first = [gs.rasterize_num_contributing_gaussians_2dgs(*_args(v))]
    first.append(gs.rasterize_contributing_gaussian_ids_2dgs(*_args(v), first[0][0]))
    first.append(gs.rasterize_top_contributing_gaussian_ids_2dgs(*_args(v), 8))
    again = [gs.rasterize_num_contributing_gaussians_2dgs(*_args(v))]
    again.append(gs.rasterize_contributing_gaussian_ids_2dgs(*_args(v), first[0][0]))
    again.append(gs.rasterize_top_contributing_gaussian_ids_2dgs(*_args(v), 8))
    for a, b in zip(first, again):
        assert all(torch.equal(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------
# the sparse forms: the dense queries gathered at the pixels
def _patches64(C):
    corners = [(0, 0), (96, 160), (136, 256)]  # the last one reaches the image's bottom-right corner
    a = np.array([(y0 + y, x0 + x, i) for i in range(C) for (y0, x0) in corners for y in range(64) for x in range(64)],
                 np.int64)
    return torch.from_numpy(a[:, :2].astype(np.int32)).to(DEV), torch.from_numpy(a[:, 2].astype(np.int32)).to(DEV)


def _sparse_equals_dense(gs, rows, pixels, image_ids, what):
    """the three sparse queries against the dense ones at the full tile grid (so that margin pixels exist)"""
    off, fl = s2._dense_lists(gs, rows)
    v = dict(rows, isect_offsets=off, flatten_ids=fl, W=W, H=GRID_H)
    counts, alphas = gs.rasterize_num_contributing_gaussians_2dgs(*_args(v))
    ids, w = gs.rasterize_contributing_gaussian_ids_2dgs(*_args(v), counts)
    layout, t_off, t_fl = s2._sparse_pipeline(gs, rows, pixels, image_ids)
    active, _, words, cum, pmap = layout
    rs = (rows["means2d"], rows["ray_transforms"], rows["opacities"])
    lay = (active, t_off, t_fl, words, cum, pmap)
    grid = (W, H, 16, TW, TH)
    gather = lambda t: s2._gather(t if t.dim() > counts.dim() else t[..., None], pixels, image_ids)  # noqa: E731
    s_counts, s_alphas = gs.rasterize_num_contributing_gaussians_2dgs_sparse(*rs, *lay, *grid)
    P = pixels.shape[0]
    assert s_counts.shape == (P,) and s_alphas.shape == (P,)
    assert torch.equal(s_counts, gather(counts)[:, 0]) and torch.equal(s_alphas, gather(alphas)[:, 0]), what
    s_ids, s_w = gs.rasterize_contributing_gaussian_ids_2dgs_sparse(*rs, *lay, s_counts, *grid)
    Ks = s_ids.shape[-1]
    assert s_ids.shape == (P, Ks) and Ks == (int(s_counts.max()) if P else 0)
    assert torch.equal(s_ids, gather(ids)[:, :Ks]) and torch.equal(s_w, gather(w)[:, :Ks]), what
    for k in (1, 8):
        ti, tw = gs.rasterize_top_contributing_gaussian_ids_2dgs(*_args(v), k)
        s_ti, s_tw = gs.rasterize_top_contributing_gaussian_ids_2dgs_sparse(*rs, *lay, *grid, k)
        assert s_ti.shape == (P, k) and torch.equal(s_ti, gather(ti)) and torch.equal(s_tw, gather(tw)), (what, k)
    return layout, t_off, s_counts


@pytest.mark.parametrize("C", [1, 2])
def test_sparse_equals_dense(gs, C):
    rows = s2._rows(gs, 0, C, 3)
    for kind in ("random", "patches64", "margin", "one"):
        pixels, image_ids = _patches64(C) if kind == "patches64" else _pixel_set(kind, C, np.random.RandomState(C))
        _sparse_equals_dense(gs, rows, pixels, image_ids, kind)


def test_sparse_batch_dimension(gs):
    rows = s2._rows(gs, 2, 2, 3, n=10000)
    pixels, image_ids = _pixel_set("random", 4, np.random.RandomState(7))
    _sparse_equals_dense(gs, rows, pixels, image_ids, "batch")


def test_sparse_active_tile_with_empty_list(gs):
    rows = s2._rows(gs, 0, 1, 3)
    t = 5 * TW + 7  # tile (7, 5): drop every surfel whose box reaches it
    offsets, fl = s2._dense_lists(gs, rows)
    off = np.concatenate([offsets.cpu().numpy().reshape(-1), [fl.shape[0]]])
    hit = torch.from_numpy(fl.cpu().numpy()[off[t]: off[t + 1]].astype(np.int64)).to(DEV)
    assert hit.numel() > 0
    radii = rows["radii"].clone()
    radii.view(-1, 2)[hit] = 0
    rows = dict(rows, radii=radii)
    pixels = torch.tensor([[5 * 16 + 3, 7 * 16 + 9], [5 * 16 + 15, 7 * 16], [10, 10]], device=DEV, dtype=torch.int32)
    image_ids = torch.zeros(3, device=DEV, dtype=torch.int32)
    layout, t_off, s_counts = _sparse_equals_dense(gs, rows, pixels, image_ids, "empty list")
    a = int(np.nonzero(layout[0].cpu().numpy() == t)[0][0])
    assert t_off[a] == t_off[a + 1]
    assert (s_counts[:2] == 0).all()


# ------------------------------------------------------------------------------------------
# empty inputs
def test_empty_inputs(gs):
    v = _view(gs, 0, 2, n=2000)
    m2, rt, op, off, fl = (v[k] for k in ("means2d", "ray_transforms", "opacities", "isect_offsets", "flatten_ids"))
    zoff = torch.zeros_like(off)
    cases = {
        "no lists": (m2, rt, op, zoff, fl[:0]),
        "N = 0": (m2[:, :0], rt[:, :0], op[:, :0], zoff, fl[:0]),
    }
    for name, a in cases.items():
        counts, alphas = gs.rasterize_num_contributing_gaussians_2dgs(*a, W, H, 16)
        assert counts.shape == (2, H, W) and (counts == 0).all() and (alphas == 0).all(), name
        ids, w = gs.rasterize_contributing_gaussian_ids_2dgs(*a, W, H, 16, counts)
        assert ids.shape == (2, H, W, 0) and w.shape == (2, H, W, 0), name
        ti, tw = gs.rasterize_top_contributing_gaussian_ids_2dgs(*a, W, H, 16, 3)
        assert ti.shape == (2, H, W, 3) and (ti == -1).all() and (tw == 0).all(), name
    # all-zero counts on a non-empty scene: ids [..., 0]
    ids, w = gs.rasterize_contributing_gaussian_ids_2dgs(*_args(v), torch.zeros((2, H, W), device=DEV, dtype=torch.int32))
    assert ids.shape == (2, H, W, 0) and w.shape == (2, H, W, 0)
    # a zero-sized image
    counts, alphas = gs.rasterize_num_contributing_gaussians_2dgs(m2, rt, op, off, fl, 0, H, 16)
    assert counts.shape == (2, H, 0) and alphas.shape == (2, H, 0)
    # no pixels, and no lists in any active tile
    rows = s2._rows(gs, 0, 1, 3, n=2000)
    rs = (rows["means2d"], rows["ray_transforms"], rows["opacities"])
    grid = (W, H, 16, TW, TH)
    for name, rws, kind in (("no pixels", rows, "empty"), ("no lists", dict(rows, radii=torch.zeros_like(rows["radii"])), "random")):
        pixels, image_ids = _pixel_set(kind, 1, np.random.RandomState(0))
        (active, _, words, cum, pmap), t_off, t_fl = s2._sparse_pipeline(gs, rws, pixels, image_ids)
        lay = (active, t_off, t_fl, words, cum, pmap)
        P = pixels.shape[0]
        s_counts, s_alphas = gs.rasterize_num_contributing_gaussians_2dgs_sparse(*rs, *lay, *grid)
        assert s_counts.shape == (P,) and (s_counts == 0).all() and (s_alphas == 0).all(), name
        s_ids, s_w = gs.rasterize_contributing_gaussian_ids_2dgs_sparse(*rs, *lay, s_counts, *grid)
        assert s_ids.shape == (P, 0) and s_w.shape == (P, 0), name
        s_ti, s_tw = gs.rasterize_top_contributing_gaussian_ids_2dgs_sparse(*rs, *lay, *grid, 4)
        assert s_ti.shape == (P, 4) and (s_ti == -1).all() and (s_tw == 0).all(), name
