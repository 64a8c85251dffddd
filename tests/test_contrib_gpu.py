"""The per-pixel contributor queries on the GPU: every output is the pair-query walk's, so each is checked against
rasterize_to_indices_in_range(0, inf, T = 1) and rasterize_to_pixels on the same inputs.

* Counts equal the per-pixel pair counts and alphas equal render_alphas bit for bit (garden view [2, 2] at 256 x 256,
  the tests/raster_edges.py sweep, one 1080p view).
* Padded ids are the pairs in order, -1 / 0 after them; a float64 accumulate of the weights reproduces the render.
* Counts that are too small keep the first K pairs of every pixel.
* Top-K equals a numpy model of the reference's rule applied to the padded lists.
* The _sparse forms equal the dense queries gathered at the pixels (320 x 200, one and two cameras, dense and packed).
* Empty inputs, and the reference's own ops (tests/golden/ref_contrib.npz, tests/golden/make_ref_contrib_golden.py).
"""
import math
import os

import numpy as np
import pytest
import torch

from tests import raster_edges as re_
from tests import scene
from tests import test_sparse_raster_gpu as sp
from tests.test_indices_gpu import _n, _pixel, _t, garden_view

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_contrib.npz")
EMPTY_POS = np.iinfo(np.int64).max


@pytest.fixture(scope="module")
def gs():
    import gsplat_b200

    assert torch.cuda.is_available(), "needs a GPU"
    return gsplat_b200


def _lists(gs, v):
    """the pairs of rasterize_to_indices_in_range(0, inf, T = 1): (gaussian ids, flat pixel index, rank in the pixel)"""
    W, H = v["W"], v["H"]
    dims = tuple(v["isect_offsets"].shape[:-2])
    ones = torch.ones(dims + (H, W), device=DEV)
    ids = gs.rasterize_to_indices_in_range(0, 10**10, ones, v["means2d"], v["conics"], v["opacities"], W, H, 16,
                                           v["isect_offsets"], v["flatten_ids"])
    g, lin = _pixel(ids, H, W)
    first = np.r_[True, lin[1:] != lin[:-1]] if len(lin) else np.zeros(0, bool)
    start = np.maximum.accumulate(np.where(first, np.arange(len(lin)), 0)) if len(lin) else lin
    return g, lin, np.arange(len(lin)) - start


def _args(v):
    return (v["means2d"], v["conics"], v["opacities"], v["isect_offsets"], v["flatten_ids"], v["W"], v["H"], 16)


def top_model(ids, weights, K):
    """The reference's top-K rule over padded lists ids / weights [P, L] (id -1 = no pair): K slots of (id, weight,
    position) start as (-1, 0, +inf); a pair replaces the first lowest-weight slot only when strictly heavier; the slots
    are then sorted by position (stable)."""
    P, L = ids.shape
    s_id = np.full((P, K), -1, np.int32)
    s_w = np.zeros((P, K), np.float32)
    s_pos = np.full((P, K), EMPTY_POS, np.int64)
    rows = np.arange(P)
    for k in range(L):
        live = ids[:, k] >= 0
        m = np.argmin(s_w, axis=1)  # the first minimum
        take = live & (weights[:, k] > s_w[rows, m])
        r, mm = rows[take], m[take]
        s_id[r, mm], s_w[r, mm], s_pos[r, mm] = ids[take, k], weights[take, k], k
    order = np.argsort(s_pos, axis=1, kind="stable")
    return np.take_along_axis(s_id, order, 1), np.take_along_axis(s_w, order, 1)


def _check_view(gs, v, colors, top_ks, n_model=None, seed=0):
    """checks 1-4 on one dense view (on the device where the arrays are large); returns the largest count"""
    W, H = v["W"], v["H"]
    dims = tuple(v["isect_offsets"].shape[:-2])
    P = int(np.prod(dims)) * H * W
    g, lin, rank = _lists(gs, v)
    g_t, lin_t, rank_t = (torch.from_numpy(x).to(DEV) for x in (g, lin, rank))
    # 1. counts and alphas
    counts, alphas = gs.rasterize_num_contributing_gaussians(*_args(v))
    assert counts.dtype == torch.int32 and counts.shape == dims + (H, W) and alphas.shape == dims + (H, W)
    assert np.array_equal(_n(counts).reshape(-1), np.bincount(lin, minlength=P)), "counts differ from the pair counts"
    rc, ra = gs.rasterize_to_pixels(v["means2d"], v["conics"], colors, v["opacities"], W, H, 16, v["isect_offsets"], v["flatten_ids"])
    bad = int((alphas != ra[..., 0]).sum())
    assert bad == 0, f"{bad} alphas differ from render_alphas"
    # 2. padded ids: the pairs in order, then -1 / 0
    ids, w = gs.rasterize_contributing_gaussian_ids(*_args(v), counts)
    K = int(counts.max()) if P else 0
    assert ids.dtype == torch.int32 and w.dtype == torch.float32 and ids.shape == dims + (H, W, K)
    want = torch.full((P, K), -1, device=DEV, dtype=torch.int32)
    want[lin_t, rank_t] = g_t.to(torch.int32)
    ids2, w2 = ids.reshape(P, K), w.reshape(P, K)
    assert torch.equal(ids2, want), f"{int((ids2 != want).sum())} ids differ from the pairs"
    assert bool((w2[want < 0] == 0).all()) and bool((w2[want >= 0] > 0).all())
    N = v["means2d"].shape[-2]
    rows = g_t + (lin_t // (H * W)) * N
    wp = w2[lin_t, rank_t].double()
    col = colors.reshape(-1, colors.shape[-1]).double()[rows]
    c64 = torch.zeros((P, col.shape[1]), device=DEV, dtype=torch.float64).index_add_(0, lin_t, wp[:, None] * col)
    a64 = torch.zeros(P, device=DEV, dtype=torch.float64).index_add_(0, lin_t, wp)
    assert float((c64 - rc.reshape(P, -1).double()).abs().max()) < 1e-4
    assert float((a64 - ra.reshape(-1).double()).abs().max()) < 1e-4
    # 3. counts too small: every pixel keeps its first pairs, nothing lands outside its row
    for cap in (1, max(K // 3, 1)):
        short = torch.clamp(counts, max=cap)
        short.view(-1)[0] = cap
        ids_s, w_s = gs.rasterize_contributing_gaussian_ids(*_args(v), short)
        assert torch.equal(ids_s, ids[..., :cap]) and torch.equal(w_s, w[..., :cap])
    # 4. top-K against the model of the reference's rule
    rng = np.random.RandomState(seed)
    sel = np.arange(P) if n_model is None or n_model >= P else np.sort(rng.choice(P, n_model, replace=False))
    sel_t = torch.from_numpy(sel).to(DEV)
    ids_n, w_n = _n(ids2[sel_t]), _n(w2[sel_t])
    for k in top_ks:
        top_i, top_w = gs.rasterize_top_contributing_gaussian_ids(*_args(v), k)
        assert top_i.shape == dims + (H, W, k) and top_w.shape == dims + (H, W, k)
        mi, mw = top_model(ids_n, w_n, k)
        ti, tw = _n(top_i.reshape(P, k)[sel_t]), _n(top_w.reshape(P, k)[sel_t])
        assert np.array_equal(ti, mi) and np.array_equal(tw, mw), f"K = {k}: {int((ti != mi).any(1).sum())} pixels differ from the model"
        if k >= K:
            pad = (0, k - K)
            assert torch.equal(top_i.reshape(P, k), torch.nn.functional.pad(ids2, pad, value=-1))
            assert torch.equal(top_w.reshape(P, k), torch.nn.functional.pad(w2, pad))
    return K


def test_garden_view(gs):
    v = garden_view(gs)
    bound = gs.ops._max_depth_samples(torch.device(DEV))
    assert bound >= 32
    _check_view(gs, v, v["colors"], (1, 3, 16, bound), n_model=20000)
    with pytest.raises(ValueError):
        gs.rasterize_top_contributing_gaussian_ids(*_args(v), bound + 1)


def test_raster_sweep(gs):
    sw = re_.make_sweep()
    v = {k: _t(sw[k]) for k in ("means2d", "conics", "opacities", "isect_offsets", "flatten_ids")}
    v.update(W=re_.W, H=re_.H)
    K = _check_view(gs, v, _t(sw["colors3"]), (1, 3))
    _check_view(gs, v, _t(sw["colors3"]), (K, K + 2))


def test_1080p_view(gs):
    v = garden_view(gs, W=1920, H=1080, batch=(1, 1), n_max=100000)
    _check_view(gs, v, v["colors"], (8,), n_model=20000)


# ------------------------------------------------------------------------------------------
# 5. sparse forms: the dense queries gathered at the pixels
@pytest.mark.parametrize("packed", [False, True], ids=["dense", "packed"])
@pytest.mark.parametrize("C", [1, 2])
def test_sparse_equals_dense(gs, C, packed):
    garden = (scene.make_scene(n_max=30000, sh_degree=0),)
    garden = (garden[0], scene.rescale_K(garden[0]["Ks"], garden[0]["width"], garden[0]["height"], sp.W, sp.H))
    rows = sp._project(gs, garden, C, packed)
    off, fl = sp._dense_lists(gs, rows, C)
    rs = (rows["means2d"], rows["conics"], rows["opacities"])
    dense = (*rs, off, fl, sp.W, sp.H, 16)
    counts, alphas = gs.rasterize_num_contributing_gaussians(*dense)
    ids, w = gs.rasterize_contributing_gaussian_ids(*dense, counts)
    tops = {k: gs.rasterize_top_contributing_gaussian_ids(*dense, k) for k in (1, 8)}
    for kind in ("random", "patches", "one"):
        pixels, image_ids = sp._pixel_set(kind, C, np.random.RandomState(C))
        layout, t_off, t_fl = sp._sparse_pipeline(gs, rows, pixels, image_ids, C)
        active, _, words, cum, pmap = layout
        lay = (active, t_off, t_fl, words, cum, pmap)
        grid = (sp.W, sp.H, 16, sp.TW, sp.TH)
        gather = lambda t: t.reshape((C,) + t.shape[-3 if t.dim() > 3 else -2:])[image_ids.long(), pixels[:, 0].long(), pixels[:, 1].long()]  # noqa: E731
        s_counts, s_alphas = gs.rasterize_num_contributing_gaussians_sparse(*rs, *lay, *grid)
        assert torch.equal(s_counts, gather(counts)) and torch.equal(s_alphas, gather(alphas)), kind
        s_ids, s_w = gs.rasterize_contributing_gaussian_ids_sparse(*rs, *lay, s_counts, *grid)
        Ks = s_ids.shape[-1]
        assert Ks == (int(s_counts.max()) if len(s_counts) else 0)
        assert torch.equal(s_ids, gather(ids)[:, :Ks]) and torch.equal(s_w, gather(w)[:, :Ks]), kind
        for k, (ti, tw) in tops.items():
            s_ti, s_tw = gs.rasterize_top_contributing_gaussian_ids_sparse(*rs, *lay, *grid, k)
            assert torch.equal(s_ti, gather(ti)) and torch.equal(s_tw, gather(tw)), (kind, k)
    if packed:
        # packed ids index the nnz rows; through gaussian_ids they are the dense projection's ids
        sc = garden[0]
        tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
        gid = gs.fully_fused_projection(tt(sc["means"]), None, tt(sc["quats"]), tt(sc["scales"]), tt(sc["viewmats"][:C]),
                                        tt(garden[1][:C]), sp.W, sp.H, packed=True)[2]
        d_rows = sp._project(gs, garden, C, False)
        d_off, d_fl = sp._dense_lists(gs, d_rows, C)
        d_counts, _ = gs.rasterize_num_contributing_gaussians(d_rows["means2d"], d_rows["conics"], d_rows["opacities"], d_off,
                                                              d_fl, sp.W, sp.H, 16)
        d_ids, _ = gs.rasterize_contributing_gaussian_ids(d_rows["means2d"], d_rows["conics"], d_rows["opacities"], d_off, d_fl,
                                                          sp.W, sp.H, 16, d_counts)
        mapped = torch.where(ids >= 0, gid.to(torch.int32)[ids.clamp(min=0).long()], ids)
        assert torch.equal(mapped, d_ids)


# ------------------------------------------------------------------------------------------
# 6. empty inputs
def test_empty_inputs(gs):
    v = garden_view(gs, W=64, H=48, batch=(1, 2), n_max=2000)
    W, H = v["W"], v["H"]
    m2, con, op, off, fl = (v[k] for k in ("means2d", "conics", "opacities", "isect_offsets", "flatten_ids"))
    zoff = torch.zeros_like(off)
    cases = {
        "no lists": (m2, con, op, zoff, fl[:0]),
        "N = 0": (m2[:, :, :0], con[:, :, :0], op[:, :, :0], zoff, fl[:0]),
        "nnz = 0": (m2.reshape(-1, 2)[:0], con.reshape(-1, 3)[:0], op.reshape(-1)[:0], zoff, fl[:0]),
    }
    for name, a in cases.items():
        counts, alphas = gs.rasterize_num_contributing_gaussians(*a, W, H, 16)
        assert counts.shape == (1, 2, H, W) and (counts == 0).all() and (alphas == 0).all(), name
        ids, w = gs.rasterize_contributing_gaussian_ids(*a, W, H, 16, counts)
        assert ids.shape == (1, 2, H, W, 0) and w.shape == (1, 2, H, W, 0), name
        ti, tw = gs.rasterize_top_contributing_gaussian_ids(*a, W, H, 16, 3)
        assert (ti == -1).all() and (tw == 0).all(), name
    # all-zero counts on a non-empty scene: ids [..., 0]
    ids, w = gs.rasterize_contributing_gaussian_ids(*_args(v), torch.zeros((1, 2, H, W), device=DEV, dtype=torch.int32))
    assert ids.shape == (1, 2, H, W, 0) and w.shape == (1, 2, H, W, 0)
    # a zero-sized image
    counts, alphas = gs.rasterize_num_contributing_gaussians(m2, con, op, off, fl, 0, H, 16)
    assert counts.shape == (1, 2, H, 0)


# ------------------------------------------------------------------------------------------
# 7. the reference's own ops
def _explained(d, p, a, b, T_ULP=2.0**-24):
    """pixel p's lists a (ours) and b (the reference's) differ only at pairs within the float32 budget of a threshold
    decision (the 1/255 cull or the 1e-4 stop), as test_indices_gpu.test_matches_reference_op decides it"""
    from tests.test_indices_gpu import T_TH, _alpha3

    W, H = int(d["W"]), int(d["H"])
    m2, con, op = d["means2d"].reshape(-1, 2), d["conics"].reshape(-1, 3), d["opacities"].reshape(-1)
    N = d["means2d"].shape[-2]
    img = p // (H * W)

    def alpha_of(gg):
        return _alpha3(m2, con, op, np.array([img * N + gg]), np.array([p]), H, W)

    def near(gg):
        al, sig, dsig, dl = (float(x[0]) for x in alpha_of(gg))
        lx = math.log(float(op[img * N + gg])) - sig if op[img * N + gg] > 0 else -math.inf
        return abs(sig) <= dsig or abs(lx - math.log(re_.ALPHA_TH)) <= dl

    a2, b2 = [x for x in a if not near(x)], [x for x in b if not near(x)]
    short, long_ = (a2, b2) if len(a2) <= len(b2) else (b2, a2)
    if long_[:len(short)] != short:
        return False
    if len(long_) == len(short):
        return True
    for walk in (a, b):
        T, rel = 1.0, 0.0
        for x in walk:
            if x == long_[len(short)]:
                break
            al = float(alpha_of(x)[0][0])
            T *= 1.0 - al
            rel += al * math.expm1(float(alpha_of(x)[3][0])) / (1.0 - al) + 2 * T_ULP
        nT = T * (1.0 - float(alpha_of(long_[len(short)])[0][0]))
        if abs(nT - T_TH) <= T_TH * (1e-5 + rel):
            return True
    return False


def test_matches_reference_ops(gs):
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/ref_contrib.npz not recorded")
    d = np.load(GOLDEN)
    W, H = int(d["W"]), int(d["H"])
    v = dict(means2d=_t(d["means2d"]), conics=_t(d["conics"]), opacities=_t(d["opacities"]),
             isect_offsets=_t(d["isect_offsets"]), flatten_ids=_t(d["flatten_ids"]), W=W, H=H)
    counts, alphas = gs.rasterize_num_contributing_gaussians(*_args(v))
    ids, w = gs.rasterize_contributing_gaussian_ids(*_args(v), counts)
    P, K = int(np.prod(counts.shape)), ids.shape[-1]
    ours_c, ids_n, w_n = _n(counts).reshape(-1), _n(ids).reshape(P, K), _n(w).reshape(P, K)
    ref_c = d["counts"].astype(np.int64).reshape(-1)
    ref_g, ref_w = d["ids"].astype(np.int64), d["weights"]
    rs = np.r_[0, np.cumsum(ref_c)]
    diff = []
    same = ours_c == ref_c
    ref_pad = np.full((P, max(K, int(ref_c.max()))), -1, np.int64)
    rank = np.arange(len(ref_g)) - np.repeat(rs[:-1], ref_c)
    ref_pad[np.repeat(np.arange(P), ref_c), rank] = ref_g
    ours_pad = np.full_like(ref_pad, -1)
    ours_pad[:, :K] = ids_n
    same &= (ours_pad == ref_pad).all(1)
    for p in np.nonzero(~same)[0]:
        a, b = [int(x) for x in ids_n[p, :ours_c[p]]], [int(x) for x in ref_g[rs[p]:rs[p + 1]]]
        if not _explained(d, p, a, b):
            diff.append(p)
    assert not diff, f"{len(diff)} pixels differ from the reference's ops unexplained, e.g. {diff[:5]}"
    # where the lists agree, the alphas and weights agree to float32 rounding of the two exponentials
    ref_wpad = np.zeros(ref_pad.shape, np.float32)
    ref_wpad[np.repeat(np.arange(P), ref_c), rank] = ref_w
    assert np.abs(_n(alphas).reshape(-1)[same] - d["alphas"].reshape(-1)[same]).max() < 1e-5
    assert np.abs(w_n[same] - ref_wpad[same, :K]).max() < 1e-5
    # the reference's own top-K output is the model of its rule applied to its own lists
    k = d["top_ids"].shape[-1]
    mi, mw = top_model(np.where(ref_pad >= 0, ref_pad, -1).astype(np.int32), ref_wpad, k)
    assert np.array_equal(mi, d["top_ids"].reshape(P, k).astype(np.int32)) and np.array_equal(mw, d["top_weights"].reshape(P, k))
    print(f"\nreference ops: {P} pixels, {int((~same).sum())} differ (all at threshold decisions)")
