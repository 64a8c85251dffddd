"""rasterize_to_indices_in_range / _2dgs on the GPU: the pairs are the compositing forward's own.

* The garden view (3DGS, batch dims [2, 2], 256 x 256, T = 1): the last pair of every pixel is the forward's last_ids,
  the pixels with pairs are those with render_alphas > 0, and a float64 accumulate over the pairs reproduces the
  render; the same for 2DGS against rasterize_to_pixels_2dgs.
* The adversarial sweeps of tests/raster_edges.py and tests/surfel_edges.py: the pixel set of every gaussian is the
  forward's, and the float64 truth's wherever the truth is decided.
* Ranges: per-batch calls add up to the full call on a scene that never saturates; empty and clamped ranges.
* Given transmittances: per-pixel counts against a float64 walk outside the float32 budget of its decisions.
* The reference's own op (tests/golden/ref_indices.npz, recorded by tests/golden/make_ref_indices_golden.py).
"""
import math
import os

import numpy as np
import pytest
import torch

from oracle import surfel
from tests import raster_edges as re_
from tests import scene
from tests import surfel_edges as se
from tests.golden import make_ref_indices_golden as make_ref

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_indices.npz")
ULP = 2.0**-24
T_TH = float(np.float32(1e-4))


@pytest.fixture(scope="module")
def gs():
    import gsplat_b200

    assert torch.cuda.is_available(), "needs a GPU"
    return gsplat_b200


def _t(a):
    return torch.from_numpy(np.array(a, order="C")).to(DEV)


def _n(t):
    return t.detach().cpu().numpy()


def garden_view(gs, W=256, H=256, batch=(2, 2), n_max=30000, seed=42):
    """The garden crop projected into batch[-1] cameras for batch[0] copies of the scene (the second moved along x),
    intersected with the ellipse test: dict of float32 / int32 tensors with image dims `batch`."""
    sc = scene.make_scene(n_max=n_max, seed=seed)
    B, C = batch
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:C]
    shift = np.arange(B, dtype=np.float32)[:, None, None] * np.array([0.3, 0.0, 0.0], np.float32)
    means = sc["means"][None] + shift
    rep = lambda a: np.ascontiguousarray(np.broadcast_to(a[None], (B,) + a.shape))  # noqa: E731
    radii, m2, dep, con, _ = gs.fully_fused_projection(
        _t(means), None, _t(rep(sc["quats"])), _t(rep(sc["scales"])), _t(rep(sc["viewmats"][:C])), _t(rep(Ks)), W, H)
    op = _t(np.ascontiguousarray(np.broadcast_to(sc["opacities"], (B, C, len(sc["opacities"])))))
    tw, th = math.ceil(W / 16), math.ceil(H / 16)
    _, isect_ids, fl = gs.isect_tiles(m2, radii, dep, 16, tw, th, conics=con, opacities=op)
    off = gs.isect_offset_encode(isect_ids, B * C, tw, th).reshape(B, C, th, tw)
    colors = _t(np.ascontiguousarray(np.broadcast_to(sc["colors"], (B, C) + sc["colors"].shape)))
    return dict(means2d=m2, conics=con, opacities=op, colors=colors, isect_offsets=off, flatten_ids=fl, W=W, H=H)


def _pixel(ids, H, W):
    g, p, i = (_n(x) for x in ids)
    return g, i.astype(np.int64) * H * W + p


def _accumulate(lin, alpha, colors, n_pix):
    """float64 front-to-back compositing of pairs sorted by pixel: (colour [n_pix, D], alpha [n_pix])"""
    la = np.log1p(-alpha)
    cum = np.cumsum(la)
    first = np.r_[True, lin[1:] != lin[:-1]]
    start = np.maximum.accumulate(np.where(first, np.arange(len(lin)), 0))
    excl = cum - la - (cum[start] - la[start])  # sum of log(1 - alpha) of the pixel's earlier pairs
    w = alpha * np.exp(excl)
    col = np.zeros((n_pix, colors.shape[-1]))
    for k in range(colors.shape[-1]):
        col[:, k] = np.bincount(lin, w * colors[:, k], minlength=n_pix)
    T = np.exp(np.bincount(lin, la, minlength=n_pix))
    return col, 1.0 - T


def _alpha3(m2, con, op, g, lin, H, W):
    """float64 alpha of 3DGS pairs (g: flat row index into [I * N]) at pixel lin, with its budget: (alpha_c, sigma,
    dsig, dl) as in tests/raster_edges.py"""
    px = (lin % W).astype(np.float64) + 0.5
    py = ((lin // W) % H).astype(np.float64) + 0.5
    dx, dy = m2[g, 0].astype(np.float64) - px, m2[g, 1].astype(np.float64) - py
    a, b, c = (con[g, k].astype(np.float64) for k in range(3))
    o = op[g].astype(np.float64)
    with np.errstate(all="ignore"):
        sigma = 0.5 * (a * dx * dx + c * dy * dy) + b * dx * dy
        S = 0.5 * (np.abs(a) * dx * dx + np.abs(c) * dy * dy) + np.abs(b * dx * dy)
        alpha_c = np.minimum(re_.MAX_ALPHA, o * np.exp(-sigma))
    dsig = 16.0 * ULP * S
    return alpha_c, sigma, dsig, dsig + 32.0 * ULP


# ------------------------------------------------------------------------------------------
# 1. the forward's decisions
def test_garden_pairs_are_the_forward_pairs(gs):
    from gsplat_b200._cabi import lib, ptr, stream

    v = garden_view(gs)
    W, H = v["W"], v["H"]
    m2, con, op, col, off, fl = (v[k] for k in ("means2d", "conics", "opacities", "colors", "isect_offsets", "flatten_ids"))
    I, N = 4, m2.shape[-2]
    rc, ra = gs.rasterize_to_pixels(m2, con, col, op, W, H, 16, off, fl)
    # last_ids straight from the forward's C ABI
    S = fl.shape[0]
    records = torch.empty(lib().gsb200_raster_records_bytes(S, 3, I * 16 * 16), device=DEV, dtype=torch.uint8)
    rc2, ra2 = torch.empty_like(rc), torch.empty_like(ra)
    last_ids = torch.empty((2, 2, H, W), device=DEV, dtype=torch.int32)
    assert lib().gsb200_raster_fwd(I, N, 3, ptr(m2), ptr(con), ptr(col), ptr(op), None, None, W, H, 16, 16, 16, ptr(off), ptr(fl),
                                   S, ptr(records), ptr(rc2), ptr(ra2), ptr(last_ids), stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(rc, rc2) and torch.equal(ra, ra2)

    ids = gs.rasterize_to_indices_in_range(0, 10**10, torch.ones((2, 2, H, W), device=DEV), m2, con, op, W, H, 16, off, fl)
    g, lin = _pixel(ids, H, W)
    assert len(g) > 100000 and (np.diff(lin) >= 0).all(), "pixel-major order"
    alive = _n(ra).reshape(-1) > 0
    has = np.zeros(I * H * W, bool)
    has[lin] = True
    assert np.array_equal(has, alive), f"{int((has != alive).sum())} pixels differ between pairs and render_alphas > 0"
    last = np.r_[lin[1:] != lin[:-1], True]
    want = _n(fl)[_n(last_ids).reshape(-1)[lin[last]]] % N
    assert np.array_equal(g[last], want), f"{int((g[last] != want).sum())} pixels end on another gaussian than last_ids"

    rows = g + (lin // (H * W)) * N
    alpha, *_ = _alpha3(_n(m2).reshape(-1, 2), _n(con).reshape(-1, 3), _n(op).reshape(-1), rows, lin, H, W)
    c64, a64 = _accumulate(lin, alpha, _n(col).reshape(-1, 3)[rows], I * H * W)
    assert np.abs(c64 - _n(rc).reshape(-1, 3)).max() < 1e-4
    assert np.abs(a64 - _n(ra).reshape(-1)).max() < 1e-4


def _surfel_alpha(m2, rt, op, g, lin, H, W):
    px = (lin % W).astype(np.float64) + 0.5
    py = ((lin // W) % H).astype(np.float64) + 0.5
    M = rt[g].astype(np.float64).reshape(-1, 3, 3)
    hu = px[:, None] * M[:, 2] - M[:, 0]
    hv = py[:, None] * M[:, 2] - M[:, 1]
    s = np.cross(hu, hv)
    with np.errstate(all="ignore"):
        u, w = s[:, 0] / s[:, 2], s[:, 1] / s[:, 2]
        g3 = u * u + w * w
        g2 = 2.0 * ((m2[g, 0] - px) ** 2 + (m2[g, 1] - py) ** 2)
        return np.minimum(re_.MAX_ALPHA, op[g].astype(np.float64) * np.exp(-0.5 * np.minimum(g3, g2)))


def test_garden_pairs_are_the_2dgs_forward_pairs(gs):
    sc = scene.make_scene(n_max=20000)
    W = H = 256
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:2]
    radii, m2, dep, rt, nrm = gs.fully_fused_projection_2dgs(
        _t(sc["means"]), _t(sc["quats"]), _t(sc["scales"] * 2), _t(sc["viewmats"][:2]), _t(Ks), W, H)
    tw = th = 16
    _, isect_ids, fl = gs.isect_tiles(m2, radii, dep, 16, tw, th)
    off = gs.isect_offset_encode(isect_ids, 2, tw, th)
    N = m2.shape[-2]
    op = _t(np.ascontiguousarray(np.broadcast_to(sc["opacities"], (2, N))))
    col = _t(np.ascontiguousarray(np.broadcast_to(sc["colors"], (2, N, 3))))
    rc, ra, *_ = gs.rasterize_to_pixels_2dgs(m2, rt, col, op, nrm, torch.zeros_like(m2), W, H, 16, off, fl)
    ids = gs.rasterize_to_indices_in_range_2dgs(0, 2**30, torch.ones((2, H, W), device=DEV), m2, rt, op, W, H, 16, off, fl)
    g, lin = _pixel(ids, H, W)
    assert len(g) > 50000 and (np.diff(lin) >= 0).all()
    has = np.zeros(2 * H * W, bool)
    has[lin] = True
    alive = _n(ra).reshape(-1) > 0
    assert np.array_equal(has, alive), f"{int((has != alive).sum())} pixels differ between pairs and render_alphas > 0"
    rows = g + (lin // (H * W)) * N
    alpha = _surfel_alpha(_n(m2).reshape(-1, 2).astype(np.float64), _n(rt).reshape(-1, 9), _n(op).reshape(-1), rows, lin, H, W)
    c64, a64 = _accumulate(lin, alpha, _n(col).reshape(-1, 3)[rows], 2 * H * W)
    assert np.abs(c64 - _n(rc).reshape(-1, 3)).max() < 1e-4
    assert np.abs(a64 - _n(ra).reshape(-1)).max() < 1e-4


# ------------------------------------------------------------------------------------------
# 2. threshold sweeps
def test_raster_sweep_pixel_sets(gs):
    sw = re_.make_sweep()
    tr = re_.truth(sw)
    W, H = re_.W, re_.H
    m2, con, op = _t(sw["means2d"]), _t(sw["conics"]), _t(sw["opacities"])
    off, fl = _t(sw["isect_offsets"]), _t(sw["flatten_ids"])
    I = sw["means2d"].shape[0]
    _, ra = gs.rasterize_to_pixels(m2, con, _t(sw["colors3"]), op, W, H, 16, off, fl)
    ids = gs.rasterize_to_indices_in_range(0, 1, torch.ones((I, H, W), device=DEV), m2, con, op, W, H, 16, off, fl)
    g, lin = _pixel(ids, H, W)
    assert (g == 0).all() and len(np.unique(lin)) == len(lin)
    has = np.zeros(I * H * W, bool)
    has[lin] = True
    fwd = _n(ra).reshape(-1) > 0
    assert np.array_equal(has, fwd), f"{int((has != fwd).sum())} pixels differ from the forward"
    dec = tr["decided"].reshape(-1)
    truth = tr["alpha"].reshape(-1) > 0
    bad = dec & (has != truth)
    assert not bad.any(), f"{int(bad.sum())} decided pixels differ from the float64 truth"
    print(f"\nraster sweep: {I} gaussians, {len(lin)} pairs, {int((~dec).sum())} undecided pixels")


def test_surfel_sweep_pixel_sets(gs):
    ti = se.tie_images()
    W, H = se.IW, se.IH
    I = ti["means2d"].shape[0]
    t = {k: _t(ti[k]) for k in ("means2d", "ray_transforms", "colors", "opacities", "normals", "isect_offsets", "flatten_ids")}
    _, ra, *_ = gs.rasterize_to_pixels_2dgs(t["means2d"], t["ray_transforms"], t["colors"], t["opacities"], t["normals"],
                                            torch.zeros_like(t["means2d"]), W, H, 16, t["isect_offsets"], t["flatten_ids"])
    ids = gs.rasterize_to_indices_in_range_2dgs(0, 1, torch.ones((I, H, W), device=DEV), t["means2d"], t["ray_transforms"],
                                                t["opacities"], W, H, 16, t["isect_offsets"], t["flatten_ids"])
    g, lin = _pixel(ids, H, W)
    has = np.zeros(I * H * W, bool)
    has[lin] = True
    fwd = _n(ra).reshape(-1) > 0
    assert np.array_equal(has, fwd), f"{int((has != fwd).sum())} pixels differ from the forward"
    f64 = torch.float64
    ref = surfel.rasterize(*(torch.tensor(ti[k], dtype=f64) for k in ("means2d", "ray_transforms", "colors", "opacities", "normals")),
                           W, H, 16, ti["isect_offsets"], ti["flatten_ids"])
    truth = ref["render_alphas"].numpy().reshape(-1) > 0
    assert np.array_equal(has, truth), f"{int((has != truth).sum())} pixels differ from the float64 truth"
    # the stop image: the fifth surfel brings next_T to 1e-4 exactly and is not a pair
    x, y = ti["centres"][2]
    last, _ = se.stop_chain_float32()
    assert int((lin == (2 * H + y) * W + x).sum()) == last + 1


# ------------------------------------------------------------------------------------------
# 3. ranges
def _faint_scene(I=2, N=700, W=40, H=36, seed=3):
    """N faint isotropic gaussians per image (opacity <= 0.02: T never falls near 1e-4), every one listed on every
    tile in index order, so that each tile's list spans ceil(N / 256) batches"""
    rng = np.random.RandomState(seed)
    m2 = np.stack([rng.uniform(0, W, (I, N)), rng.uniform(0, H, (I, N))], -1).astype(np.float32)
    s2 = rng.uniform(2.0, 40.0, (I, N))
    con = np.stack([1.0 / s2, rng.uniform(-0.1, 0.1, (I, N)) / s2, 1.0 / s2], -1).astype(np.float32)
    op = rng.uniform(0.004, 0.02, (I, N)).astype(np.float32)
    tw, th = math.ceil(W / 16), math.ceil(H / 16)
    fl = np.concatenate([np.arange(N, dtype=np.int32) + i * N for i in range(I) for _ in range(tw * th)])
    off = (np.arange(I * th * tw, dtype=np.int32) * N).reshape(I, th, tw)
    return dict(means2d=m2, conics=con, opacities=op, isect_offsets=off, flatten_ids=fl, W=W, H=H)


def test_batches_add_up_to_the_full_range(gs):
    f = _faint_scene()
    W, H, I = f["W"], f["H"], 2
    args = [_t(f[k]) for k in ("means2d", "conics", "opacities")] + [W, H, 16] + [_t(f[k]) for k in ("isect_offsets", "flatten_ids")]
    ones = torch.ones((I, H, W), device=DEV)
    full = [_n(x) for x in gs.rasterize_to_indices_in_range(0, 10**10, ones, *args)]
    n_b = math.ceil(700 / 256)
    parts = [[_n(x) for x in gs.rasterize_to_indices_in_range(k, k + 1, ones, *args)] for k in range(n_b)]
    cat = [np.concatenate([p[j] for p in parts]) for j in range(3)]
    lin = cat[2] * H * W + cat[1]
    order = np.argsort(lin, kind="stable")
    for j in range(3):
        assert np.array_equal(cat[j][order], full[j])
    assert all(len(p[0]) > 0 for p in parts) and len(full[0]) > 100000
    for k in (n_b, n_b + 5, 2**40):
        assert all(len(x) == 0 for x in gs.rasterize_to_indices_in_range(k, k + 3, ones, *args))
    assert all(len(x) == 0 for x in gs.rasterize_to_indices_in_range(2, 2, ones, *args))
    assert all(len(x) == 0 for x in gs.rasterize_to_indices_in_range(2, 1, ones, *args))
    for end in (2**30, 1e10):
        got = gs.rasterize_to_indices_in_range(1, end, ones, *args)
        want = gs.rasterize_to_indices_in_range(1, 10**10, ones, *args)
        assert all(torch.equal(a, b) for a, b in zip(got, want))


# ------------------------------------------------------------------------------------------
# 4. given transmittances against a float64 walk
def _walk64(m2, con, op, off, fl, T0, W, H, n_isects):
    """Per-pixel float64 walk of every tile's full list from T0 [I, H, W] (torch, float64 on the GPU): pair counts and
    whether every alpha and stop decision lies outside its float32 budget (decided)."""
    I, th, tw = off.shape
    n_tiles = I * th * tw
    starts = off.reshape(-1).long()
    ends = torch.cat([starts[1:], torch.tensor([n_isects], device=DEV)])
    lens = ends - starts
    Lmax = int(lens.max())
    tile = torch.arange(n_tiles, device=DEV)
    img, ty, tx = tile // (th * tw), (tile // tw) % th, tile % tw
    k = torch.arange(256, device=DEV)
    py, px = ty[:, None] * 16 + k[None] // 16, tx[:, None] * 16 + k[None] % 16
    inside = (py < H) & (px < W)
    lin = (img[:, None] * H + py.clamp(max=H - 1)) * W + px.clamp(max=W - 1)
    T = T0.reshape(-1)[lin].double()
    done = ~inside
    decided = torch.ones_like(done)
    relT = torch.zeros_like(T)  # relative budget of the float32 transmittance
    cnt = torch.zeros(T.shape, dtype=torch.int64, device=DEV)
    m2, con, op = m2.double(), con.double(), op.double()
    for l in range(Lmax):
        valid = (l < lens)[:, None]
        g = fl[(starts + l).clamp(max=n_isects - 1)].long()
        dx = m2[g, 0][:, None] - (px.double() + 0.5)
        dy = m2[g, 1][:, None] - (py.double() + 0.5)
        a, b, c = (con[g, j][:, None] for j in range(3))
        sigma = 0.5 * (a * dx * dx + c * dy * dy) + b * dx * dy
        S = 0.5 * (a.abs() * dx * dx + c.abs() * dy * dy) + (b * dx * dy).abs()
        o = op[g][:, None]
        alpha = torch.clamp(o * torch.exp(-sigma), max=re_.MAX_ALPHA)
        dsig = 16.0 * ULP * S
        dl = dsig + 32.0 * ULP
        lx = torch.log(o) - sigma
        keep = (sigma >= 0) & (alpha >= re_.ALPHA_TH)
        near = ((sigma.abs() <= dsig) & (S > 0)) | ((sigma >= -dsig) & ((lx - math.log(re_.ALPHA_TH)).abs() <= dl))
        live = valid & ~done
        decided &= ~(live & near)
        nT = T * (1.0 - alpha)
        beta = torch.expm1(dl)
        rel_after = relT + alpha * beta / (1.0 - alpha) + 2.0 * ULP
        take = live & keep
        decided &= ~(take & ((nT - T_TH).abs() <= T_TH * rel_after))
        stop = take & (nT <= T_TH)
        done |= stop
        go = take & ~stop
        cnt += go.long()
        T = torch.where(go, nT, T)
        relT = torch.where(go, rel_after, relT)
    out_cnt = torch.zeros(I * H * W, dtype=torch.int64, device=DEV)
    out_dec = torch.zeros(I * H * W, dtype=torch.bool, device=DEV)
    out_cnt[lin[inside]] = cnt[inside]
    out_dec[lin[inside]] = decided[inside]
    return _n(out_cnt), _n(out_dec)


def test_given_transmittances_vs_float64_walk(gs):
    v = garden_view(gs, batch=(1, 2))
    W, H = v["W"], v["H"]
    rng = np.random.RandomState(7)
    T0 = _t(np.exp(rng.uniform(math.log(1e-3), 0.0, (1, 2, H, W))).astype(np.float32))
    m2, con, op, off, fl = (v[k] for k in ("means2d", "conics", "opacities", "isect_offsets", "flatten_ids"))
    ids = gs.rasterize_to_indices_in_range(0, 10**10, T0, m2, con, op, W, H, 16, off, fl)
    _, lin = _pixel(ids, H, W)
    got = np.bincount(lin, minlength=2 * H * W)
    want, dec = _walk64(m2.reshape(-1, 2), con.reshape(-1, 3), op.reshape(-1), off.reshape(2, 16, 16), fl, T0, W, H, fl.shape[0])
    bad = dec & (got != want)
    assert dec.mean() > 0.9, f"only {dec.mean():.1%} of the pixels decided"
    assert not bad.any(), f"{int(bad.sum())} decided pixels with another pair count than the float64 walk"
    print(f"\ngiven T: {len(lin)} pairs, {dec.mean():.2%} of the pixels decided")


# ------------------------------------------------------------------------------------------
# 5. the reference's op
def test_matches_reference_op(gs):
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/ref_indices.npz not recorded")
    d = np.load(GOLDEN)
    W, H = int(d["W"]), int(d["H"])
    m2, con, op = d["means2d"], d["conics"], d["opacities"]
    I, N = m2.shape[:2]
    args = [_t(m2), _t(con), _t(op), W, H, 16, _t(d["isect_offsets"]), _t(d["flatten_ids"])]
    m2f, conf, opf = m2.reshape(-1, 2), con.reshape(-1, 3), op.reshape(-1)
    report = {}
    for case in [str(c) for c in d["cases"]]:
        rs, re_end = (int(x) for x in d[f"{case}/range"])
        T0 = make_ref.transmittances(int(d[f"{case}/t_seed"]), (I, H, W))
        ids = gs.rasterize_to_indices_in_range(rs, re_end, _t(T0), *args)
        g, lin = _pixel(ids, H, W)
        rg, rcnt = d[f"{case}/gaussian_ids"].astype(np.int64), d[f"{case}/counts"].astype(np.int64)
        rlin = np.repeat(np.arange(len(rcnt)), rcnt)
        ours = np.bincount(lin, minlength=len(rcnt))
        diff_pix = np.nonzero((ours != rcnt) | (np.bincount(lin, g + 1, minlength=len(rcnt)) != np.bincount(rlin, rg + 1, minlength=len(rcnt))))[0]
        so, sr = np.r_[0, np.cumsum(ours)], np.r_[0, np.cumsum(rcnt)]
        unexplained, n_pairs = [], 0
        for p in diff_pix:
            a, b = list(g[so[p]:so[p + 1]]), list(rg[sr[p]:sr[p + 1]])
            sym = set(a) ^ set(b)
            n_pairs += len(sym)
            img = p // (H * W)

            def alpha_of(gg):
                return _alpha3(m2f, conf, opf, np.array([img * N + gg]), np.array([p]), H, W)

            def near_threshold(gg):
                al, sig, dsig, dl = (float(x[0]) for x in alpha_of(gg))
                lx = math.log(float(opf[img * N + gg])) - sig if opf[img * N + gg] > 0 else -math.inf
                return abs(sig) <= dsig or abs(lx - math.log(re_.ALPHA_TH)) <= dl

            a2, b2 = [x for x in a if not near_threshold(x)], [x for x in b if not near_threshold(x)]
            short, long_ = (a2, b2) if len(a2) <= len(b2) else (b2, a2)
            if long_[:len(short)] != short:
                unexplained.append((p, "order"))
                continue
            if len(long_) == len(short):
                continue
            # the first extra pair of the longer list: its stop product must lie at 1e-4 within the float32 budget
            ok = False
            for walk in (a, b):
                T, rel = float(T0.reshape(-1)[p]), 0.0
                for x in walk:
                    if x == long_[len(short)]:
                        break
                    al = float(alpha_of(x)[0][0])
                    T *= 1.0 - al
                    rel += al * math.expm1(float(alpha_of(x)[3][0])) / (1.0 - al) + 2 * ULP
                al = float(alpha_of(long_[len(short)])[0][0])
                nT = T * (1.0 - al)
                ok |= abs(nT - T_TH) <= T_TH * (1e-5 + rel)
            if not ok:
                unexplained.append((p, "stop"))
        report[case] = (len(g), len(rg), len(diff_pix), n_pairs)
        assert not unexplained, f"{case}: {len(unexplained)} pixels differ from the reference op unexplained, e.g. {unexplained[:5]}"
    print("\nreference op (ours, theirs, pixels that differ, pairs that differ): " + str(report))


# ------------------------------------------------------------------------------------------
# 6. edge cases
def test_empty_inputs_and_determinism(gs):
    f = _faint_scene(N=300)
    W, H = f["W"], f["H"]
    ones = torch.ones((2, H, W), device=DEV)
    m2, con, op, off, fl = (_t(f[k]) for k in ("means2d", "conics", "opacities", "isect_offsets", "flatten_ids"))
    for fn, rows in ((gs.rasterize_to_indices_in_range, con), (gs.rasterize_to_indices_in_range_2dgs, None)):
        if rows is None:
            rows = torch.zeros((2, 300, 3, 3), device=DEV)
            rows[..., 0, 0] = rows[..., 1, 1] = 0.2
            rows[..., 0, 2], rows[..., 1, 2], rows[..., 2, 2] = m2[..., 0], m2[..., 1], 1.0  # screen mean m2
        # no intersections, N = 0
        e = fn(0, 5, ones, m2, rows, op, W, H, 16, torch.zeros_like(off), fl[:0])
        assert all(x.dtype == torch.int64 and x.numel() == 0 for x in e)
        e = fn(0, 5, ones, m2[:, :0], rows[:, :0], op[:, :0], W, H, 16, torch.zeros_like(off), fl[:0])
        assert all(x.numel() == 0 for x in e)
        # nothing lands on tile (0, 0) of image 1: its list is empty
        fl2 = fl.clone()
        off2 = off.clone()
        off2.view(-1)[off2.numel() // 2] = off2.view(-1)[off2.numel() // 2 + 1]
        out = fn(0, 10**10, ones, m2, rows, op, W, H, 16, off2, fl2)
        lin = _n(out[2]) * H * W + _n(out[1])
        y, x = (lin % (H * W)) // W, lin % W
        assert len(lin) > 0 and not ((_n(out[2]) == 1) & (y < 16) & (x < 16)).any()
        a, b = fn(0, 10**10, ones, m2, rows, op, W, H, 16, off, fl), fn(0, 10**10, ones, m2, rows, op, W, H, 16, off, fl)
        assert all(torch.equal(u, v) for u, v in zip(a, b)) and len(a[0]) > 1000
