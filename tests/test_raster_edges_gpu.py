"""The compositing kernels at their edges, against float64 truth.

* The adversarial single-gaussian sweep of tests/raster_edges.py: the warp-level cull must never drop a pair that
  reaches alpha >= 1/255 (forward on every decided pixel, gradients per gaussian against the float64 oracle).
* Every compiled channel width and the padded ones (D = 2, 5, 16; 6, 12, 20, 31) on a 327 x 203 garden crop, whose
  tiles are partial on the right AND the bottom edge, plus masks in the backward, leading batch dims and packed rows.
* rasterization() at 327 x 203 (SH3, dense and packed) and with 33 / 64 feature channels (chunked compositing).
* The longest-list-first tile order: replicas of one view rendered with and without it, and a tile of > 9000
  intersections that falls into the order's clamped length bin.
* The registry binding (rasterize_to_pixels_3dgs / _bwd called as Python functions) against rasterize_to_pixels.
"""
import math

import numpy as np
import pytest
import torch

from oracle import gso
from tests import raster_edges as re_
from tests import scene
from tests.test_gpu_parity import DEV, _n, _pipeline_case, _project_scene, _raster_case, _t, gs  # noqa: F401  (gs: fixture)

pytestmark = pytest.mark.gpu

W_EDGE, H_EDGE = 327, 203  # 20.4 x 12.7 tiles: partial tiles on the right and on the bottom


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------
# adversarial single-gaussian sweep
@pytest.fixture(scope="module")
def sweep():
    sw = re_.make_sweep()
    return sw, re_.truth(sw)


@pytest.mark.parametrize("D", [3, 5])
def test_cull_sweep_vs_float64_truth(gs, sweep, D):
    sw, tr = sweep
    W, H = re_.W, re_.H
    m2, con, op = sw["means2d"], sw["conics"], sw["opacities"]
    col, bg = sw[f"colors{D}"], sw[f"bg{D}"]
    off, fl = sw["isect_offsets"], sw["flatten_ids"]
    tm2, tcon, tcol, top, tbg = (_t(a, True) for a in (m2, con, col, op, bg))
    rc, ra = gs.rasterize_to_pixels(tm2, tcon, tcol, top, W, H, 16, _t(off), _t(fl), backgrounds=tbg)
    msgs = re_.check_render(sw, tr, _n(rc), _n(ra), D, what=f"D={D}")
    assert not msgs, "\n".join(msgs)

    # backward: per gaussian against the float64 oracle, within its `mag` bound widened by the gaussian's alpha budget
    rng = np.random.RandomState(100 + D)
    v_rc = rng.standard_normal(rc.shape).astype(np.float32)
    v_ra = rng.standard_normal(ra.shape).astype(np.float32)
    grads = torch.autograd.grad((rc * _t(v_rc)).sum() + (ra * _t(v_ra)).sum(), (tm2, tcon, top, tcol))
    d = lambda a: a.astype(np.float64)  # noqa: E731
    _, ora, oli, _ = gso.rasterize_to_pixels(d(m2), d(con), d(col), d(op), W, H, 16, off, fl, d(bg), None, True)
    og = gso.rasterize_to_pixels_bwd(d(m2), d(con), d(col), d(op), W, H, 16, off, fl, ora, oli, d(v_rc), d(v_ra), d(bg))
    undecided = ~tr["decided"].all(axis=(1, 2))
    excluded = undecided | tr["nan_alpha"].any(axis=(1, 2))  # the oracle composites a NaN alpha at the clamp
    assert excluded.mean() < 0.35, f"{excluded.mean():.2%} of the gaussians excluded from the gradient check"
    beta_g = np.where(tr["alpha"] > 0, tr["beta"], 0.0).max(axis=(1, 2))
    untouched = ~excluded & (tr["alpha"] == 0).all(axis=(1, 2))
    for a, key, mi in ((grads[0], "v_means2d", 0), (grads[1], "v_conics", 1), (grads[2], "v_opacities", 2),
                       (grads[3], "v_colors", 3)):
        got = _n(a).astype(np.float64).reshape(len(beta_g), -1)
        assert np.isfinite(got).all(), f"D={D} {key}: non-finite gradients for {np.unique(np.nonzero(~np.isfinite(got))[0])[:5]}"
        ref = og[key].reshape(len(beta_g), -1)
        tol = (1e-4 + 4.0 * beta_g[:, None]) * og["mag"][:, 0, mi][:, None] + 1e-5
        bad = ((np.abs(got - ref) > tol).any(-1)) & ~excluded
        if bad.any():
            i = int(np.nonzero(bad)[0][0])
            pytest.fail(f"D={D} {key}: {int(bad.sum())} gaussians out of bound, e.g. {re_.describe(sw, i)}: "
                        f"got {got[i]}, oracle {ref[i]}, tolerance {tol[i]}")
        # a gaussian that touches no pixel gets exactly zero
        assert (got[untouched] == 0).all(), f"D={D} {key}: gradient on a gaussian that touches no pixel"
    print(f"\nsweep D={D}: {len(beta_g)} gaussians, {excluded.mean():.2%} excluded from the gradient check")


# ------------------------------------------------------------------------------------------
# channel widths, partial right + bottom tiles, masks, batch dims, packed rows
@pytest.fixture(scope="module")
def edge_view():
    sc = scene.make_scene(n_max=30000)
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W_EDGE, H_EDGE)
    return sc, Ks


def _edge_inputs(sc, Ks, C=2, shift=0.0):
    sc2 = dict(sc, means=sc["means"] + np.float32(shift) * np.array([1, 0, 0], np.float32)) if shift else sc
    radii, m2, dep, con, _ = _project_scene(sc2, W_EDGE, H_EDGE, Ks, C=C)
    op = np.ascontiguousarray(np.broadcast_to(sc["opacities"][None], dep.shape)).copy()
    op[:, ::50] = 1.0  # saturating gaussians exercise the 0.99 clamp
    return radii, m2, dep, con, op


@pytest.mark.parametrize("D,bg,absgrad", [(2, True, False), (5, False, True), (16, True, True), (6, False, False),
                                          (12, True, False), (20, False, True), (31, True, False)])
def test_raster_channels_partial_edges_vs_oracle(gs, edge_view, D, bg, absgrad):
    sc, Ks = edge_view
    C = 2
    radii, m2, dep, con, op = _edge_inputs(sc, Ks, C)
    tw, th = math.ceil(W_EDGE / 16), math.ceil(H_EDGE / 16)
    _, ids, fl = gso.isect_tiles(m2, radii, dep, 16, tw, th, True, con, op)
    off = gso.isect_offset_encode(ids, C, tw, th)
    rng = np.random.RandomState(D)
    col = rng.random_sample(m2.shape[:-1] + (D,)).astype(np.float32)
    bgv = rng.random_sample((C, D)).astype(np.float32) if bg else None
    rc, ra = _raster_case(gs, m2, con, col, op, W_EDGE, H_EDGE, off, fl, bgv, absgrad, seed=D)
    # the right-most column and bottom row of pixels are rendered, not left at the background
    assert (_n(ra)[:, :, -1] > 0).mean() > 0.3 and (_n(ra)[:, -1, :] > 0).mean() > 0.3


def test_raster_masked_backward_vs_oracle(gs, edge_view):
    sc, Ks = edge_view
    C, D = 2, 5
    radii, m2, dep, con, op = _edge_inputs(sc, Ks, C)
    tw, th = math.ceil(W_EDGE / 16), math.ceil(H_EDGE / 16)
    _, ids, fl = gso.isect_tiles(m2, radii, dep, 16, tw, th, True, con, op)
    off = gso.isect_offset_encode(ids, C, tw, th)
    rng = np.random.RandomState(7)
    col = rng.random_sample(m2.shape[:-1] + (D,)).astype(np.float32)
    bgv = rng.random_sample((C, D)).astype(np.float32)
    masks = rng.random_sample((C, th, tw)) > 0.3
    masks[:, -1, -1] = False  # the bottom-right partial tile
    # the first non-empty tile's list starts at intersection 0, which is also the last_ids value the forward writes
    # for a masked pixel: only the mask keeps the backward from walking it
    lens = np.diff(np.concatenate([off.reshape(-1), [len(fl)]]))
    first = int(np.nonzero(lens)[0][0])
    masks.reshape(-1)[first] = False
    assert (~masks).sum() > 50 and (lens[~masks.reshape(-1)] > 0).sum() > 50
    rc, ra = _raster_case(gs, m2, con, col, op, W_EDGE, H_EDGE, off, fl, bgv, True, seed=7, masks=masks)
    assert (_n(ra)[0, -7:, -7:] == 0).all()


def test_raster_batch_dims_vs_oracle(gs, edge_view):
    """Leading batch dims [2, 2]: batch element 1 sees the scene shifted along x."""
    sc, Ks = edge_view
    C, D = 2, 3
    parts = [_edge_inputs(sc, Ks, C, shift=0.05 * b) for b in range(2)]
    radii, m2, dep, con, op = (np.stack([p[k] for p in parts]) for k in range(5))
    tw, th = math.ceil(W_EDGE / 16), math.ceil(H_EDGE / 16)
    flat = lambda a: a.reshape((4,) + a.shape[2:])  # noqa: E731
    _, ids, fl = gso.isect_tiles(flat(m2), flat(radii), flat(dep), 16, tw, th, True, flat(con), flat(op))
    off = gso.isect_offset_encode(ids, 4, tw, th).reshape(2, 2, th, tw)
    rng = np.random.RandomState(22)
    col = rng.random_sample(m2.shape[:-1] + (D,)).astype(np.float32)
    bgv = rng.random_sample((2, 2, D)).astype(np.float32)
    rc, _ = _raster_case(gs, m2, con, col, op, W_EDGE, H_EDGE, off, fl, bgv, True, seed=22)
    assert tuple(rc.shape) == (2, 2, H_EDGE, W_EDGE, D)


def test_raster_packed_rows_vs_oracle(gs, edge_view):
    """Packed rows [nnz, *] render exactly what the same rows scattered into the dense layout render, and that
    dense rendering is checked against the float64 oracle."""
    sc, Ks = edge_view
    C, D = 2, 5
    radii, m2, dep, con, op = _edge_inputs(sc, Ks, C)
    tw, th = math.ceil(W_EDGE / 16), math.ceil(H_EDGE / 16)
    _, ids, fl = gso.isect_tiles(m2, radii, dep, 16, tw, th, True, con, op)
    off = gso.isect_offset_encode(ids, C, tw, th)
    rng = np.random.RandomState(31)
    col = rng.random_sample(m2.shape[:-1] + (D,)).astype(np.float32)
    bgv = rng.random_sample((C, D)).astype(np.float32)
    _raster_case(gs, m2, con, col, op, W_EDGE, H_EDGE, off, fl, bgv, True, seed=31)
    sel = (radii > 0).all(-1).reshape(-1)
    row_of = np.cumsum(sel) - 1  # dense row -> packed row
    fl_p = row_of[fl].astype(np.int32)
    assert sel[fl].all() and sel.sum() < sel.size
    flat = lambda a: np.ascontiguousarray(a.reshape((-1,) + a.shape[2:])[sel])  # noqa: E731
    v_rc = _t(rng.standard_normal((C, H_EDGE, W_EDGE, D)).astype(np.float32))
    v_ra = _t(rng.standard_normal((C, H_EDGE, W_EDGE, 1)).astype(np.float32))
    outs = []
    for packed in (False, True):
        ins = [m2, con, col, op] if not packed else [flat(m2), flat(con), flat(col), flat(op)]
        ts = [_t(a, True) for a in ins] + [_t(bgv, True)]
        rc, ra = gs.rasterize_to_pixels(*ts[:4], W_EDGE, H_EDGE, 16, _t(off), _t(fl_p if packed else fl), backgrounds=ts[4],
                                        packed=packed, absgrad=True)
        g = torch.autograd.grad((rc * v_rc).sum() + (ra * v_ra).sum(), ts)
        if not packed:  # gather the dense rows that are packed
            g = [x.reshape((-1,) + x.shape[2:])[_t(sel)] for x in g[:4]] + [g[4]]
            ab = ts[0].absgrad.reshape(-1, 2)[_t(sel)]
        else:
            ab = ts[0].absgrad
        outs.append((rc, ra, g, ab))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    for a, b, name in zip(outs[1][2], outs[0][2], ("v_means2d", "v_conics", "v_colors", "v_opacities", "v_backgrounds")):
        assert _rel(a, b) < 1e-6, (name, _rel(a, b))
    assert _rel(outs[1][3], outs[0][3]) < 1e-6


# ------------------------------------------------------------------------------------------
# rasterization() at non-multiple-of-16 sizes and with chunked channels
@pytest.mark.parametrize("packed", [False, True])
def test_rasterization_sh3_partial_edges(gs, packed):
    sc = scene.make_scene(n_max=30000, sh_degree=3)
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W_EDGE, H_EDGE)
    rc, ra, meta, _ = _pipeline_case(gs, sc, W_EDGE, H_EDGE, Ks, 2, 3, packed=packed, backgrounds=True)
    assert tuple(rc.shape) == (2, H_EDGE, W_EDGE, 3)
    assert (_n(ra)[:, :, -1] > 0).mean() > 0.3 and (_n(ra)[:, -1, :] > 0).mean() > 0.3


@pytest.mark.parametrize("D", [33, 64])
def test_rasterization_chunked_channels_vs_oracle(gs, D):
    sc = scene.make_scene(n_max=20000, sh_degree=0)
    W, H = 200, 120
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)
    col = np.random.RandomState(D).random_sample((sc["means"].shape[0], D)).astype(np.float32)
    rc, _, _, _ = _pipeline_case(gs, sc, W, H, Ks, 1, None, colors=col, backgrounds=True)
    assert rc.shape[-1] == D


# ------------------------------------------------------------------------------------------
# tile order and long lists
def _sm_count():
    return torch.cuda.get_device_properties(torch.device(DEV)).multi_processor_count


def test_tile_order_replicas_bit_identical(gs):
    """One view below the tile-order threshold (n_tiles < 2 * SMs) and the same view replicated until it is above it:
    the forward of every replica is the single render bit for bit, the gradients C x the single ones."""
    sc = scene.make_scene(n_max=30000)
    W, H = 160, 96
    tw, th = math.ceil(W / 16), math.ceil(H / 16)
    sms = _sm_count()
    assert tw * th < 2 * sms
    R = -(-2 * sms // (tw * th)) + 1
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)
    radii, m2, dep, con, _ = _project_scene(sc, W, H, Ks, C=1)
    op = np.broadcast_to(sc["opacities"][None], dep.shape).copy()
    _, ids, fl = gso.isect_tiles(m2, radii, dep, 16, tw, th, True, con, op)
    off = gso.isect_offset_encode(ids, 1, tw, th)
    lens = np.diff(np.concatenate([off.reshape(-1), [len(fl)]]))
    assert lens.max() > 4 * np.median(lens) > 0, "the order must be non-trivial"
    N, S = m2.shape[1], len(fl)
    rng = np.random.RandomState(5)
    col = rng.random_sample((1, N, 3)).astype(np.float32)
    bg = rng.random_sample((1, 3)).astype(np.float32)
    rep = lambda a: np.ascontiguousarray(np.repeat(a, R, axis=0))  # noqa: E731
    off_r = np.concatenate([off + k * S for k in range(R)]).astype(np.int32)
    fl_r = np.concatenate([fl + k * N for k in range(R)]).astype(np.int32)
    v_rc = rng.standard_normal((1, H, W, 3)).astype(np.float32)
    v_ra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    res = []
    for ins, o, f, vr, va in (((m2, con, col, op, bg), off, fl, v_rc, v_ra),
                              (tuple(rep(a) for a in (m2, con, col, op, bg)), off_r, fl_r, rep(v_rc), rep(v_ra))):
        ts = [_t(a, True) for a in ins]
        rc, ra = gs.rasterize_to_pixels(*ts[:4], W, H, 16, _t(o), _t(f), backgrounds=ts[4], absgrad=True)
        g = torch.autograd.grad((rc * _t(vr)).sum() + (ra * _t(va)).sum(), ts)
        res.append((rc, ra, g, ts[0].absgrad))
    (rc1, ra1, g1, ab1), (rcR, raR, gR, abR) = res
    assert rcR.shape[0] == R and R * tw * th >= 2 * sms
    for k in range(R):
        assert torch.equal(rcR[k], rc1[0]) and torch.equal(raR[k], ra1[0]), f"replica {k} differs from the single render"
    for a, b, name in zip(gR + (abR,), g1 + (ab1,), ("v_means2d", "v_conics", "v_colors", "v_opacities", "v_backgrounds", "absgrad")):
        assert _rel(a.sum(0, keepdim=True), R * b) < 1e-6, name
        for k in range(R):
            assert _rel(a[k], b[0]) < 1e-6, (name, k)


def test_long_tile_list_vs_oracle(gs):
    """A tile with > 9000 intersections (more than 70 ring batches, past the order's clamped 255 x 32 length bin) of
    mostly sub-pixel, faint gaussians, in an image whose other tiles are short and whose size crosses the tile-order
    threshold; partial tiles on the right and bottom."""
    sms = _sm_count()
    th = 14
    tw = -(-2 * sms // th) + 1
    W, H = 16 * tw - 5, 16 * th - 3
    rng = np.random.RandomState(9)
    n_small, n_big = 9300, 600
    m_small = rng.uniform(19.0, 29.0, (n_small, 2))
    m_big = np.stack([rng.uniform(0, W, n_big), rng.uniform(0, H, n_big)], -1)
    s = np.concatenate([rng.uniform(0.15, 0.45, n_small), rng.uniform(2.0, 12.0, n_big)])
    m2 = np.concatenate([m_small, m_big]).astype(np.float32)[None]
    rho = rng.uniform(-0.5, 0.5, s.shape)
    sx, sy = s, s * rng.uniform(0.5, 2.0, s.shape)
    det = (sx * sy) ** 2 * (1 - rho**2)
    con = np.stack([sy**2 / det, -rho * sx * sy / det, sx**2 / det], -1).astype(np.float32)[None]
    op = np.concatenate([rng.uniform(0.02, 0.12, n_small), rng.uniform(0.1, 0.6, n_big)]).astype(np.float32)[None]
    dep = rng.uniform(1.0, 5.0, op.shape).astype(np.float32)
    radii = np.ceil(3.0 * np.maximum(sx, sy) * 1.5).astype(np.int32)[None, :, None].repeat(2, -1)
    _, ids, fl = gso.isect_tiles(m2, radii, dep, 16, tw, th, True, con, op)
    off = gso.isect_offset_encode(ids, 1, tw, th)
    lens = np.diff(np.concatenate([off.reshape(-1), [len(fl)]]))
    assert lens[1 * tw + 1] > 9000 and (lens >> 5).max() > 255 and np.median(lens) < 100 and tw * th >= 2 * sms
    col = rng.random_sample((1, m2.shape[1], 3)).astype(np.float32)
    bg = rng.random_sample((1, 3)).astype(np.float32)
    rc, ra = _raster_case(gs, m2, con, col, op, W, H, off, fl, bg, False, seed=9, strict_frac=0.99)
    # the long tile is not saturated: its pixels walk the whole list
    assert (_n(ra)[0, 16:32, 16:32] < 0.99).mean() > 0.5


# ------------------------------------------------------------------------------------------
def test_registry_pair_matches_autograd(gs, edge_view):
    """registry.rasterize_to_pixels_3dgs / _bwd (the pair a gsplat build's op registry would call; the backward rebuilds
    the records with gsb200_raster_pack) against rasterize_to_pixels: forward bit for bit, gradients within 1e-6."""
    from gsplat_b200 import registry

    sc, Ks = edge_view
    C, D = 2, 3
    radii, m2, dep, con, op = _edge_inputs(sc, Ks, C)
    tw, th = math.ceil(W_EDGE / 16), math.ceil(H_EDGE / 16)
    assert C * tw * th >= 2 * _sm_count()  # the tile order is written by the pack the backward runs
    _, ids, fl = gso.isect_tiles(m2, radii, dep, 16, tw, th, True, con, op)
    off = gso.isect_offset_encode(ids, C, tw, th)
    rng = np.random.RandomState(41)
    col = rng.random_sample(m2.shape[:-1] + (D,)).astype(np.float32)
    bg = rng.random_sample((C, D)).astype(np.float32)
    masks = rng.random_sample((C, th, tw)) > 0.2
    v_rc = _t(rng.standard_normal((C, H_EDGE, W_EDGE, D)).astype(np.float32))
    v_ra = _t(rng.standard_normal((C, H_EDGE, W_EDGE, 1)).astype(np.float32))
    ts = [_t(a, True) for a in (m2, con, col, op, bg)]
    toff, tfl, tmask = _t(off), _t(fl), _t(masks)
    rc, ra = gs.rasterize_to_pixels(*ts[:4], W_EDGE, H_EDGE, 16, toff, tfl, backgrounds=ts[4], masks=tmask, absgrad=True)
    g = torch.autograd.grad((rc * v_rc).sum() + (ra * v_ra).sum(), ts)
    plain = [x.detach() for x in ts]
    with torch.no_grad():
        r_rc, r_ra, holder, last_ids = registry.rasterize_to_pixels_3dgs(
            *plain[:4], plain[4], tmask, W_EDGE, H_EDGE, 16, toff, tfl, False, True
        )
        assert torch.equal(r_rc, rc) and torch.equal(r_ra, ra)
        assert holder.shape == plain[0].shape and last_ids.dtype == torch.int32
        v_abs, v_m2, v_con, v_col, v_op, v_bg = registry.rasterize_to_pixels_3dgs_bwd(
            *plain[:4], plain[4], tmask, toff, tfl, r_ra, last_ids, W_EDGE, H_EDGE, 16, True, v_rc, v_ra, True
        )
    for a, b, name in ((v_m2, g[0], "v_means2d"), (v_con, g[1], "v_conics"), (v_col, g[2], "v_colors"),
                       (v_op, g[3], "v_opacities"), (v_bg, g[4], "v_backgrounds"), (v_abs, ts[0].absgrad, "absgrad")):
        assert a.shape == b.shape and _rel(a, b) < 1e-6, (name, _rel(a, b))
