"""The projection and tile-intersection kernels on the adversarial sweep of tests/projection_edges.py.

* Dense projection for every camera x {quats / scales, covars} x {with, without opacities} x calc_compensations, and
  with radius_clip = 5 and eps2d = 0: on every decided row the radii equal the float64 truth, and means2d, depths,
  conics and compensations are within their budgets.
* Packed projection (with and without sparse_grad) returns exactly the dense rows; the fused projection + SH
  (C = 1 and 2, with and without the row side outputs) returns the dense projection's values bit for bit on every row.
* The backward of the dense, packed (dense_out and sparse_grad) and fused (C = 1) projection, for seeded cotangents
  of means2d, depths and conics on the decided rows, against the float64 oracle backward within the per-gaussian
  budgets of tests/projection_edges.py (the configurations of GRAD_CONFIGS), and v_viewmats with leading batch dims
  [2] and N = 4113 (warps straddle the two batch elements) within the l1 of the per-row budgets.
* A radius of 2^31 or more saturates to INT32_MAX and goes through the AABB count / emit and the masked count / emit.
* Tile intersection on the GPU's own projected rows and on a 2D adversarial set: accu and AABB, sorted and unsorted,
  equal the float32 oracle bit for bit; the offsets of isect_tiles_sorted equal isect_offset_encode, and the fused row
  side outputs equal isect_tiles; isect_tiles_sparse equals the masked subset of the AABB list; every decided pixel of
  alpha >= 1/255 is listed; and the one-thread-per-row emit lists the same intersections as the warp-cooperative one.
"""
import math

import numpy as np
import pytest
import torch

from oracle import gso
from tests import projection_edges as pe
from tests.test_gpu_parity import _n, _t, gs, isect_sorted_equals_stable_sort  # noqa: F401  (gs: fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sweep():
    return pe.make_sweep()


_truths = {}


def _truth(sweep, cfg):
    if cfg not in _truths:
        _truths[cfg] = pe.truth(sweep[cfg.family], cfg)
    return _truths[cfg]


def _gpu_project(gs, rows, cfg, packed=False, sparse_grad=False):
    vm, Ks = cfg.camera_arrays()
    kw = cfg.kwargs()
    return gs.fully_fused_projection(
        _t(rows["means"]), _t(rows["covars"]) if cfg.covars else None, _t(rows["quats"]), _t(rows["scales"]), _t(vm),
        _t(Ks), kw["width"], kw["height"], eps2d=kw["eps2d"], near_plane=kw["near_plane"], far_plane=kw["far_plane"],
        radius_clip=kw["radius_clip"], packed=packed, sparse_grad=sparse_grad, calc_compensations=cfg.comp,
        camera_model=kw["camera_model"], opacities=_t(rows["opacities"]) if cfg.opacities else None,
    )


@pytest.mark.parametrize("cfg", pe.CONFIGS, ids=str)
def test_dense_projection_vs_truth(gs, sweep, cfg):
    rows = sweep[cfg.family]
    tr = _truth(sweep, cfg)
    out = [None if o is None else _n(o) for o in _gpu_project(gs, rows, cfg)]
    msgs = pe.check_forward(rows, cfg, tr, *out, what=f"GPU {cfg}")
    assert not msgs, "\n".join(msgs)


@pytest.mark.parametrize("cfg", [pe.Config("pinhole", C=2), pe.Config("pinhole", C=2, covars=True, comp=True),
                                 pe.Config("fisheye", comp=True), pe.Config("ortho", opacities=False)], ids=str)
@pytest.mark.parametrize("sparse_grad", [False, True])
def test_packed_projection_equals_dense(gs, sweep, cfg, sparse_grad):
    rows = sweep[cfg.family]
    dense = [None if o is None else _n(o) for o in _gpu_project(gs, rows, cfg)]
    bids, cids, gids, indptr, radii, m2, dep, con, comp = _gpu_project(gs, rows, cfg, packed=True, sparse_grad=sparse_grad)
    vis = (dense[0] > 0).all(-1)
    c, n = np.nonzero(vis)
    assert np.array_equal(_n(cids), c) and np.array_equal(_n(gids), n) and (_n(bids) == 0).all()
    assert np.array_equal(_n(indptr), np.concatenate([[0], np.cumsum(vis.sum(-1))]))
    for got, ref in ((radii, dense[0]), (m2, dense[1]), (dep, dense[2]), (con, dense[3]), (comp, dense[4])):
        if ref is not None:
            assert np.array_equal(_n(got), ref[vis], equal_nan=True), "packed rows differ from the dense ones"


@pytest.mark.parametrize("C", [1, 2])
@pytest.mark.parametrize("rows_out", [False, True])
def test_fused_project_sh_equals_dense(gs, sweep, C, rows_out):
    """every row, decided or not: the fused kernel and the dense projection share project_one (-fmad=false)"""
    rows = sweep["pinhole"]
    cfg = pe.Config("pinhole", C=C)
    vm, Ks = cfg.camera_arrays()
    kw = cfg.kwargs()
    N = rows["means"].shape[0]
    sh = np.random.RandomState(3).standard_normal((N, 4, 3)).astype(np.float32) * 0.3
    ro = gs.ops.RowSideOutputs(16, math.ceil(pe.W / 16), math.ceil(pe.H / 16)) if rows_out else None
    fr, fm, fd, fc, fcol, _ = gs.ops.fused_project_sh(
        _t(rows["means"]), _t(rows["quats"]), _t(rows["scales"]), _t(rows["opacities"]), _t(sh), _t(vm), _t(Ks), pe.W,
        pe.H, 1, eps2d=kw["eps2d"], near_plane=kw["near_plane"], far_plane=kw["far_plane"], rows_out=ro,
    )
    dense = [_n(o) for o in _gpu_project(gs, rows, cfg)[:4]]
    for got, ref, name in ((fr, dense[0], "radii"), (fm, dense[1], "means2d"), (fd, dense[2], "depths"), (fc, dense[3], "conics")):
        assert np.array_equal(_n(got), ref), f"fused {name} differs from the dense projection"
    tr = _truth(sweep, cfg)
    msgs = pe.check_forward(rows, cfg, tr, _n(fr), _n(fm), _n(fd), _n(fc), None, what=f"fused C={C}")
    assert not msgs, "\n".join(msgs)
    if rows_out:
        tpg, _, _ = gs.isect_tiles(fm, fr, fd, 16, ro.tile_width, ro.tile_height, conics=fc,
                                   opacities=_t(np.ascontiguousarray(np.broadcast_to(rows["opacities"], (C, N)))))
        assert torch.equal(ro.tiles_per_gauss, tpg)
        t = _n(tpg)
        assert int(ro.totals[0]) == t.sum() and int(ro.totals[1]) == (t > 0).sum() and int(ro.totals[2]) == t.max()


_grads = {}


def _grad_truth(sweep, cfg):
    if cfg not in _grads:
        rows = sweep[cfg.family]
        _grads[cfg] = pe.grad_truth(rows, cfg, _truth(sweep, cfg), pe.cotangents(cfg, rows["means"].shape[0]))
    return _grads[cfg]


def _leaves(rows, cfg):
    vm, Ks = cfg.camera_arrays()
    return [_t(rows[k], True) for k in ("means", "quats", "scales")] + [_t(vm, True), _t(Ks)]


def _loss(outs, cot, rows_sel=None):
    m2, dep, con = outs
    c = [_t(cot[k]) for k in ("v_means2d", "v_depths", "v_conics")]
    if rows_sel is not None:
        c = [x[rows_sel] for x in c]
    return (m2 * c[0]).sum() + (dep * c[1]).sum() + (con * c[2]).sum()


@pytest.mark.parametrize("cfg", pe.GRAD_CONFIGS, ids=str)
@pytest.mark.parametrize("path", ["dense", "packed", "sparse_grad", "fused"])
def test_projection_backward_vs_truth(gs, sweep, cfg, path):
    rows = sweep[cfg.family]
    tr = _truth(sweep, cfg)
    ref, beta, cot = _grad_truth(sweep, cfg)
    means, quats, scales, vm, Ks = _leaves(rows, cfg)
    kw = cfg.kwargs()
    common = dict(eps2d=kw["eps2d"], near_plane=kw["near_plane"], far_plane=kw["far_plane"], radius_clip=kw["radius_clip"])
    op = _t(rows["opacities"])
    if path == "fused":
        N = rows["means"].shape[0]
        sh = _t(np.zeros((N, 1, 3), np.float32), True)
        _, m2, dep, con, _, _ = gs.ops.fused_project_sh(means, quats, scales, op, sh, vm.detach(), Ks, pe.W, pe.H, 0, **common)
        g = torch.autograd.grad(_loss((m2, dep, con), cot), (means, quats, scales))
        got = dict(v_means=g[0], v_quats=g[1], v_scales=g[2])
    elif path == "dense":
        _, m2, dep, con, _ = gs.fully_fused_projection(means, None, quats, scales, vm, Ks, pe.W, pe.H, opacities=op, **common)
        g = torch.autograd.grad(_loss((m2, dep, con), cot), (means, quats, scales, vm))
        got = dict(v_means=g[0], v_quats=g[1], v_scales=g[2], v_viewmats=g[3])
    else:
        _, cids, gids, _, _, m2, dep, con, _ = gs.fully_fused_projection(
            means, None, quats, scales, vm, Ks, pe.W, pe.H, opacities=op, packed=True, sparse_grad=path == "sparse_grad",
            **common)
        sel = (cids, gids)
        g = torch.autograd.grad(_loss((m2, dep, con), cot, sel), (means, quats, scales, vm))
        got = dict(v_means=g[0], v_quats=g[1], v_scales=g[2], v_viewmats=g[3])
        if path == "sparse_grad":
            got = {k: (v.to_dense() if v.is_sparse else v) for k, v in got.items()}
    got = {k: _n(v) for k, v in got.items()}
    msgs = pe.check_grads(rows, tr, got, ref, beta, f"{path} {cfg}")
    assert not msgs, "\n".join(msgs)


def test_batch_dims_straddling_warps(gs, sweep):
    """leading batch dims [2] with N = 4113: a warp straddles the two batch elements, and the per-camera v_viewmats
    leave the warp reduction for per-lane atomics; each batch element's v_viewmats against the l1 of its rows' budgets"""
    rows_all = sweep["pinhole"]
    cfg = pe.Config("pinhole")
    N = 4113
    # ordinary rows, so that the l1 budget is not dominated by a needle's: moving the 15 rows of batch element 1 in the
    # straddling warp to element 0 must show
    bulk = np.nonzero(rows_all["cls"] == "bulk")[0]
    idx = [bulk[np.arange(N) % len(bulk)], bulk[(np.arange(N) * 7 + 11) % len(bulk)]]
    parts = [pe.subset(rows_all, i) for i in idx]
    truths = [pe.truth(p, cfg) for p in parts]
    gts = [pe.grad_truth(p, cfg, t, pe.cotangents(cfg, N, seed=b)) for b, (p, t) in enumerate(zip(parts, truths))]
    st = lambda k: np.ascontiguousarray(np.stack([p[k] for p in parts]))  # noqa: E731
    vm, Ks = cfg.camera_arrays()
    vm2, Ks2 = np.ascontiguousarray(np.stack([vm, vm])), np.ascontiguousarray(np.stack([Ks, Ks]))
    means, quats, scales, tvm = _t(st("means"), True), _t(st("quats"), True), _t(st("scales"), True), _t(vm2, True)
    kw = cfg.kwargs()
    radii, m2, dep, con, _ = gs.fully_fused_projection(
        means, None, quats, scales, tvm, _t(Ks2), pe.W, pe.H, eps2d=kw["eps2d"], near_plane=kw["near_plane"],
        far_plane=kw["far_plane"], opacities=_t(st("opacities")))
    cot = {k: np.ascontiguousarray(np.stack([g[2][k] for g in gts])) for k in ("v_means2d", "v_depths", "v_conics")}
    g = torch.autograd.grad(_loss((m2, dep, con), cot), (means, quats, scales, tvm))
    for b in range(2):
        assert np.array_equal(_n(radii)[b][truths[b].decided], truths[b].radii[truths[b].decided])
        got = dict(v_means=_n(g[0])[b], v_quats=_n(g[1])[b], v_scales=_n(g[2])[b], v_viewmats=_n(g[3])[b])
        msgs = pe.check_grads(parts[b], truths[b], got, gts[b][0], gts[b][1], f"batch element {b}")
        assert not msgs, "\n".join(msgs)


def test_radius_beyond_int32_on_gpu(gs, sweep):
    """the GPU keeps the (1e7, 1e7, 1e-3) rows with radius INT32_MAX, like the truth; the AABB and the masked
    count / emit list every tile (of the mask) for them"""
    rows = sweep["pinhole"]
    cfg = pe.Config("pinhole")
    tr = _truth(sweep, cfg)
    sel = np.nonzero((tr.cls == "radius>=2^31") & tr.decided[0])[0]
    radii, m2, dep, con, _ = _gpu_project(gs, rows, cfg)
    r = _n(radii)[0, sel]
    print(f"\nradius >= 2^31 rows on the GPU: radii {r.tolist()}")
    assert (r == pe.INT32_MAX).all()
    tw, th = math.ceil(pe.W / 16), math.ceil(pe.H / 16)
    pick = lambda a: a[:, torch.from_numpy(sel).to(a.device)].contiguous()  # noqa: E731
    tpg, ids, fl = gs.isect_tiles(pick(m2), pick(radii), pick(dep), 16, tw, th)
    assert (_n(tpg) == tw * th).all() and len(fl) == len(sel) * tw * th
    mask = np.random.RandomState(5).random_sample((1, th, tw)) > 0.6
    active = np.nonzero(mask.reshape(-1))[0].astype(np.int32)
    offs, fl_s = gs.isect_tiles_sparse(pick(m2), pick(radii), pick(dep), _t(mask), _t(active), 1, 16, tw, th)
    assert len(fl_s) == len(sel) * len(active) and np.array_equal(np.diff(_n(offs)), np.full(len(active), len(sel)))


def _isect_sets(gs, sweep):
    """(name, means2d, radii, depths, conics, opacities, W, H) of the GPU-projected pinhole rows (C = 2) and of the 2D
    adversarial sets on 304 x 208 (247 tiles) and 400 x 272 (425 tiles)"""
    rows = sweep["pinhole"]
    cfg = pe.Config("pinhole", C=2)
    radii, m2, dep, con, _ = (_n(o) if o is not None else None for o in _gpu_project(gs, rows, cfg))
    op = np.ascontiguousarray(np.broadcast_to(rows["opacities"], dep.shape))
    out = [("projected", m2, radii, dep, con, op, pe.W, pe.H)]
    for W2, H2 in ((304, 208), (400, 272)):
        a = pe.adversarial_2d(W2, H2)
        out.append((f"2d {W2}x{H2}", a["means2d"], a["radii"], a["depths"], a["conics"], a["opacities"], W2, H2))
    return out


def test_isect_vs_oracle_and_coverage(gs, sweep):
    for name, m2, radii, dep, con, op, W2, H2 in _isect_sets(gs, sweep):
        tw, th = math.ceil(W2 / 16), math.ceil(H2 / 16)
        I, N = m2.shape[:2]
        bits = gso.bits_for_count(tw * th)
        req = pe.required_tiles(m2, con, op, radii, W2, H2)
        for accu in (True, False):
            sorted_lists = None
            kw_o = dict(conics=con, opacities=op) if accu else {}
            kw_g = dict(conics=_t(con), opacities=_t(op)) if accu else {}
            for sort in (True, False):
                tpg, ids, fl = gs.isect_tiles(_t(m2), _t(radii), _t(dep), 16, tw, th, sort=sort, **kw_g)
                otpg, oids, ofl = gso.isect_tiles(m2, radii, dep, 16, tw, th, sort, **kw_o)
                what = f"{name} {'accu' if accu else 'aabb'} {'sorted' if sort else 'unsorted'}"
                assert np.array_equal(_n(tpg), otpg), f"{what}: tiles_per_gauss differ in {np.nonzero(_n(tpg) != otpg)}"
                if sort:
                    assert np.array_equal(_n(ids), oids) and np.array_equal(_n(fl), ofl), f"{what}: lists differ"
                else:  # emit order is per gaussian; compare as sets of (key, id) pairs
                    g = np.lexsort((_n(fl), _n(ids)))
                    o = np.lexsort((ofl, oids))
                    assert np.array_equal(_n(ids)[g], oids[o]) and np.array_equal(_n(fl)[g], ofl[o]), f"{what}: lists differ"
                if sort:
                    sorted_lists = (tpg, ids, fl)
                    miss = pe.missing_tiles(req, pe.listed_tiles(_n(ids), _n(fl), N, bits))
                    assert not miss, f"{what}: {len(miss)} gaussians miss tiles with decided pixels, e.g. {miss[:3]}"
            # the offsets of the sorted pipeline against the stand-alone offsets kernel
            _, ids, _ = sorted_lists
            si = gs.ops.isect_tiles_sorted(_t(m2), _t(radii), _t(dep), 16, tw, th, **kw_g)
            assert torch.equal(si.isect_offsets, gs.isect_offset_encode(ids, I, tw, th))
        if name != "projected":  # needles over 64 tiles take the cooperative emit
            atpg, _, _ = gso.isect_tiles(m2, radii, dep, 16, tw, th, True, con, op)
            assert (atpg > 64).sum() >= 10
        # masked AABB lists: the subset of the dense AABB list in the masked tiles, same order
        rng = np.random.RandomState(11)
        mask = rng.random_sample((I, th, tw)) > 0.5
        active = np.nonzero(mask.reshape(-1))[0].astype(np.int32)
        offs, fl_s = gs.isect_tiles_sparse(_t(m2), _t(radii), _t(dep), _t(mask), _t(active), I, 16, tw, th)
        _, oids, ofl = gso.isect_tiles(m2, radii, dep, 16, tw, th, True)
        key = (oids >> 32) & ((1 << (bits + gso.bits_for_count(I))) - 1)
        img, tile = key >> bits, key & ((1 << bits) - 1)
        keep = mask.reshape(-1)[img * tw * th + tile]
        assert np.array_equal(_n(fl_s), ofl[keep]), f"{name}: isect_tiles_sparse differs from the masked AABB list"
        lens = np.bincount(np.searchsorted(active, (img * tw * th + tile)[keep]), minlength=len(active))
        assert np.array_equal(np.diff(_n(offs)), lens)


def test_serial_emit_equals_cooperative(gs, sweep):
    """Sorted dense isect_tiles picks its emit kernel from the largest tile count of a row: one thread per row up to 96
    tiles, warp-cooperative above; the unsorted path always emits cooperatively.  With the rows of more than 96 tiles
    culled (radius 0), the sorted lists come from the one-thread-per-row kernel and must equal a stable sort of the
    cooperative emission; on the full sets both sides are cooperative."""
    for name, m2, radii, dep, con, op, W2, H2 in _isect_sets(gs, sweep):
        tw, th = math.ceil(W2 / 16), math.ceil(H2 / 16)
        kw = dict(conics=_t(con), opacities=_t(op))
        tpg = _n(gs.isect_tiles(_t(m2), _t(radii), _t(dep), 16, tw, th, **kw)[0])
        few = radii.copy()
        few[tpg > 96] = 0
        for rows, r in (("rows of <= 96 tiles", few), ("all rows", radii)):
            a = isect_sorted_equals_stable_sort(gs, m2, r, dep, tw, th, **kw)
            t = _n(a[0])
            assert a[2].numel() > 1000, f"{name}, {rows}"
            assert (t.max() <= 96) == (r is few), f"{name}, {rows}: largest row lists {t.max()} tiles"
