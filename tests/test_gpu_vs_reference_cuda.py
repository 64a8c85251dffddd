"""GPU parity against the REAL reference CUDA operators (nerfstudio-project/gsplat v1.6.0).

The reference's outputs are stored in tests/golden/ref_cuda.npz, recorded on an H100 by
tests/golden/make_ref_cuda_golden.py from the reference's own kernels (built by oracle/build_ref.py) on the same
seeded inputs the tests build here.  To keep the file small the store holds a fixed, seeded sample: per-gaussian
outputs at sampled gaussians, images at sampled pixels, and the full visibility / tile-count arrays.  Per-gaussian
backward passes are independent across gaussians, so ours runs on exactly the sampled rows the reference saw.

The reference is built with -use_fast_math (its default) and accumulates gradients with float atomics,
so it is itself only reproducible to ~1e-6 relative; its own tests compare at rtol 1e-5..2.5e-4 /
atol 1e-3..2e-3 for gradients (tests/test_basic.py:2664-2692).  Here: rtol 1e-4 / atol 1e-5
on rendered colours / alphas (with a bounded count of threshold-flip pixels), relative-L2 bounds on
gradients, exact equality on sort keys when fed identical projections.
"""
import math
import os

import numpy as np
import pytest
import torch

from tests import scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_cuda.npz")
# the reference's stock rasterization() (its Python package + orchestrator + registered autograd), see STOCK_RECORDERS
GOLDEN_STOCK = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_cuda_stock.npz")
_cache = {}


def golden(name):
    """The stored reference outputs of one recorder (see RECORDERS / STOCK_RECORDERS), as torch tensors on the device."""
    if not _cache:
        for path in (GOLDEN, GOLDEN_STOCK):
            d = np.load(path)
            _cache.update({k: d[k] for k in d.files})
    out = {k.split("/", 1)[1]: v for k, v in _cache.items() if k.startswith(name + "/")}
    assert out, f"{name}: no reference data in {GOLDEN} / {GOLDEN_STOCK}"
    return {k: torch.from_numpy(v).to(DEV) for k, v in out.items()}


@pytest.fixture(scope="module")
def gs():
    import gsplat_b200

    return gsplat_b200


def _t(a, rg=False):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    return t.requires_grad_(True) if rg else t


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _scene(n_max, W, H, C, sh_degree=3, grid=1):
    sc = scene.make_scene(scene_grid=grid, n_max=n_max, sh_degree=sh_degree)
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:C]
    return sc, _t(sc["viewmats"][:C]), _t(Ks)


def _sample(n, k, seed):
    """Sorted, seeded sample of k indices out of n (as a device tensor)."""
    return _t(np.sort(np.random.RandomState(seed).choice(n, min(k, n), replace=False)).astype(np.int64))


def _randn(shape, seed):
    return _t(np.random.RandomState(seed).standard_normal(shape).astype(np.float32))


def _vis_bits(radii):
    return _t(np.packbits((radii > 0).all(-1).cpu().numpy().astype(np.uint8).reshape(-1)))


def _unpack_vis(bits, shape):
    return _t(np.unpackbits(bits.cpu().numpy())[: int(np.prod(shape))].reshape(shape).astype(bool))


def _sub(x, idx, dim=0):
    return x.index_select(dim, idx).contiguous()


def _np(d):
    return {k: v.detach().cpu().numpy() for k, v in d.items()}


# ---------------------------------------------------------------------------------------------------------------
# fused projection + SH
PROJ_SH = dict(W=960, H=540, C=2, N=80000, K=512)


def record_projection_sh(ref):
    W, H, C, K = PROJ_SH["W"], PROJ_SH["H"], PROJ_SH["C"], PROJ_SH["K"]
    sc, vm, Ks = _scene(PROJ_SH["N"], W, H, C)
    means, quats, scales, opac, sh = (_t(sc[k]) for k in ("means", "quats", "scales", "opacities", "sh"))
    r_radii, r_m2, r_dep, r_con, _ = ref.projection_ewa_3dgs_fused(means, None, quats, scales, opac, vm, Ks, W, H, 0.3, 0.01, 1e10, 0.0, False, 0)
    rv = (r_radii > 0).all(-1)
    r_col = torch.clamp_min(ref.spherical_harmonics(3, means, vm, sh, rv, None, None, None, None) + 0.5, 0.0)
    idx = _sample(len(means), K, 0)
    s = lambda x: _sub(x, idx, 1)  # noqa: E731
    v_m2, v_dep, v_con, v_col = (_randn(sh_, i) for i, sh_ in enumerate(((C, K, 2), (C, K), (C, K, 3), (C, K, 3))))
    rb = ref.projection_ewa_3dgs_fused_bwd(
        _sub(means, idx), None, _sub(quats, idx), _sub(scales, idx), vm, Ks, W, H, 0.3, 0, s(r_radii), s(r_con), None,
        v_m2, v_dep, v_con, None, False,
    )
    r_vcoef, r_vmeans_sh, _, _ = ref.spherical_harmonics_bwd(
        3, _sub(means, idx), vm, _sub(sh, idx), s(rv), None, None, None, None, (v_col * (s(r_col) > 0)).contiguous(), True, False, False
    )
    return _np(dict(vis=_vis_bits(r_radii), radii=s(r_radii), m2=s(r_m2), dep=s(r_dep), con=s(r_con), col=s(r_col),
                    v_means=rb[0] + r_vmeans_sh, v_quats=rb[2], v_scales=rb[3], v_sh=r_vcoef))


def test_projection_and_sh_vs_reference(gs):
    W, H, C, K = PROJ_SH["W"], PROJ_SH["H"], PROJ_SH["C"], PROJ_SH["K"]
    R = golden("projection_sh")
    sc, vm, Ks = _scene(PROJ_SH["N"], W, H, C)
    means, quats, scales, opac, sh = (_t(sc[k]) for k in ("means", "quats", "scales", "opacities", "sh"))
    N = len(means)
    radii, m2, dep, con, col, _ = gs.fused_project_sh(means, quats, scales, opac, sh, vm, Ks, W, H, 3)
    rv_all, ov_all = _unpack_vis(R["vis"], (C, N)), (radii > 0).all(-1)
    assert (rv_all != ov_all).float().mean() < 1e-4, "visibility sets differ"
    assert (rv_all & ov_all).sum() > 10000
    idx = _sample(N, K, 0)
    s = lambda x: _sub(x, idx, 1)  # noqa: E731
    rv, ov = (R["radii"] > 0).all(-1), (s(radii) > 0).all(-1)
    both = rv & ov
    assert ((R["radii"][both] - s(radii)[both]).abs() <= 1).all() and (R["radii"][both] != s(radii)[both]).float().mean() < 1e-3
    torch.testing.assert_close(s(m2)[both], R["m2"][both], rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(s(dep)[both], R["dep"][both], rtol=1e-5, atol=1e-6)
    assert _rel(s(con)[both], R["con"][both]) < 1e-4
    torch.testing.assert_close(s(con)[both], R["con"][both], rtol=5e-3, atol=1e-5)  # fast-math conic of tiny gaussians
    torch.testing.assert_close(s(col)[both], R["col"][both], rtol=1e-4, atol=1e-5)
    # backward of both ops with common cotangents, on the reference's own forward outputs of the sampled gaussians
    v_m2, v_dep, v_con, v_col = (_randn(sh_, i) for i, sh_ in enumerate(((C, K, 2), (C, K), (C, K, 3), (C, K, 3))))
    L = gs._cabi.lib()
    from gsplat_b200._cabi import ptr, stream

    sm, sq, ss, ssh = (_sub(x, idx) for x in (means, quats, scales, sh))
    v_means, v_quats, v_scales, v_sh = (torch.empty_like(x) for x in (sm, sq, ss, ssh))
    rc = L.gsb200_project_sh_bwd(
        C, K, 16, 3, ptr(sm), ptr(sq), ptr(ss), ptr(ssh), ptr(vm), ptr(Ks), W, H, 0.3, ptr(R["radii"]),
        ptr(R["con"]), None, ptr(R["col"]), ptr(v_m2), 2, ptr(v_dep), 1, ptr(v_con), 3, ptr(v_col), 3, None,
        ptr(v_means), ptr(v_quats), ptr(v_scales), ptr(v_sh), None, stream(),
    )
    assert rc == 0
    assert _rel(v_means, R["v_means"]) < 1e-4
    assert _rel(v_quats, R["v_quats"]) < 1e-3 and _rel(v_scales, R["v_scales"]) < 1e-3
    assert _rel(v_sh, R["v_sh"]) < 1e-5


# ---------------------------------------------------------------------------------------------------------------
# orthographic / fisheye projection
CAMS = dict(W=960, H=540, C=2, N=60000, K=1024)


def _cam_inputs(model):
    sc, vm, Ks = _scene(CAMS["N"], CAMS["W"], CAMS["H"], CAMS["C"])
    if model == "ortho":
        Ks = Ks.clone()
        Ks[:, 0, 0], Ks[:, 1, 1] = 180.0, 170.0
    return sc, vm, Ks


def record_camera_model(ref, model, cam_id):
    W, H, C, K = CAMS["W"], CAMS["H"], CAMS["C"], CAMS["K"]
    sc, vm, Ks = _cam_inputs(model)
    means, quats, scales, opac = (_t(sc[k]) for k in ("means", "quats", "scales", "opacities"))
    r = ref.projection_ewa_3dgs_fused(means, None, quats, scales, opac, vm, Ks, W, H, 0.3, 0.01, 1e10, 0.0, False, cam_id)
    idx = _sample(len(means), K, 1)
    s = lambda x: _sub(x, idx, 1)  # noqa: E731
    v_m2, v_dep, v_con = (_randn(sh_, 10 + i) for i, sh_ in enumerate(((C, K, 2), (C, K), (C, K, 3))))
    rb = ref.projection_ewa_3dgs_fused_bwd(
        _sub(means, idx), None, _sub(quats, idx), _sub(scales, idx), vm, Ks, W, H, 0.3, cam_id, s(r[0]), s(r[3]), None,
        v_m2, v_dep, v_con, None, True,
    )
    return _np(dict(vis=_vis_bits(r[0]), radii=s(r[0]), m2=s(r[1]), dep=s(r[2]), con=s(r[3]),
                    v_means=rb[0], v_quats=rb[2], v_scales=rb[3], v_vm=rb[4]))


@pytest.mark.parametrize("model,cam_id", [("ortho", 1), ("fisheye", 2)])
def test_projection_camera_models_vs_reference(gs, model, cam_id):
    """Ortho / fisheye projection fwd + bwd against the reference CUDA kernels (CameraModelType 1 / 2)."""
    W, H, C, K = CAMS["W"], CAMS["H"], CAMS["C"], CAMS["K"]
    R = golden(f"camera_{model}")
    sc, vm, Ks = _cam_inputs(model)
    means, quats, scales, opac = (_t(sc[k]) for k in ("means", "quats", "scales", "opacities"))
    N = len(means)
    o = gs.fully_fused_projection(means, None, quats, scales, vm, Ks, W, H, opacities=opac, camera_model=model)
    rv_all, ov_all = _unpack_vis(R["vis"], (C, N)), (o[0] > 0).all(-1)
    assert (rv_all != ov_all).float().mean() < 1e-4
    assert (rv_all & ov_all).sum() > 5000
    idx = _sample(N, K, 1)
    s = lambda x: _sub(x, idx, 1)  # noqa: E731
    both = (R["radii"] > 0).all(-1) & (s(o[0]) > 0).all(-1)
    assert ((R["radii"][both] - s(o[0])[both]).abs() <= 1).all()
    torch.testing.assert_close(s(o[1])[both], R["m2"][both], rtol=1e-4, atol=2e-3)
    torch.testing.assert_close(s(o[2])[both], R["dep"][both], rtol=1e-5, atol=1e-6)
    assert _rel(s(o[3])[both], R["con"][both]) < 1e-4
    v_m2, v_dep, v_con = (_randn(sh_, 10 + i) for i, sh_ in enumerate(((C, K, 2), (C, K), (C, K, 3))))
    L = gs._cabi.lib()
    from gsplat_b200._cabi import ptr, stream

    sm, sq, ss = (_sub(x, idx) for x in (means, quats, scales))
    v_means, v_quats, v_scales, v_vm = (torch.empty_like(x) for x in (sm, sq, ss, vm))
    rc = L.gsb200_projection_bwd(
        1, C, K, ptr(sm), None, ptr(sq), ptr(ss), ptr(vm), ptr(Ks), W, H, 0.3, cam_id, ptr(R["radii"]), ptr(R["con"]), None,
        ptr(v_m2), 2, ptr(v_dep), 1, ptr(v_con), 3, None, ptr(v_means), None, ptr(v_quats), ptr(v_scales), ptr(v_vm), stream(),
    )
    assert rc == 0
    assert _rel(v_means, R["v_means"]) < 2e-4 and _rel(v_quats, R["v_quats"]) < 2e-4 and _rel(v_scales, R["v_scales"]) < 2e-4
    assert _rel(v_vm, R["v_vm"]) < 2e-3


# ---------------------------------------------------------------------------------------------------------------
# tile intersection on an identical projection (ours)
ISECT = dict(W=1280, H=720, C=2, N=100000, K=4096)


def _our_projection(gs, n, W, H, C):
    sc, vm, Ks = _scene(n, W, H, C)
    means, quats, scales, opac = (_t(sc[k]) for k in ("means", "quats", "scales", "opacities"))
    radii, m2, dep, con, _ = gs.fully_fused_projection(means, None, quats, scales, vm, Ks, W, H, opacities=opac)
    return radii, m2, dep, con, opac[None].expand(C, -1).contiguous()


def _ref_isect(ref, m2, radii, dep, con, op, C, tw, th):
    tpg, ids, fl = ref.intersect_tile(m2, radii, dep, con, op, None, None, C, 16, tw, th, True, False)
    off = ref.intersect_offset(ids, C, tw, th)
    return tpg, ids, fl, off


def record_isect(ref, gs):
    W, H, C = ISECT["W"], ISECT["H"], ISECT["C"]
    radii, m2, dep, con, op = _our_projection(gs, ISECT["N"], W, H, C)
    tpg, ids, _, _ = _ref_isect(ref, m2, radii, dep, con, op, C, math.ceil(W / 16), math.ceil(H / 16))
    pos = _sample(ids.numel(), ISECT["K"], 2)
    return _np(dict(tpg=tpg, n_ids=torch.tensor([ids.numel()]), ids=ids[pos]))


def test_isect_vs_reference_on_identical_projection(gs):
    W, H, C = ISECT["W"], ISECT["H"], ISECT["C"]
    R = golden("isect")
    radii, m2, dep, con, op = _our_projection(gs, ISECT["N"], W, H, C)
    tw, th = math.ceil(W / 16), math.ceil(H / 16)
    tpg, ids, fl = gs.isect_tiles(m2, radii, dep, 16, tw, th, conics=con, opacities=op)
    # the reference evaluates the ellipse bounds with fast-math (approximate div / sqrt / log): a gaussian
    # whose bound falls within an ulp of a tile edge may gain or lose a tile.  Such tiles hold no pixel with
    # alpha >= 1/255, so images are unaffected; here the symmetric difference must stay below 1e-4.
    diff = (tpg != R["tpg"]).float().mean()
    assert diff < 1e-4, f"tiles_per_gauss differs on {diff * 100:.4f}% of gaussians"
    n_ref = int(R["n_ids"][0])
    if ids.numel() == n_ref:
        same = (ids[_sample(n_ref, ISECT["K"], 2)] == R["ids"]).float().mean()
        assert same > 0.999
    assert abs(ids.numel() - n_ref) <= 1e-4 * ids.numel() + 2


# ---------------------------------------------------------------------------------------------------------------
# compositing on an identical projection (ours), fwd + bwd
RASTER = dict(W=1280, H=720, C=1, N=150000, PIX=4096, K=512)
RASTER_CASES = [(3, False), (3, True), (4, False), (1, False)]


def _raster_inputs(gs, D, with_bg):
    W, H, C = RASTER["W"], RASTER["H"], RASTER["C"]
    radii, m2, dep, con, op = _our_projection(gs, RASTER["N"], W, H, C)
    g = torch.Generator(device=DEV).manual_seed(D)
    col = torch.rand((C, m2.shape[1], D), device=DEV, generator=g)
    bg = torch.rand((C, D), device=DEV, generator=g) if with_bg else None
    v_rc, v_ra = _randn((C, H, W, D), 20 + D), _randn((C, H, W, 1), 30 + D)
    return radii, m2, dep, con, op, col, bg, v_rc, v_ra


def record_raster(ref, gs, D, with_bg):
    W, H, C = RASTER["W"], RASTER["H"], RASTER["C"]
    radii, m2, dep, con, op, col, bg, v_rc, v_ra = _raster_inputs(gs, D, with_bg)
    _, _, fl, off = _ref_isect(ref, m2, radii, dep, con, op, C, math.ceil(W / 16), math.ceil(H / 16))
    r_rc, r_ra, _, r_last = ref.rasterize_to_pixels_3dgs(m2, con, col, op, bg, None, W, H, 16, off, fl, False, False)
    rb = ref.rasterize_to_pixels_3dgs_bwd(m2, con, col, op, bg, None, off, fl, r_ra, r_last, W, H, 16, False, v_rc, v_ra, False)
    rb2 = ref.rasterize_to_pixels_3dgs_bwd(m2, con, col, op, bg, None, off, fl, r_ra, r_last, W, H, 16, False, v_rc, v_ra, False)
    pix, idx = _sample(W * H, RASTER["PIX"], 3), _sample(m2.shape[1], RASTER["K"], 4)
    out = dict(rc=r_rc.reshape(C, W * H, D)[:, pix], ra=r_ra.reshape(C, W * H, 1)[:, pix],
               max_rc=r_rc.abs().amax().reshape(1), max_ra=r_ra.abs().amax().reshape(1))
    for name, i in (("v_means2d", 1), ("v_conics", 2), ("v_colors", 3), ("v_opacities", 4)):
        out[name] = _sub(rb[i], idx, 1)
        out[name + "_spread"] = torch.tensor([_rel(rb2[i], rb[i])])
    return _np(out)


@pytest.mark.parametrize("D,with_bg", RASTER_CASES)
def test_raster_vs_reference(gs, D, with_bg):
    W, H, C = RASTER["W"], RASTER["H"], RASTER["C"]
    R = golden(f"raster_D{D}_bg{int(with_bg)}")
    radii, m2, dep, con, op, col, bg, v_rc, v_ra = _raster_inputs(gs, D, with_bg)
    tw, th = math.ceil(W / 16), math.ceil(H / 16)
    _, ids, fl = gs.isect_tiles(m2, radii, dep, 16, tw, th, conics=con, opacities=op)
    off = gs.isect_offset_encode(ids, C, tw, th)
    ins = [x.detach().clone().requires_grad_(True) for x in (m2, con, col, op)]
    rc, ra = gs.rasterize_to_pixels(*ins, W, H, 16, off, fl, backgrounds=bg)
    pix = _sample(W * H, RASTER["PIX"], 3)
    s_rc, s_ra = rc.detach().reshape(C, W * H, D)[:, pix], ra.detach().reshape(C, W * H, 1)[:, pix]
    err = (s_rc - R["rc"]).abs() - (1e-4 * R["rc"].abs() + 1e-5)
    bad = (err.amax(-1) > 0).float().mean()
    # __expf and the alpha >= 1/255 / T <= 1e-4 decisions can flip on a few pixels between two correct
    # implementations; a flip changes a pixel by at most ~0.4 % of a colour
    assert bad < 2e-4, f"{bad * 100:.4f}% of pixels exceed rtol 1e-4 / atol 1e-5"
    assert (s_rc - R["rc"]).abs().max() < 2e-2 and (s_ra - R["ra"]).abs().max() < 2e-2
    assert abs(float(rc.abs().max()) - float(R["max_rc"][0])) < 2e-2 and abs(float(ra.abs().max()) - float(R["max_ra"][0])) < 2e-2
    grads = torch.autograd.grad((rc * v_rc).sum() + (ra * v_ra).sum(), ins)
    idx = _sample(m2.shape[1], RASTER["K"], 4)
    # two runs of the reference itself differ by its atomic order; its spread was measured when recording, and ours
    # must be within a small multiple of it (and within absolute bounds)
    for name, a, lim in (("v_means2d", grads[0], 2e-4), ("v_conics", grads[1], 2e-4), ("v_colors", grads[2], 5e-5), ("v_opacities", grads[3], 2e-4)):
        spread = float(R[name + "_spread"][0])
        rel = _rel(_sub(a, idx, 1), R[name])
        assert rel < max(lim, 20 * spread), f"{name}: rel L2 {rel:.3e} (reference run-to-run {spread:.3e})"


# ---------------------------------------------------------------------------------------------------------------
# the whole path at 1080p, the reference's ops chained as its orchestrator chains them
FULL = dict(W=1920, H=1080, C=1, PIX=4096, K=256)


def record_full_path(ref):
    W, H, C = FULL["W"], FULL["H"], FULL["C"]
    sc, vm, Ks = _scene(None, W, H, C)
    means, quats, scales, opac, sh = (_t(sc[k]) for k in ("means", "quats", "scales", "opacities", "sh"))
    r_radii, r_m2, r_dep, r_con, _ = ref.projection_ewa_3dgs_fused(means, None, quats, scales, opac, vm, Ks, W, H, 0.3, 0.01, 1e10, 0.0, False, 0)
    rv = (r_radii > 0).all(-1)
    r_raw = ref.spherical_harmonics(3, means, vm, sh, rv, None, None, None, None)
    r_col = (torch.clamp_min(r_raw + 0.5, 0.0) * rv[..., None]).contiguous()
    op = opac[None].expand(C, -1).contiguous()
    _, _, fl, off = _ref_isect(ref, r_m2, r_radii, r_dep, r_con, op, C, math.ceil(W / 16), math.ceil(H / 16))
    r_rc, r_ra, _, r_last = ref.rasterize_to_pixels_3dgs(r_m2, r_con, r_col, op, None, None, W, H, 16, off, fl, False, False)
    v_rc, v_ra = _randn((C, H, W, 3), 40), _randn((C, H, W, 1), 41)
    rb = ref.rasterize_to_pixels_3dgs_bwd(r_m2, r_con, r_col, op, None, None, off, fl, r_ra, r_last, W, H, 16, False, v_rc, v_ra, False)
    v_m2, v_con, v_col, v_op = rb[1], rb[2], rb[3], rb[4]
    r_vcoef, r_vmeans_sh, _, _ = ref.spherical_harmonics_bwd(3, means, vm, sh, rv, None, None, None, None, (v_col * (r_col > 0)).contiguous(), True, False, False)
    pb = ref.projection_ewa_3dgs_fused_bwd(means, None, quats, scales, vm, Ks, W, H, 0.3, 0, r_radii, r_con, None, v_m2, torch.zeros_like(r_dep), v_con, None, False)
    pix, idx = _sample(W * H, FULL["PIX"], 5), _sample(len(means), FULL["K"], 6)
    grads = dict(sh=r_vcoef, opacities=v_op.sum(0), means=pb[0] + r_vmeans_sh, quats=pb[2], scales=pb[3])
    out = dict(rc=r_rc.reshape(C, W * H, 3)[:, pix], max_rc=r_rc.abs().amax().reshape(1))
    for k, v in grads.items():
        out["v_" + k] = _sub(v, idx)
        out["v_" + k + "_norm"] = v.double().norm().reshape(1)
    return _np(out)


def test_full_path_vs_reference_1080p(gs):
    """The BASELINE.json configs[1] scene: ~100k gaussians, 1 camera 1080p, SH3, fwd + bwd vs the reference CUDA ops chained
    exactly as its orchestrator does (csrc/Rendering.cpp:976-1447)."""
    W, H, C = FULL["W"], FULL["H"], FULL["C"]
    R = golden("full_path")
    sc, vm, Ks = _scene(None, W, H, C)
    P = {k: _t(sc[k], True) for k in ("means", "quats", "scales", "opacities", "sh")}
    rc, ra, meta = gs.rasterization(P["means"], P["quats"], P["scales"], P["opacities"], P["sh"], vm, Ks, W, H, sh_degree=3, packed=False)
    pix = _sample(W * H, FULL["PIX"], 5)
    s_rc = rc.detach().reshape(C, W * H, 3)[:, pix]
    err = (s_rc - R["rc"]).abs() - (1e-4 * R["rc"].abs() + 1e-5)
    bad = (err.amax(-1) > 0).float().mean()
    assert bad < 1e-3, f"{bad * 100:.4f}% of pixels exceed rtol 1e-4 / atol 1e-5 vs the reference CUDA rasterizer"
    assert (s_rc - R["rc"]).abs().max() < 5e-2 and abs(float(rc.abs().max()) - float(R["max_rc"][0])) < 5e-2
    v_rc, v_ra = _randn((C, H, W, 3), 40), _randn((C, H, W, 1), 41)
    ((rc * v_rc).sum() + (ra * v_ra).sum()).backward()
    idx = _sample(len(P["means"]), FULL["K"], 6)
    for k, lim in (("sh", 1e-3), ("opacities", 1e-3), ("means", 2e-3), ("quats", 5e-3), ("scales", 5e-3)):
        g = P[k].grad
        assert _rel(_sub(g, idx), R["v_" + k]) < lim, f"v_{k}: sampled rows"
        assert abs(float(g.double().norm()) / float(R["v_" + k + "_norm"][0]) - 1) < lim, f"v_{k}: norm"


# ---------------------------------------------------------------------------------------------------------------
# trainer-side ops
ADAM = dict(N=20000, K=128)


def _adam_inputs():
    g = torch.Generator(device=DEV).manual_seed(3)
    N, cases = ADAM["N"], []
    for shape in ((N, 3), (N, 16, 3)):
        p = torch.randn(shape, device=DEV, generator=g)
        grad = torch.randn(shape, device=DEV, generator=g) * 0.1
        m = torch.randn(shape, device=DEV, generator=g) * 0.01
        v = torch.rand(shape, device=DEV, generator=g) * 1e-3
        vis = torch.rand(N, device=DEV, generator=g) < 0.3
        cases.append((p, grad, m, v, vis))
    n_max = 51
    binoms = torch.zeros((n_max, n_max), device=DEV)
    for n in range(n_max):
        for k in range(n + 1):
            binoms[n, k] = math.comb(n, k)
    opac = torch.rand(N, device=DEV, generator=g) * 0.98 + 0.01
    scales = torch.rand((N, 3), device=DEV, generator=g) * 0.1 + 1e-3
    ratios = torch.randint(1, 12, (N,), device=DEV, generator=g)
    return cases, (opac, scales, ratios, binoms, n_max)


def record_adam_relocation(ref):
    cases, (opac, scales, ratios, binoms, n_max) = _adam_inputs()
    idx, out = _sample(ADAM["N"], ADAM["K"], 7), {}
    for c, (p, grad, m, v, vis) in enumerate(cases):
        a = [x.clone() for x in (p, m, v)]
        ref.adam(a[0], grad, a[1], a[2], vis, 1e-2, 0.9, 0.999, 1e-8)
        for name, x in zip(("p", "m", "v"), a):
            out[f"{name}{c}"] = _sub(x, idx)
    ro, rs = ref.relocation(opac, scales, ratios.int(), binoms, n_max, 0.005)
    out["opac"], out["scales"] = _sub(ro, idx), _sub(rs, idx)
    return _np(out)


def test_adam_and_relocation_vs_reference(gs):
    """Trainer-side ops against the reference kernels (csrc/AdamCUDA.cu, RelocationCUDA.cu)."""
    R = golden("adam_relocation")
    cases, (opac, scales, ratios, binoms, n_max) = _adam_inputs()
    idx = _sample(ADAM["N"], ADAM["K"], 7)
    for c, (p, grad, m, v, vis) in enumerate(cases):
        b = [x.clone() for x in (p, m, v)]
        gs.adam(b[0], grad, b[1], b[2], vis, 1e-2, 0.9, 0.999, 1e-8)
        for name, y in zip(("p", "m", "v"), b):
            torch.testing.assert_close(_sub(y, idx), R[f"{name}{c}"], rtol=1e-5, atol=1e-7)  # the reference is built with fast-math (FMA: cancellation in m)
        assert torch.equal(b[0][~vis], p[~vis])
    o, s = gs.compute_relocation(opac, scales, ratios.clone(), binoms, 0.005)
    torch.testing.assert_close(_sub(o, idx), R["opac"], rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(_sub(s, idx), R["scales"], rtol=1e-4, atol=1e-8)


# ---------------------------------------------------------------------------------------------------------------
# two-pass compacting (packed) projection
PACKED = dict(W=960, H=540, C=3, N=70000, K=1024)


def record_packed(ref):
    W, H, C, K = PACKED["W"], PACKED["H"], PACKED["C"], PACKED["K"]
    sc, vm, Ks = _scene(PACKED["N"], W, H, C)
    means, quats, scales, opac = (_t(sc[k]) for k in ("means", "quats", "scales", "opacities"))
    N = len(means)
    rb, rc_, rg, rind, _, rm2, rdep, rcon, rcomp = ref.projection_ewa_3dgs_packed(
        means, None, quats, scales, opac, vm, Ks, W, H, 0.3, 0.01, 1e10, 0.0, False, True, 0
    )
    vis = torch.zeros((C, N), dtype=torch.bool, device=DEV)
    vis[rc_.long(), rg.long()] = True
    idx = _sample(N, K, 8)
    pos = torch.full((N,), -1, dtype=torch.long, device=DEV)
    pos[idx] = torch.arange(K, device=DEV)
    keep = pos[rg.long()] >= 0  # the rows of the sampled gaussians, in the reference's order
    nnz = int(keep.sum())
    v_m2, v_dep, v_con = _randn((nnz, 2), 50), _randn((nnz,), 51), _randn((nnz, 3), 52)
    sb, scam, sg = rb[keep].contiguous(), rc_[keep].contiguous(), pos[rg.long()][keep].to(rg.dtype).contiguous()
    rbw = ref.projection_ewa_3dgs_packed_bwd(
        _sub(means, idx), None, _sub(quats, idx), _sub(scales, idx), vm, Ks, W, H, 0.3, 0, False, sb, scam, sg,
        rcon[keep].contiguous(), None, v_m2, v_dep, v_con, None, True,
    )
    return _np(dict(vis=_vis_bits(vis[..., None].float()), indptr=rind, rows_b=sb, rows_c=scam, rows_g=sg, m2=rm2[keep], dep=rdep[keep],
                    con=rcon[keep], comp=rcomp[keep], v_means=rbw[0], v_quats=rbw[2], v_scales=rbw[3], v_vm=rbw[4]))


def test_packed_projection_vs_reference(gs):
    """Two-pass compacting projection fwd + bwd against the reference's projection_ewa_3dgs_packed kernels."""
    W, H, C, K = PACKED["W"], PACKED["H"], PACKED["C"], PACKED["K"]
    R = golden("packed")
    sc, vm, Ks = _scene(PACKED["N"], W, H, C)
    means, quats, scales, opac = (_t(sc[k]) for k in ("means", "quats", "scales", "opacities"))
    N = len(means)
    o = gs.fully_fused_projection(means, None, quats, scales, vm, Ks, W, H, opacities=opac, packed=True, calc_compensations=True)
    # visibility differs on a handful of borderline rows (fast-math radius): compare on the common (camera, gaussian) keys
    rvis = _unpack_vis(R["vis"], (C, N))
    ok = o[1].long() * N + o[2].long()
    assert (torch.diff(ok) > 0).all(), "rows must be in ascending (camera, gaussian) order"
    ovis = torch.zeros((C, N), dtype=torch.bool, device=DEV)
    ovis.view(-1)[ok] = True
    n_ref = int(rvis.sum())
    assert abs(n_ref - len(ok)) <= max(2, int(1e-4 * n_ref))
    assert (rvis & ovis).sum() > 0.999 * n_ref
    if n_ref == len(ok):
        assert torch.equal(o[3], R["indptr"])
    # rows of the sampled gaussians: ours at the reference's (camera, gaussian) keys
    idx = _sample(N, K, 8)
    rk = R["rows_c"].long() * N + idx[R["rows_g"].long()]
    row_of = torch.full((C * N,), -1, dtype=torch.long, device=DEV)
    row_of[ok] = torch.arange(len(ok), device=DEV)
    oi = row_of[rk]
    common = oi >= 0
    assert common.float().mean() > 0.999
    oi = oi[common]
    torch.testing.assert_close(o[5][oi], R["m2"][common], rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(o[6][oi], R["dep"][common], rtol=1e-5, atol=1e-6)
    assert _rel(o[7][oi], R["con"][common]) < 1e-4 and _rel(o[8][oi], R["comp"][common]) < 1e-5
    # backward on the reference's own rows / conics of the sampled gaussians (dense accumulation)
    nnz = len(rk)
    v_m2, v_dep, v_con = _randn((nnz, 2), 50), _randn((nnz,), 51), _randn((nnz, 3), 52)
    L = gs._cabi.lib()
    from gsplat_b200._cabi import ptr, stream

    sm, sq, ss = (_sub(x, idx) for x in (means, quats, scales))
    v_means, v_quats, v_scales, v_vm = (torch.empty_like(x) for x in (sm, sq, ss, vm))
    rc = L.gsb200_projection_packed_bwd(
        1, C, K, nnz, ptr(sm), None, ptr(sq), ptr(ss), ptr(vm), ptr(Ks), W, H, 0.3, 0, ptr(R["rows_b"]), ptr(R["rows_c"]),
        ptr(R["rows_g"]), ptr(R["con"]), None, ptr(v_m2), 2, ptr(v_dep), 1, ptr(v_con), 3, None, 0, ptr(v_means), None,
        ptr(v_quats), ptr(v_scales), ptr(v_vm), stream(),
    )
    assert rc == 0
    assert _rel(v_means, R["v_means"]) < 1e-4 and _rel(v_quats, R["v_quats"]) < 1e-4 and _rel(v_scales, R["v_scales"]) < 1e-4
    assert _rel(v_vm, R["v_vm"]) < 1e-3


# ---------------------------------------------------------------------------------------------------------------
# the reference's STOCK path: gsplat.rasterization() -> rasterization_3dgs orchestrator + its registered autograd
STOCK = dict(PIX=4096, K=256)
STOCK_CFGS = ["cfg1_garden_256_sh0", "cfg2_100k_1080p_sh3"]
GRAD_NAMES = ("means", "quats", "scales", "opacities", "sh")


def _stock_inputs(cfg):
    if cfg.startswith("cfg1"):
        sc = scene.make_scene(sh_degree=0)
        W = H = 256
        vm, Ks, deg = _t(sc["viewmats"][:1]), _t(sc["Ks"][:1]), 0
    else:
        W, H, deg = 1920, 1080, 3
        sc, vm, Ks = _scene(100000, W, H, 1)
    P = {k: _t(sc[k]) for k in GRAD_NAMES}
    return sc, P, vm, Ks, W, H, deg, _randn((1, H, W, 3), 60), _randn((1, H, W, 1), 61)


def _stock_step(G, P, vm, Ks, W, H, deg, v_rc, v_ra):
    """fwd + bwd through a rasterization() callable G; returns render, alpha and the parameter gradients."""
    ins = {k: v.detach().clone().requires_grad_(True) for k, v in P.items()}
    rc, ra, _ = G(ins["means"], ins["quats"], ins["scales"], ins["opacities"], ins["sh"], vm, Ks, W, H, sh_degree=deg, packed=False)
    ((rc * v_rc).sum() + (ra * v_ra).sum()).backward()
    return rc.detach(), ra.detach(), {k: ins[k].grad.detach() for k in ins}


def _oracle_grads(sc, W, H, v_rc, v_ra):
    """float64 CPU oracle gradients of the cfg1 step (the ground truth of the reference's formulas)."""
    from oracle import gso

    f8 = lambda a: np.ascontiguousarray(a, np.float64)  # noqa: E731
    _, og = gso.rasterization_fwd_bwd(
        f8(sc["means"]), f8(sc["quats"]), f8(sc["scales"]), f8(sc["opacities"]), f8(sc["sh"]), f8(sc["viewmats"][:1]),
        f8(sc["Ks"][:1]), W, H, 0, f8(v_rc.cpu().numpy()), f8(v_ra.cpu().numpy()),
    )
    return {k: torch.from_numpy(np.asarray(og["v_" + k])).to(DEV) for k in GRAD_NAMES}


def record_stock(gsplat_ref, cfg):
    sc, P, vm, Ks, W, H, deg, v_rc, v_ra = _stock_inputs(cfg)
    r1 = _stock_step(gsplat_ref.rasterization, P, vm, Ks, W, H, deg, v_rc, v_ra)
    r2 = _stock_step(gsplat_ref.rasterization, P, vm, Ks, W, H, deg, v_rc, v_ra)
    pix, idx = _sample(W * H, STOCK["PIX"], 9), _sample(P["means"].shape[0], STOCK["K"], 10)
    out = dict(rc=r1[0].reshape(1, W * H, 3)[:, pix], ra=r1[1].reshape(1, W * H, 1)[:, pix], max_rc=r1[0].abs().amax().reshape(1))
    oracle = _oracle_grads(sc, W, H, v_rc, v_ra) if cfg.startswith("cfg1") else None
    for k in GRAD_NAMES:
        g, g2 = r1[2][k], r2[2][k]
        out[f"v_{k}"] = _sub(g, idx)
        out[f"v_{k}_norm"] = g.double().norm().reshape(1)
        out[f"v_{k}_scale"] = g.abs().max().reshape(1)
        out[f"v_{k}_spread_rel_l2"] = torch.tensor([_rel(g2, g)])
        if oracle is not None:
            og = oracle[k].reshape(g.shape)
            out[f"v_{k}_vs_oracle64_rel_l2"] = ((g.double() - og).norm() / og.norm()).reshape(1)
    return _np(out)


@pytest.mark.parametrize("cfg", STOCK_CFGS)
def test_stock_rasterization_with_gradient_spread(gs, cfg):
    """BASELINE.json configs[0] / configs[1] against the reference's STOCK path -- the unmodified gsplat package:
    gsplat.rasterization() -> rasterization_3dgs orchestrator + its registered autograd (stored outputs).

    Per gradient tensor the recording keeps the reference's own run-to-run spread (two runs, same inputs), its full
    norm and max |g|, sampled rows, and for cfg1 its distance to the float64 CPU oracle.  The reference's spread is
    far below what separates two correct implementations: ours and the reference differ because the reference is a
    -use_fast_math build (approximate division / rsqrt / log in the projection and conic inversion) while our
    per-gaussian kernels are bit-exact against the float32 oracle, and because discrete decisions (alpha >= 1/255,
    T <= 1e-4, radius / tile cuts) flip on a few (pixel, gaussian) pairs.
    Asserted: render / alpha rtol 1e-4, atol 1e-5 on all but < 0.1 % decision-flip pixels; every gradient tensor within
    1e-3 relative L2 of the reference (sampled rows and full norm) and >= 99 % of the sampled elements within
    rtol 1e-4 + atol 1e-5 * max|g|; on cfg1 ours at least as close to the float64 oracle as the reference is
    (factor 1.5 + 2e-5)."""
    R = golden(f"stock_{cfg}")
    sc, P, vm, Ks, W, H, deg, v_rc, v_ra = _stock_inputs(cfg)
    o1 = _stock_step(gs.rasterization, P, vm, Ks, W, H, deg, v_rc, v_ra)
    pix, idx = _sample(W * H, STOCK["PIX"], 9), _sample(P["means"].shape[0], STOCK["K"], 10)
    s_rc, s_ra = o1[0].reshape(1, W * H, 3)[:, pix], o1[1].reshape(1, W * H, 1)[:, pix]
    bad = float((((s_rc - R["rc"]).abs() - (1e-4 * R["rc"].abs() + 1e-5)).amax(-1) > 0).float().mean())
    bad_a = float(((((s_ra - R["ra"]).abs() - (1e-4 * R["ra"].abs() + 1e-5))) > 0).float().mean())
    oracle = _oracle_grads(sc, W, H, v_rc, v_ra) if cfg.startswith("cfg1") else None
    report = {"cfg": cfg, "n_gaussians": int(P["means"].shape[0]), "render_pixels_out_of_1e-4_1e-5": bad, "alpha_pixels_out": bad_a, "grads": {}}
    fails = []
    for k in GRAD_NAMES:
        ref_g, our_g, scale = R[f"v_{k}"], _sub(o1[2][k], idx), float(R[f"v_{k}_scale"][0])
        tol = 1e-4 * ref_g.abs() + 1e-5 * scale
        row = {
            "ref_run_to_run_rel_l2": float(R[f"v_{k}_spread_rel_l2"][0]), "ours_vs_ref_rel_l2": _rel(our_g, ref_g),
            "ours_vs_ref_norm_ratio": float(o1[2][k].double().norm()) / float(R[f"v_{k}_norm"][0]),
            "ours_vs_ref_frac_outside_rtol1e-4_atol1e-5scale": float(((our_g - ref_g).abs() > tol).float().mean()),
        }
        if oracle is not None:
            og64 = oracle[k].reshape(o1[2][k].shape)
            row["ours_vs_oracle64_rel_l2"] = float((o1[2][k].double() - og64).norm() / og64.norm())
            row["ref_vs_oracle64_rel_l2"] = float(R[f"v_{k}_vs_oracle64_rel_l2"][0])
            # (sh is reported but not asserted against the oracle: the garden colours contain exact zeros, whose SH
            # value sits exactly on the relu edge of clamp_min(sh + 0.5, 0) -- float32 and float64 evaluations fall on
            # different sides of it, for the reference and for us alike)
            if k != "sh" and not row["ours_vs_oracle64_rel_l2"] <= 1.5 * row["ref_vs_oracle64_rel_l2"] + 2e-5:
                fails.append(f"{k}: ours vs float64 oracle {row['ours_vs_oracle64_rel_l2']:.3e}, reference vs oracle {row['ref_vs_oracle64_rel_l2']:.3e}")
        report["grads"][k] = row
        if not (row["ours_vs_ref_rel_l2"] <= 1e-3 and abs(row["ours_vs_ref_norm_ratio"] - 1) <= 1e-3):
            fails.append(f"{k}: rel L2 {row['ours_vs_ref_rel_l2']:.3e}, norm ratio {row['ours_vs_ref_norm_ratio']:.6f} vs the reference")
        if not row["ours_vs_ref_frac_outside_rtol1e-4_atol1e-5scale"] <= 1e-2:
            fails.append(f"{k}: {row['ours_vs_ref_frac_outside_rtol1e-4_atol1e-5scale'] * 100:.3f} % of the elements outside rtol 1e-4 + atol 1e-5 max|g|")
    print(report)
    assert bad < 1e-3 and bad_a < 1e-3, report
    assert (s_rc - R["rc"]).abs().max() < 5e-2 and abs(float(o1[0].abs().max()) - float(R["max_rc"][0])) < 5e-2
    assert not fails, (fails, report)


def STOCK_RECORDERS(gsplat_ref):
    """name -> thunk producing the stored outputs of the reference's stock path (tests/golden/make_ref_cuda_golden.py)."""
    return {f"stock_{cfg}": (lambda cfg=cfg: record_stock(gsplat_ref, cfg)) for cfg in STOCK_CFGS}


def RECORDERS(ref, gs):
    """name -> thunk producing the stored reference outputs of one test (tests/golden/make_ref_cuda_golden.py)."""
    rec = {
        "projection_sh": lambda: record_projection_sh(ref),
        "camera_ortho": lambda: record_camera_model(ref, "ortho", 1),
        "camera_fisheye": lambda: record_camera_model(ref, "fisheye", 2),
        "isect": lambda: record_isect(ref, gs),
        "full_path": lambda: record_full_path(ref),
        "adam_relocation": lambda: record_adam_relocation(ref),
        "packed": lambda: record_packed(ref),
    }
    for D, bg in RASTER_CASES:
        rec[f"raster_D{D}_bg{int(bg)}"] = (lambda D=D, bg=bg: record_raster(ref, gs, D, bg))
    return rec
