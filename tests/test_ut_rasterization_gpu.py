"""rasterization(with_ut=True, with_eval3d=True) on the GPU: the same as the hand-chained 3DGUT operators, against the
float64 oracle (oracle/ut.py with float64 SH), against the reference's own orchestrator (ref_ut_rasterization.npz),
render modes, channel chunks and padding, batch dims, edge cases, the drop-in and a short fit."""
import os
import sys
import types

import numpy as np
import pytest
import torch

import gsplat_b200 as gs
from oracle import gso
from oracle import ut as U
from tests import scene
from tests.test_ut_gpu import CAMS, KEYS, W, H

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_NPZ = os.path.join(ROOT, "tests", "golden", "ref_ut_rasterization.npz")
TW, TH = (W + 15) // 16, (H + 15) // 16


def _t(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)


def _scene(C=1, n=400):
    """The 96x64 crop of test_ut_gpu with SH degree 3 (the SH draw comes after every other parameter of the seed)."""
    sc = scene.make_scene(n_max=n, sh_degree=3, seed=0)
    K = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:C].astype(np.float32)
    return dict(means=sc["means"], quats=sc["quats"], scales=(sc["scales"] * 4.0).astype(np.float32),
                opacities=sc["opacities"], sh=sc["sh"], colors=sc["colors"].astype(np.float32),
                viewmats=sc["viewmats"][:C].copy(), Ks=K)


def _coeffs(coeffs, shape=(1,)):
    return {KEYS[k]: _t(np.tile(np.float32(v), shape + (1,))) for k, v in coeffs.items()}


def _leaves(p, colour, grad=True):
    names = ("means", "quats", "scales", "opacities") + (("sh",) if colour == "sh" else ("colors",))
    return {k: _t(p[k], grad) for k in names}


def _rasterize(L, p, kind, co, colour="sh", vm=None, **kw):
    vm = _t(p["viewmats"]) if vm is None else vm
    return gs.rasterization(
        L["means"], L["quats"], L["scales"], L["opacities"], L["sh"] if colour == "sh" else L["colors"], vm, _t(p["Ks"]),
        W, H, sh_degree=3 if colour == "sh" else None, packed=False, with_ut=True, with_eval3d=True, camera_model=kind,
        **co, **kw,
    )


def _chain(L, p, kind, co, colour, vm, bg):
    """The hand chain: UT projection, SH + clamp, isect_tiles + isect_offset_encode, eval3d compositing."""
    C, N = vm.shape[0], p["means"].shape[0]
    r, m2, d, _, _ = gs.fully_fused_projection_with_ut(
        L["means"].detach(), L["quats"].detach(), L["scales"].detach(), L["opacities"].detach(), vm.detach(), _t(p["Ks"]),
        W, H, camera_model=kind, **co,
    )
    if colour == "sh":
        feat = gs.spherical_harmonics(3, L["means"], vm, L["sh"], masks=(r > 0).all(-1))
        feat = torch.clamp_min(feat + 0.5, 0.0)
    else:
        feat = torch.broadcast_to(L["colors"][None], (C, N, 3))
    _, ii, fl = gs.isect_tiles(m2, r, d, 16, TW, TH)
    offs = gs.isect_offset_encode(ii, C, TW, TH).reshape(C, TH, TW)
    opac = torch.broadcast_to(L["opacities"][None], (C, N))
    rc, ra = gs.rasterize_to_pixels_eval3d(L["means"], L["quats"], L["scales"], feat, opac, vm, _t(p["Ks"]), W, H, 16, offs,
                                           fl, backgrounds=bg, camera_model=kind, **co)
    return rc, ra, fl, offs


# ---- 1. the same as the hand chain
@pytest.mark.parametrize("colour", ["sh", "colors"])
@pytest.mark.parametrize("kind,coeffs", CAMS)
def test_same_as_hand_chain(kind, coeffs, colour):
    C = 2
    p = _scene(C)
    co = _coeffs(coeffs, (C,))
    rng = np.random.RandomState(3)
    bg_np = rng.random_sample((C, 3)).astype(np.float32)
    v_rc = _t(rng.standard_normal((C, H, W, 3)).astype(np.float32))
    v_ra = _t(rng.standard_normal((C, H, W, 1)).astype(np.float32))
    grads = []
    outs = []
    for run in ("rasterization", "chain"):
        L = _leaves(p, colour)
        vm, bg = _t(p["viewmats"], True), _t(bg_np, True)
        if run == "rasterization":
            rc, ra, meta = _rasterize(L, p, kind, co, colour, vm=vm, backgrounds=bg)
            fl, offs = meta["flatten_ids"], meta["isect_offsets"]
            assert meta["tile_size"] == 16 and meta["batch_ids"] is None and meta["gaussian_ids"] is None
        else:
            rc, ra, fl, offs = _chain(L, p, kind, co, colour, vm, bg)
        ((rc * v_rc).sum() + (ra * v_ra).sum()).backward()
        outs.append((rc, ra, fl, offs))
        grads.append({**{k: v.grad for k, v in L.items()}, "viewmats": vm.grad, "backgrounds": bg.grad})
    (a, b) = outs
    assert b[2].numel() > 50
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    for k in grads[1]:
        g, h = grads[0][k], grads[1][k]
        if k == "viewmats" and colour == "colors":
            assert g is None and h is None  # nothing reaches the viewmats without SH directions
            continue
        # the compositing backward accumulates with float atomics, so two runs agree only up to the order of the sums
        assert g is not None and torch.isfinite(g).all(), k
        assert float((g - h).norm()) <= 1e-5 * float(h.norm()), k
        assert float((g - h).abs().max()) <= 1e-4 * float(h.abs().max()), k


# ---- 2. against the float64 oracle: eval3d compositing of float64 SH colours
@pytest.mark.parametrize("kind,coeffs", CAMS)
def test_against_float64_oracle(kind, coeffs):
    p = _scene(1)
    co = _coeffs(coeffs)
    rng = np.random.RandomState(1)
    bg_np = rng.random_sample((1, 3)).astype(np.float32)
    L = _leaves(p, "sh")
    bg = _t(bg_np, True)
    rc, ra, meta = _rasterize(L, p, kind, co, backgrounds=bg)
    fl, offs = meta["flatten_ids"], meta["isect_offsets"]
    assert fl.numel() > 50
    v_rc = rng.standard_normal(rc.shape).astype(np.float32)
    v_ra = rng.standard_normal(ra.shape).astype(np.float32)
    ((rc * _t(v_rc)).sum() + (ra * _t(v_ra)).sum()).backward()

    N = len(p["means"])
    f64 = lambda a: np.asarray(a, np.float64)  # noqa: E731
    masks = (meta["radii"] > 0).all(-1).cpu().numpy()
    x = gso.spherical_harmonics(3, f64(p["means"]), f64(p["viewmats"]), f64(p["sh"]), masks=masks)  # [1, N, 3]
    col = torch.from_numpy(np.maximum(x + 0.5, 0.0)[0]).requires_grad_(True)
    f8 = [torch.from_numpy(f64(p[k])).requires_grad_(True) for k in ("means", "quats", "scales", "opacities")]
    bg8 = torch.from_numpy(f64(bg_np[0])).requires_grad_(True)
    cam = U.Camera(kind, p["Ks"][0], W, H, **coeffs)
    oc, oa, margin = U.eval3d_render(f8[0], f8[1], f8[2], col, f8[3], p["viewmats"][0], cam, offs.cpu(), fl.cpu().tolist(),
                                     1, N, 0, background=bg8)
    ((oc * torch.from_numpy(f64(v_rc[0]))).sum() + (oa * torch.from_numpy(f64(v_ra[0]))).sum()).backward()
    v_col = col.grad.numpy() * (x[0] + 0.5 > 0)
    v_sh, v_means_dir = gso.spherical_harmonics_bwd(3, f64(p["means"]), f64(p["viewmats"]), f64(p["sh"]), masks, v_col[None])
    ref = {"means": f8[0].grad.numpy() + v_means_dir, "quats": f8[1].grad.numpy(), "scales": f8[2].grad.numpy(),
           "opacities": f8[3].grad.numpy(), "sh": v_sh, "backgrounds": bg8.grad.numpy()[None]}

    # the budgets of test_ut_gpu.py::test_eval3d_forward_and_gradients_against_oracle
    clear = (margin > 1e-3).numpy()
    err = np.abs(rc[0].detach().cpu().numpy() - oc.detach().numpy()).max(-1)
    bad = err > 2e-4
    assert (bad & clear).sum() <= max(1, clear.size // 1000), (bad & clear).sum()
    assert (bad & ~clear).sum() <= max(8, clear.size // 50), (bad & ~clear).sum()
    aerr = np.abs(ra[0, ..., 0].detach().cpu().numpy() - oa[..., 0].detach().numpy())
    assert ((aerr > 2e-4) & clear).sum() <= max(1, clear.size // 1000)
    got = {**{k: v.grad for k, v in L.items()}, "backgrounds": bg.grad}
    for k, r in ref.items():
        g, gr = got[k].detach().cpu().numpy().reshape(-1), r.reshape(-1)
        rel = np.linalg.norm(g - gr) / max(np.linalg.norm(gr), 1e-12)
        assert rel < 2e-2, (k, rel)


# ---- 3. against the reference's own orchestrator (make_ref_ut_rasterization_golden.py)
from tests.test_ut_rasterization_cpu import REF_RASTER_CAMERAS  # noqa: E402


def _tile_lists(offsets, flatten_ids, drop):
    """Each (image, tile)'s list of pair ids, without the ids in ``drop``."""
    offs = offsets.reshape(-1).tolist() + [len(flatten_ids)]
    ids = flatten_ids.tolist()
    return [[i for i in ids[offs[k]:offs[k + 1]] if i not in drop] for k in range(len(offs) - 1)]


@pytest.mark.parametrize("name", REF_RASTER_CAMERAS)
def test_against_reference_orchestrator(name):
    z = np.load(REF_NPZ)
    Wr, Hr, C = int(z["width"]), int(z["height"]), z["viewmats"].shape[0]
    model = "fisheye" if name.startswith("fisheye") else "pinhole"
    co = {k: _t(z[f"{name}/{k}"]) for k in KEYS.values() if f"{name}/{k}" in z.files}
    L = {k: _t(z[k], True) for k in ("means", "quats", "scales", "opacities", "sh")}
    bg = _t(z["backgrounds"], True)
    rc, ra, meta = gs.rasterization(
        L["means"], L["quats"], L["scales"], L["opacities"], L["sh"], _t(z["viewmats"]), _t(z["Ks"]), Wr, Hr,
        sh_degree=int(z["sh_degree"]), packed=False, tile_size=16, backgrounds=bg, render_mode="RGB+ED", with_ut=True,
        with_eval3d=True, camera_model=model, **co,
    )
    ((rc * _t(z["v_render_colors"])).sum() + (ra * _t(z["v_render_alphas"])).sum()).backward()
    N = len(z["means"])
    # radii are exact except where the unrounded radius sits on an integer (two float32 evaluations may round apart)
    radii, ref_radii = meta["radii"].cpu().numpy(), z[f"{name}/radii"]
    diff = (radii != ref_radii).any(-1)  # [C, N]
    for c in range(C):
        coeffs = {short: z[f"{name}/{k}"][c] for short, k in KEYS.items() if f"{name}/{k}" in z.files}
        o = U.ut_projection(z["means"], z["quats"], z["scales"], z["opacities"], z["viewmats"][c],
                            U.Camera(model, z["Ks"][c], Wr, Hr, **coeffs))
        frac = o["radii_unrounded"].numpy()
        on_edge = (np.abs(frac - np.round(frac)) < 1e-3).any(-1)
        assert (diff[c] & ~on_edge).sum() == 0 and diff[c].sum() <= max(2, N // 100), diff[c].sum()
    # tile lists: the same radius boxes sorted by depth per tile; only the pairs of a row rounded apart may differ
    drop = set((np.nonzero(diff.reshape(-1))[0]).tolist())
    got = _tile_lists(meta["isect_offsets"].cpu().numpy(), meta["flatten_ids"].cpu().numpy(), drop)
    ref = _tile_lists(z[f"{name}/isect_offsets"], z[f"{name}/flatten_ids"], drop)
    assert got == ref
    if not drop:
        assert np.array_equal(meta["isect_offsets"].cpu().numpy(), z[f"{name}/isect_offsets"])
        assert np.array_equal(meta["flatten_ids"].cpu().numpy(), z[f"{name}/flatten_ids"])
    vis = (ref_radii > 0).all(-1) & ~diff
    np.testing.assert_allclose(meta["means2d"].cpu().numpy()[vis], z[f"{name}/means2d"][vis], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(meta["depths"].cpu().numpy()[vis], z[f"{name}/depths"][vis], rtol=1e-5)

    # colours (RGB) and alphas with the tolerances test_ut_gpu.py applies to ref_ut.npz; the oracle's margins mark the
    # pixels with a decision near a threshold
    f8 = [torch.from_numpy(np.asarray(z[k], np.float64)) for k in ("means", "quats", "scales")]
    zero_cols = torch.zeros(C * N, 1, dtype=torch.float64)
    opac8 = torch.from_numpy(np.tile(z["opacities"].astype(np.float64), C))
    got_c, got_a = rc.detach().cpu().numpy(), ra.detach().cpu().numpy()
    ref_c, ref_a = z[f"{name}/render_colors"], z[f"{name}/render_alphas"]
    for c in range(C):
        coeffs = {short: z[f"{name}/{k}"][c] for short, k in KEYS.items() if f"{name}/{k}" in z.files}
        cam = U.Camera(model, z["Ks"][c], Wr, Hr, **coeffs)
        _, _, margin = U.eval3d_render(*f8, zero_cols, opac8, z["viewmats"][c], cam, torch.from_numpy(z[f"{name}/isect_offsets"]),
                                       z[f"{name}/flatten_ids"].tolist(), C, N, c)
        clear = (margin > 1e-3).numpy()
        err = np.abs(got_c[c, ..., :3] - ref_c[c, ..., :3]).max(-1)
        aerr = np.abs(got_a[c, ..., 0] - ref_a[c, ..., 0])
        assert ((err > 2e-4) & clear).sum() == 0 and ((aerr > 2e-4) & clear).sum() == 0, ((err > 2e-4) & clear).sum()
        assert ((err > 2e-4) & ~clear).sum() <= max(4, clear.size // 100)
        # expected depth: depth / alpha, relative to the depth, where the pixel is covered
        cov = clear & (ref_a[c, ..., 0] > 0.05)
        derr = np.abs(got_c[c, ..., 3] - ref_c[c, ..., 3]) / np.maximum(np.abs(ref_c[c, ..., 3]), 1e-6)
        assert (derr[cov] < 1e-3).all(), derr[cov].max()
    for k, leaf in list(L.items()) + [("backgrounds", bg)]:
        g, gr = leaf.grad.detach().cpu().numpy().reshape(-1), z[f"{name}/v_{k}"].reshape(-1)
        rel = np.linalg.norm(g - gr) / max(np.linalg.norm(gr), 1e-12)
        assert rel < 2e-2, (k, rel)


# ---- 4. render modes
def test_render_modes():
    p = _scene(1)
    kind, coeffs = CAMS[1]
    co = _coeffs(coeffs)
    L = _leaves(p, "sh", grad=False)
    bg = torch.rand(1, 3, device=DEV)
    rgb, a, meta = _rasterize(L, p, kind, co, backgrounds=bg)
    rgbd, a_d, _ = _rasterize(L, p, kind, co, backgrounds=bg, render_mode="RGB+D")
    rgbed, a_ed, _ = _rasterize(L, p, kind, co, backgrounds=bg, render_mode="RGB+ED")
    d, a_dd, _ = _rasterize(L, p, kind, co, backgrounds=bg, render_mode="D")
    ed, _, _ = _rasterize(L, p, kind, co, backgrounds=bg, render_mode="ED")
    assert rgbd.shape[-1] == 4 and rgbed.shape[-1] == 4 and d.shape[-1] == 1 and ed.shape[-1] == 1
    assert torch.equal(rgbd[..., :3], rgb) and torch.equal(rgbed[..., :3], rgb)
    for x in (a_d, a_ed, a_dd):
        assert torch.equal(x, a)
    # D: the eval3d compositing of the projection's depths, on a zero background
    comp, _ = gs.rasterize_to_pixels_eval3d(
        L["means"], L["quats"], L["scales"], meta["depths"][..., None], meta["opacities"], _t(p["viewmats"]), _t(p["Ks"]),
        W, H, 16, meta["isect_offsets"], meta["flatten_ids"], backgrounds=torch.zeros(1, 1, device=DEV), camera_model=kind,
        **co,
    )
    assert torch.equal(d, comp) and torch.equal(rgbd[..., 3:], comp)
    assert torch.equal(ed, d / a.clamp(min=1e-10)) and torch.equal(rgbed[..., 3:], ed)
    assert (a > 0).any() and (d > 0).any()


# ---- 5. channels: chunks and padding
def test_channel_chunks_and_padding():
    p = _scene(1)
    kind, coeffs = CAMS[5]
    co = _coeffs(coeffs)
    L = _leaves(p, "sh", grad=False)
    N = len(p["means"])
    g = torch.Generator(device="cpu").manual_seed(5)
    feat = torch.rand((N, 40), generator=g).to(DEV)
    bg = torch.rand((1, 40), generator=g).to(DEV)

    def run(f, b):
        return _rasterize({**L, "colors": f.contiguous()}, p, kind, co, colour="colors", backgrounds=b.contiguous())

    f40, a40, _ = run(feat, bg)
    f32, a32, _ = run(feat[:, :32], bg[:, :32])
    assert f40.shape[-1] == 40 and torch.equal(f40[..., :32], f32)
    f8, a8, _ = run(torch.nn.functional.pad(feat[:, :6], (0, 2)), torch.nn.functional.pad(bg[:, :6], (0, 2)))
    for D in (6, 7):
        fD, aD, _ = run(feat[:, :D], bg[:, :D])
        padded, _, _ = run(torch.nn.functional.pad(feat[:, :D], (0, 8 - D)), torch.nn.functional.pad(bg[:, :D], (0, 8 - D)))
        assert fD.shape[-1] == D and torch.equal(fD, padded[..., :D])
        assert torch.equal(aD, a40)
    assert torch.equal(f8[..., :6], run(feat[:, :6], bg[:, :6])[0])
    for x in (a32, a8):
        assert torch.equal(x, a40)
    assert (a40 > 0).any()


# ---- 6. batch dims and cameras
def test_batch_dims_and_cameras():
    p = _scene(2, n=300)
    kind, coeffs = CAMS[1]
    N = len(p["means"])
    means = np.stack([p["means"], p["means"] + 0.01])
    quats, scales, opac = (np.stack([p[k]] * 2) for k in ("quats", "scales", "opacities"))
    vm, K = np.stack([p["viewmats"]] * 2), np.stack([p["Ks"]] * 2)
    rng = np.random.RandomState(9)
    colors = rng.random_sample((2, 2, N, 3)).astype(np.float32)
    bg = rng.random_sample((2, 2, 3)).astype(np.float32)
    co = {KEYS[k]: np.tile(np.float32(v), (2, 2, 1)) for k, v in coeffs.items()}
    rc, ra, meta = gs.rasterization(
        _t(means), _t(quats), _t(scales), _t(opac), _t(colors), _t(vm), _t(K), W, H, packed=False, backgrounds=_t(bg),
        with_ut=True, with_eval3d=True, camera_model=kind, **{k: _t(v) for k, v in co.items()},
    )
    assert rc.shape == (2, 2, H, W, 3) and ra.shape == (2, 2, H, W, 1)
    assert meta["n_batches"] == 2 and meta["n_cameras"] == 2 and meta["isect_offsets"].shape == (2, 2, TH, TW)
    for b in range(2):
        for c in range(2):
            one_c, one_a, _ = gs.rasterization(
                _t(means[b]), _t(quats[b]), _t(scales[b]), _t(opac[b]), _t(colors[b, c : c + 1]), _t(vm[b, c : c + 1]),
                _t(K[b, c : c + 1]), W, H, packed=False, backgrounds=_t(bg[b, c : c + 1]), with_ut=True, with_eval3d=True,
                camera_model=kind, **{k: _t(v[b, c : c + 1]) for k, v in co.items()},
            )
            assert torch.equal(one_c[0], rc[b, c]) and torch.equal(one_a[0], ra[b, c]), (b, c)
            assert (one_a > 0).any()


# ---- 7. edge cases
def test_all_culled_and_deterministic():
    p = _scene(1)
    kind, coeffs = CAMS[4]
    co = _coeffs(coeffs)
    L = _leaves(p, "sh")
    bg = torch.rand(1, 3, device=DEV)
    # a far plane in front of every Gaussian culls them all
    rc, ra, meta = _rasterize(L, p, kind, co, backgrounds=bg, far_plane=1e-3)
    assert meta["flatten_ids"].numel() == 0 and (meta["radii"] == 0).all()
    assert torch.equal(rc, bg[:, None, None, :].expand(1, H, W, 3)) and (ra == 0).all()
    (rc.sum() + ra.sum()).backward()
    for k, v in L.items():
        assert v.grad is not None and (v.grad == 0).all(), k
    # two runs give identical outputs
    L = _leaves(p, "sh", grad=False)
    a = _rasterize(L, p, kind, co, backgrounds=bg, render_mode="RGB+ED")
    b = _rasterize(L, p, kind, co, backgrounds=bg, render_mode="RGB+ED")
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(a[2]["flatten_ids"], b[2]["flatten_ids"]) and torch.equal(a[2]["isect_offsets"], b[2]["isect_offsets"])


# ---- 8. the drop-in: a 3DGUT call is served by the b200 kernels, an ftheta call goes to the package
def test_dropin_serves_3dgut(monkeypatch):
    from gsplat_b200 import dropin

    calls = []

    def stock_rasterization(*a, **k):
        calls.append(k.get("camera_model"))
        return "stock"

    Wm = types.ModuleType("gsplat.cuda._wrapper")
    for n in dropin._OPS:
        setattr(Wm, n, lambda *a, **k: None)
    Wm.adam = lambda *a, **k: None
    R = types.ModuleType("gsplat.rendering")
    R.rasterization = stock_rasterization
    G = types.ModuleType("gsplat")
    G.__file__ = "stub"
    rel = types.ModuleType("gsplat.relocation")
    rel.compute_relocation = lambda *a, **k: None
    sops = types.ModuleType("gsplat.strategy.ops")
    sops.compute_relocation = rel.compute_relocation
    for name, mod in (("gsplat", G), ("gsplat.cuda", types.ModuleType("gsplat.cuda")), ("gsplat.cuda._wrapper", Wm),
                      ("gsplat.rendering", R), ("gsplat.relocation", rel), ("gsplat.strategy", types.ModuleType("gsplat.strategy")),
                      ("gsplat.strategy.ops", sops), ("gsplat.losses", types.ModuleType("gsplat.losses")),
                      ("gsplat.optimizers", types.ModuleType("gsplat.optimizers"))):
        monkeypatch.setitem(sys.modules, name, mod)
    dropin.apply(losses=False)
    try:
        st = dropin.stats["rasterization"]
        b0, s0 = st["b200"], st["stock"]
        p = _scene(1)
        kind, coeffs = CAMS[1]
        L = _leaves(p, "sh", grad=False)
        args = (L["means"], L["quats"], L["scales"], L["opacities"], L["sh"], _t(p["viewmats"]), _t(p["Ks"]), W, H)
        rc, ra, meta = R.rasterization(*args, sh_degree=3, packed=False, with_ut=True, with_eval3d=True, camera_model=kind,
                                       **_coeffs(coeffs))
        assert rc.shape == (1, H, W, 3) and (ra > 0).any()
        assert G.rasterization(*args, sh_degree=3, packed=False, with_ut=True, with_eval3d=True,
                               camera_model="ftheta") == "stock"
        assert calls == ["ftheta"]
        assert st["b200"] == b0 + 1 and st["stock"] == s0 + 1
    finally:
        dropin.undo()
    assert R.rasterization is stock_rasterization


# ---- 9. a short fit through a distorted pinhole
def test_fit_through_distorted_pinhole():
    p = _scene(2)
    kind, coeffs = CAMS[1]
    co = _coeffs(coeffs, (2,))
    vm, K = _t(p["viewmats"]), _t(p["Ks"])
    with torch.no_grad():
        gt, _, _ = gs.rasterization(_t(p["means"]), _t(p["quats"]), _t(p["scales"]), _t(p["opacities"]), _t(p["sh"]), vm, K,
                                    W, H, sh_degree=3, packed=False, with_ut=True, with_eval3d=True, camera_model=kind, **co)
    g = torch.Generator(device="cpu").manual_seed(13)
    N = len(p["means"])
    params = {
        "means": _t(p["means"] + 0.01 * torch.randn((N, 3), generator=g).numpy(), True),
        "quats": _t(p["quats"], True),
        "log_scales": _t(np.log(p["scales"] * 0.7), True),
        "logit_opac": _t(np.full(N, 0.0, np.float32), True),
        "sh": _t(np.concatenate([p["sh"][:, :1] * 0.3, np.zeros_like(p["sh"][:, 1:])], 1), True),
    }
    opt = torch.optim.Adam([
        {"params": [params["means"]], "lr": 2e-3}, {"params": [params["quats"]], "lr": 1e-2},
        {"params": [params["log_scales"]], "lr": 1e-2}, {"params": [params["logit_opac"]], "lr": 5e-2},
        {"params": [params["sh"]], "lr": 5e-2},
    ])
    losses = []
    for _ in range(100):
        rc, _, _ = gs.rasterization(
            params["means"], params["quats"], torch.exp(params["log_scales"]), torch.sigmoid(params["logit_opac"]),
            params["sh"], vm, K, W, H, sh_degree=3, packed=False, with_ut=True, with_eval3d=True, camera_model=kind, **co,
        )
        loss = (rc - gt).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(np.isfinite(losses))
    assert losses[-1] < 0.5 * losses[0], (losses[0], losses[-1])
