"""3DGUT operators without a GPU: the reference's signatures and defaults, every out-of-scope argument and malformed
input rejected before anything is launched, and the float64 oracle's camera models."""
import inspect
import json
import math
import os

import pytest
import torch

import gsplat_b200 as gs
from oracle import ut as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("fully_fused_projection_with_ut", "rasterize_to_pixels_eval3d")


@pytest.mark.parametrize("fn", NAMES)
def test_signature_and_defaults_match_reference(fn):
    with open(os.path.join(ROOT, "tests", "golden", "ref_signatures_ut.json")) as f:
        ref = json.load(f)["params"][fn]
    p = inspect.signature(getattr(gs, fn)).parameters
    assert list(p) == ref["params"]
    for name, src in ref["defaults"].items():
        want = 4 if src == "RollingShutterType.GLOBAL" else eval(src)  # GLOBAL is 4 in the reference's IntEnum
        assert p[name].default == want, name
    assert fn in gs.__all__
    assert gs.has_3dgut() is False


def _scene(B=(), C=1, N=4):
    z = torch.zeros
    means, quats, scales = z(B + (N, 3)), z(B + (N, 4)), torch.ones(B + (N, 3))
    quats[..., 0] = 1
    vm = torch.eye(4).expand(B + (C, 4, 4)).clone()
    K = torch.tensor([[50.0, 0, 16], [0, 50.0, 16], [0, 0, 1]]).expand(B + (C, 3, 3)).clone()
    return means, quats, scales, vm, K


def _proj(**kw):
    m, q, s, vm, K = _scene()
    return gs.fully_fused_projection_with_ut(m, q, s, None, vm, K, 32, 32, **kw)


def _eval(**kw):
    m, q, s, vm, K = _scene()
    colors, opac = torch.zeros(1, 4, 3), torch.ones(1, 4)
    offs, ids = torch.zeros(1, 2, 2, dtype=torch.int32), torch.zeros(0, dtype=torch.int32)
    args = dict(means=m, quats=q, scales=s, colors=colors, opacities=opac, viewmats=vm, Ks=K, image_width=32, image_height=32,
                tile_size=16, isect_offsets=offs, flatten_ids=ids)
    args.update(kw)
    return gs.rasterize_to_pixels_eval3d(**args)


OUT_OF_SCOPE = [
    ("ftheta_coeffs", dict(ftheta_coeffs=object())),
    ("lidar_coeffs", dict(lidar_coeffs=object())),
    ("external_distortion_coeffs", dict(external_distortion_coeffs=object())),
    ("rolling_shutter", dict(rolling_shutter=0)),
    ("viewmats_rs", dict(viewmats_rs=torch.eye(4)[None])),
    ("ortho", dict(camera_model="ortho")),
    ("ftheta", dict(camera_model="ftheta")),
    ("lidar", dict(camera_model="lidar")),
]


@pytest.mark.parametrize("name,kw", OUT_OF_SCOPE + [("global_z_order", dict(global_z_order=False))])
def test_projection_rejects_out_of_scope(name, kw):
    with pytest.raises(NotImplementedError, match=name):
        _proj(**kw)


class MixedBatch:
    pass


class ParallelBatch:
    pass


MixedBatch.__name__ = "RendererConfig_MixedBatch"
ParallelBatch.__name__ = "RendererConfig_ParallelBatch"


@pytest.mark.parametrize(
    "name,kw",
    OUT_OF_SCOPE
    + [
        ("rays", dict(rays=torch.zeros(1, 32, 32, 6))),
        ("use_hit_distance", dict(use_hit_distance=True)),
        ("return_normals", dict(return_normals=True)),
        ("renderer_config", dict(renderer_config=ParallelBatch())),
        ("packed", dict(colors=torch.zeros(4, 3), opacities=torch.ones(4))),
    ],
)
def test_eval3d_rejects_out_of_scope(name, kw):
    with pytest.raises(NotImplementedError, match=name):
        _eval(**kw)


def test_mixed_batch_config_passes_checks():
    # accepted up to the device check: CPU tensors are refused by the library, not by the scope checks
    with pytest.raises(gs._cabi.GsplatB200Error):
        _eval(renderer_config=MixedBatch())


@pytest.mark.parametrize(
    "kw,exc",
    [
        (dict(radial_coeffs=torch.zeros(1, 5)), ValueError),
        (dict(tangential_coeffs=torch.zeros(1, 3)), ValueError),
        (dict(thin_prism_coeffs=torch.zeros(2, 4)), ValueError),
        (dict(camera_model="fisheye", radial_coeffs=torch.zeros(1, 6)), ValueError),
        (dict(camera_model="fisheye", tangential_coeffs=torch.zeros(1, 2)), ValueError),
        (dict(camera_model="nope"), ValueError),
        (dict(radial_coeffs=torch.zeros(1, 6, dtype=torch.float64)), TypeError),
        (dict(ut_params=type("P", (), {"alpha": 0.0})()), ValueError),
    ],
)
def test_bad_camera_arguments(kw, exc):
    with pytest.raises(exc):
        _proj(**kw)
    with pytest.raises(exc):
        _eval(**kw)


def test_bad_shapes_and_dtypes():
    m, q, s, vm, K = _scene()
    with pytest.raises(ValueError):
        gs.fully_fused_projection_with_ut(m, q[:, :3], s, None, vm, K, 32, 32)
    with pytest.raises(ValueError):
        gs.fully_fused_projection_with_ut(m, q, s, torch.ones(3), vm, K, 32, 32)
    with pytest.raises(TypeError):
        gs.fully_fused_projection_with_ut(m.double(), q, s, None, vm, K, 32, 32)
    with pytest.raises(ValueError):
        _eval(colors=torch.zeros(1, 3, 3))
    with pytest.raises(ValueError):
        _eval(opacities=torch.ones(1, 5))
    with pytest.raises(ValueError):
        _eval(backgrounds=torch.zeros(1, 4))
    with pytest.raises(ValueError):
        _eval(masks=torch.ones(1, 3, 2, dtype=torch.bool))
    with pytest.raises(ValueError):
        _eval(isect_offsets=torch.zeros(1, 1, 1, dtype=torch.int32))
    with pytest.raises(ValueError):
        _eval(flatten_ids=torch.zeros(0, dtype=torch.int64))
    with pytest.raises(ValueError):
        _eval(tile_size=8)
    with pytest.raises(NotImplementedError):
        _eval(colors=torch.zeros(1, 4, 7))
    with pytest.raises(TypeError):
        _eval(colors=torch.zeros(1, 4, 3, dtype=torch.float64))


def test_ut_params_any_object_and_defaults():
    class P:
        alpha, beta, kappa = 0.5, 1.0, 1.0

    assert gs.ops._ut_params(None) == (0.1, 2.0, 0.0, 0.1, False)
    assert gs.ops._ut_params(P()) == (0.5, 1.0, 1.0, 0.1, False)


CAMERAS = [
    ("pinhole", {}),
    ("pinhole", dict(radial=[0.1, -0.05, 0.01, 0.02, 0.0, 0.0])),
    ("pinhole", dict(tangential=[0.01, -0.005])),
    ("pinhole", dict(thin=[0.002, -0.001, 0.001, 0.0005])),
    ("pinhole", dict(radial=[0.1, -0.05, 0.01, 0.02, 0.0, 0.0], tangential=[0.01, -0.005], thin=[0.002, -0.001, 0.001, 0.0005])),
    ("fisheye", {}),
    ("fisheye", dict(radial=[0.05, -0.01, 0.002, -0.0003])),
]


@pytest.mark.parametrize("kind,coeffs", CAMERAS)
def test_oracle_camera_round_trip(kind, coeffs):
    W, H = 320, 240
    cam = U.Camera(kind, [[200.0, 0, 161.0], [0, 205.0, 119.0], [0, 0, 1]], W, H, **coeffs)
    u, v = torch.meshgrid(torch.linspace(0.5, W - 0.5, 23, dtype=U.F64), torch.linspace(0.5, H - 0.5, 17, dtype=U.F64), indexing="xy")
    d, ok = cam.unproject(u.reshape(-1), v.reshape(-1))
    assert ok.all()
    assert torch.allclose(d.norm(dim=-1), torch.ones(len(d), dtype=U.F64))
    uv, valid = cam.project(d * 3.0, 0.1)
    assert valid.all()
    err = (uv - torch.stack([u.reshape(-1), v.reshape(-1)], -1)).abs().max()
    assert err < 1e-6, err


# ---- the float64 oracle against the reference's own outputs (tests/golden/ref_ut.npz, make_ref_ut_golden.py)
REF_NPZ = os.path.join(ROOT, "tests", "golden", "ref_ut.npz")
REF_CAMERAS = ["pinhole", "pinhole_radial", "pinhole_tangential", "pinhole_thin_prism", "fisheye", "fisheye_radial"]
_KEYS = {"radial_coeffs": "radial", "tangential_coeffs": "tangential", "thin_prism_coeffs": "thin"}


def ref_case(z, name):
    model = "fisheye" if name.startswith("fisheye") else "pinhole"
    coeffs = {short: z[f"{name}/{k}"][0] for k, short in _KEYS.items() if f"{name}/{k}" in z.files}
    return model, coeffs


@pytest.mark.parametrize("name", REF_CAMERAS)
def test_oracle_reproduces_reference(name):
    import numpy as np

    z = np.load(REF_NPZ)
    W, H = int(z["width"]), int(z["height"])
    model, coeffs = ref_case(z, name)
    cam = U.Camera(model, z["Ks"][0], W, H, **coeffs)
    o = U.ut_projection(z["means"], z["quats"], z["scales"], z["opacities"], z["viewmats"][0], cam)
    r, ro = z[f"{name}/radii"][0], o["radii"].numpy()
    frac = o["radii_unrounded"].numpy()
    on_edge = (np.abs(frac - np.round(frac)) < 1e-3).any(-1)
    diff = (r != ro).any(-1)
    # radii differ only where a radius sits on an integer boundary (float32 against float64 rounding)
    assert (diff & ~on_edge).sum() == 0 and diff.sum() <= max(2, len(r) // 100), (diff.sum(), (diff & ~on_edge).sum())
    ok = (r > 0).all(-1) & (ro > 0).all(-1)
    assert ok.sum() > 100
    np.testing.assert_allclose(o["means2d"].numpy()[ok], z[f"{name}/means2d"][0][ok], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(o["depths"].numpy()[ok], z[f"{name}/depths"][0][ok], rtol=1e-5)
    cref = z[f"{name}/conics"][0][ok]
    np.testing.assert_allclose(o["conics"].numpy()[ok], cref, rtol=2e-3, atol=2e-3 * np.abs(cref).max())

    N = len(z["means"])
    f8 = [torch.from_numpy(np.asarray(z[k], np.float64)).requires_grad_(True) for k in ("means", "quats", "scales")]
    f8 += [torch.from_numpy(z["colors"].astype(np.float64)).requires_grad_(True),
           torch.from_numpy(z["opacities"].astype(np.float64)).requires_grad_(True),
           torch.from_numpy(z["backgrounds"][0].astype(np.float64)).requires_grad_(True)]
    offs = torch.from_numpy(z[f"{name}/isect_offsets"])
    fl = z[f"{name}/flatten_ids"].tolist()
    oc, oa, margin = U.eval3d_render(*f8[:5], z["viewmats"][0], cam, offs, fl, 1, N, 0, background=f8[5])
    v_rc, v_ra = z["v_render_colors"][0].astype(np.float64), z["v_render_alphas"][0].astype(np.float64)
    ((oc * torch.from_numpy(v_rc)).sum() + (oa * torch.from_numpy(v_ra)).sum()).backward()
    clear = (margin > 1e-3).numpy()
    err = np.abs(oc.detach().numpy() - z[f"{name}/render_colors"][0]).max(-1)
    aerr = np.abs(oa.detach().numpy()[..., 0] - z[f"{name}/render_alphas"][0][..., 0])
    # pixels whose decisions are all clear of a threshold agree to float32 accuracy; marginal pixels are counted
    assert ((err > 2e-4) & clear).sum() == 0, ((err > 2e-4) & clear).sum()
    assert ((aerr > 2e-4) & clear).sum() == 0
    assert ((err > 2e-4) & ~clear).sum() <= max(4, clear.size // 100)
    assert oa.detach().numpy().mean() > 0.02
    for k, leaf in zip(("means", "quats", "scales", "colors", "opacities", "backgrounds"), f8):
        g, gr = leaf.grad.numpy().reshape(-1), z[f"{name}/v_{k}"].reshape(-1)
        rel = np.linalg.norm(g - gr) / max(np.linalg.norm(gr), 1e-12)
        assert rel < 2e-2, (k, rel)


# ---- the drop-in: both names rebound where the package has them, out-of-scope calls handed to the package's op
def test_dropin_rebinds_and_delegates(monkeypatch):
    import sys
    import types

    from gsplat_b200 import dropin

    calls = []

    def stock_proj(*a, **k):
        calls.append("proj")
        return "stock-proj"

    def stock_eval(*a, **k):
        calls.append("eval")
        return "stock-eval"

    W = types.ModuleType("gsplat.cuda._wrapper")
    for n in dropin._OPS:
        setattr(W, n, lambda *a, **k: None)
    W.adam = lambda *a, **k: None
    W.fully_fused_projection_with_ut = stock_proj
    W.rasterize_to_pixels_eval3d = stock_eval
    R = types.ModuleType("gsplat.rendering")
    R.rasterization = lambda *a, **k: None
    G = types.ModuleType("gsplat")
    G.__file__ = "stub"
    G.fully_fused_projection_with_ut = stock_proj
    rel = types.ModuleType("gsplat.relocation")
    rel.compute_relocation = lambda *a, **k: None
    sops = types.ModuleType("gsplat.strategy.ops")
    sops.compute_relocation = rel.compute_relocation
    cuda = types.ModuleType("gsplat.cuda")
    strat = types.ModuleType("gsplat.strategy")
    losses = types.ModuleType("gsplat.losses")
    opt = types.ModuleType("gsplat.optimizers")
    for name, mod in (("gsplat", G), ("gsplat.cuda", cuda), ("gsplat.cuda._wrapper", W), ("gsplat.rendering", R),
                      ("gsplat.relocation", rel), ("gsplat.strategy", strat), ("gsplat.strategy.ops", sops),
                      ("gsplat.losses", losses), ("gsplat.optimizers", opt)):
        monkeypatch.setitem(sys.modules, name, mod)
    dropin.apply(losses=False)
    try:
        assert W.fully_fused_projection_with_ut.__gsb200_ours__ is gs.fully_fused_projection_with_ut
        assert G.fully_fused_projection_with_ut is W.fully_fused_projection_with_ut
        assert W.rasterize_to_pixels_eval3d.__gsb200_ours__ is gs.rasterize_to_pixels_eval3d
        m, q, s, vm, K = _scene()
        # out of scope for the b200 kernels: the package's own op runs
        assert W.fully_fused_projection_with_ut(m, q, s, None, vm, K, 32, 32, camera_model="ftheta") == "stock-proj"
        assert W.rasterize_to_pixels_eval3d(m, q, s, torch.zeros(1, 4, 3), torch.ones(1, 4), vm, K, 32, 32, 16,
                                            torch.zeros(1, 2, 2, dtype=torch.int32), torch.zeros(0, dtype=torch.int32),
                                            rays=torch.zeros(1, 32, 32, 6)) == "stock-eval"
        assert calls == ["proj", "eval"]
    finally:
        dropin.undo()
    assert W.fully_fused_projection_with_ut is stock_proj and W.rasterize_to_pixels_eval3d is stock_eval
