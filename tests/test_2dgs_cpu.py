"""2DGS without a GPU: the float64 oracle (oracle/surfel.py) against the reference's own PyTorch twins
(tests/golden/ref_2dgs.npz, written by tests/golden/make_golden_2dgs.py) and against central finite differences, the
public signatures against the reference's, the host-side argument checks, and the drop-in rebinding on a stub package."""
import ast
import importlib
import json
import os
import sys
import textwrap

import numpy as np
import pytest
import torch

from oracle import surfel

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
f64 = torch.float64


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(ROOT, "tests", "golden", "ref_2dgs.npz"))


def _t(a, grad=False):
    return torch.tensor(np.asarray(a), dtype=f64, requires_grad=grad)


def test_projection_matches_reference_twin(ref):
    """Allowed differences: the twin never culls on radius_clip (0 here) and culls |distance| <= eps instead of
    distance == 0 (no row is degenerate here); near / far are strict in both.  The twin's normal is the third column of
    R rot(q) diag(s): scaled by scales[..., 2], which the kernels (and the oracle) leave out, so that the normal is a unit
    vector.  The twin's normals are compared divided by that scale, its normals cotangent is handed to the oracle
    multiplied by it, and the twin's v_scales[..., 2] (from the normals alone) is not compared: the oracle's is zero."""
    s2 = ref["p_scales"][..., 2]
    ins = {k: _t(ref["p_" + k], True) for k in ("means", "quats", "scales", "viewmats")}
    W, H = int(ref["p_width"]), int(ref["p_height"])
    radii, m2, dep, rt, nrm = surfel.project(ins["means"], ins["quats"], ins["scales"], ins["viewmats"], _t(ref["p_Ks"]), W, H)
    np.testing.assert_array_equal(radii.numpy(), ref["p_radii"])
    vis = (ref["p_radii"] > 0).all(-1)
    assert 0 < vis.sum() < vis.size  # both visible and culled rows
    twin = dict((k, ref["p_" + k]) for k in ("means2d", "depths", "ray_transforms"))
    twin["normals"] = ref["p_normals"] / s2[None, :, None]
    for name, a in (("means2d", m2), ("depths", dep), ("ray_transforms", rt), ("normals", nrm)):
        np.testing.assert_allclose(a.detach().numpy()[vis], twin[name][vis], rtol=1e-10, atol=1e-12, err_msg=name)
    cot = {n: _t(ref["p_v_" + n]) for n in ("means2d", "depths", "ray_transforms", "normals")}
    cot["normals"] = cot["normals"] * _t(s2)[None, :, None]
    loss = sum((a * cot[n]).sum() for n, a in (("means2d", m2), ("depths", dep), ("ray_transforms", rt), ("normals", nrm)))
    grads = torch.autograd.grad(loss, [ins[k] for k in ("means", "quats", "scales", "viewmats")])
    for k, g in zip(("means", "quats", "scales", "viewmats"), grads):
        g, want = g.numpy(), ref["p_g_" + k]
        if k == "scales":
            assert np.all(g[..., 2] == 0)
            g, want = g[..., :2], want[..., :2]
        np.testing.assert_allclose(g, want, rtol=1e-9, atol=1e-10, err_msg=k)


def test_compositing_matches_reference_twin(ref):
    """The twin (accumulate_2dgs) composites the pair list it is given, with no alpha threshold and no transmittance
    stop; the fixture's pair list is every pair with alpha >= 1/255 and no pixel comes near the stop (its smallest
    transmittance is stored).  The oracle takes both decisions itself from the radius-box tile lists."""
    assert float(ref["c_min_transmittance"]) > 10 * surfel.TRANSMITTANCE_THRESHOLD
    W, H = int(ref["c_width"]), int(ref["c_height"])
    ins = {k: _t(ref["c_" + k], True) for k in ("means2d", "ray_transforms", "opacities", "colors", "normals")}
    tw, th = -(-W // 16), -(-H // 16)
    fl, off = surfel.isect(ref["c_means2d"], ref["c_radii"], ref["c_depths"], 16, tw, th)
    out = surfel.rasterize(ins["means2d"], ins["ray_transforms"], ins["colors"], ins["opacities"], ins["normals"], W, H, 16, off, fl)
    for name in ("colors", "alphas", "normals"):
        np.testing.assert_allclose(out["render_" + name].detach().numpy(), ref["c_render_" + name], rtol=1e-10, atol=1e-12, err_msg=name)
    loss = sum((out["render_" + n] * _t(ref["c_v_render_" + n])).sum() for n in ("colors", "alphas", "normals"))
    keys = ("means2d", "ray_transforms", "opacities", "colors", "normals")
    grads = torch.autograd.grad(loss, [ins[k] for k in keys])
    for k, g in zip(keys, grads):
        np.testing.assert_allclose(g.numpy(), ref["c_g_" + k], rtol=1e-8, atol=1e-10, err_msg=k)
    # the tile-by-tile vjp gives the same gradients
    cot = [_t(ref["c_v_render_colors"]), _t(ref["c_v_render_alphas"]), _t(ref["c_v_render_normals"]), None, None]
    vj = surfel.rasterize_vjp(*(ins[k] for k in ("means2d", "ray_transforms", "colors", "opacities", "normals")), W, H, 16, off, fl, cot)
    for k, g in zip(keys, grads):
        np.testing.assert_allclose(vj["v_" + k].numpy(), g.numpy(), rtol=1e-12, atol=1e-14, err_msg=k)


def _fd_scene():
    """Three surfels facing the camera, overlapping, 20 x 12 pixels; one camera."""
    means = torch.tensor([[0.02, 0.01, 2.0], [-0.05, 0.02, 2.4], [0.04, -0.03, 2.9]], dtype=f64)
    quats = torch.tensor([[1.0, 0.1, -0.05, 0.2], [0.9, -0.1, 0.15, 0.05], [1.0, 0.05, 0.1, -0.3]], dtype=f64)
    scales = torch.tensor([[0.05, 0.03, 0.01], [0.04, 0.06, 0.01], [0.07, 0.05, 0.01]], dtype=f64)
    vm = torch.eye(4, dtype=f64)[None]
    vm[0, :3, 3] = torch.tensor([0.01, -0.02, 0.05], dtype=f64)
    Ks = torch.tensor([[[70.0, 0, 10.0], [0, 70.0, 6.0], [0, 0, 1]]], dtype=f64)
    opac = torch.tensor([0.7, 0.5, 0.9], dtype=f64)
    colors = torch.tensor([[0.2, 0.8, 1.9], [0.6, 0.1, 2.3], [0.9, 0.4, 3.1]], dtype=f64)
    return means, quats, scales, vm, Ks, opac, colors


def test_oracle_autograd_matches_finite_differences():
    """Every output of the chain projection -> compositing, distortion and median depth included, differentiated by
    autograd and by central differences, on a scene whose pixels keep away from every threshold (checked)."""
    means, quats, scales, vm, Ks, opac, colors = _fd_scene()
    W, H = 20, 12
    with torch.no_grad():
        radii, m2, dep, _, _ = surfel.project(means, quats, scales, vm, Ks, W, H)
    assert (radii > 0).all()
    fl, off = surfel.isect(m2.numpy(), radii.numpy(), dep.numpy(), 16, 2, 1)

    def chain(mn, q, s, v, o, c):
        _, m2_, _, rt_, nrm_ = surfel.project(mn, q, s, v, Ks, W, H)
        return surfel.rasterize(m2_, rt_, c[None], o[None], nrm_, W, H, 16, off, fl)

    base = chain(means, quats, scales, vm, opac, colors)
    assert base["margins"].min() > 1e-3 and base["grad_margins"].min() > 1e-4  # far beyond what a step of 1e-6 moves
    assert (base["render_alphas"] > 0).double().mean() > 0.3 and base["render_distort"].abs().sum() > 0
    gen = torch.Generator().manual_seed(0)
    leaves = [means, quats, scales, vm, opac, colors]
    for name in surfel._OUT_NAMES:
        cot = torch.randn(base[name].shape, generator=gen, dtype=f64)
        xs = [x.clone().requires_grad_(True) for x in leaves]
        g = torch.autograd.grad((chain(*xs)[name] * cot).sum(), xs, allow_unused=True)
        for li, (x, gx) in enumerate(zip(leaves, g)):
            gx = torch.zeros_like(x) if gx is None else gx
            fd = torch.zeros_like(x).reshape(-1)
            for e in range(x.numel()):
                if li == 3 and e >= 12:  # the last row of the view matrix is not an input of the projection
                    continue
                h = 1e-6
                vals = []
                for sgn in (1.0, -1.0):
                    xp = [y.clone() for y in leaves]
                    xp[li].reshape(-1)[e] += sgn * h
                    vals.append(float((chain(*xp)[name] * cot).sum()))
                fd[e] = (vals[0] - vals[1]) / (2 * h)
            fd = fd.reshape(x.shape)
            gx = gx.clone()
            if li == 3:
                gx[..., 3, :] = 0
            np.testing.assert_allclose(gx.numpy(), fd.numpy(), rtol=2e-5, atol=2e-6, err_msg=f"{name} wrt leaf {li}")


def test_densify_gradient_identity():
    rt = torch.randn(2, 5, 3, 3, dtype=f64)
    v = torch.randn(2, 5, 3, 3, dtype=f64)
    np.testing.assert_array_equal(surfel.densify_grad(v, rt).numpy(), torch.stack([v[..., 0, 2], v[..., 1, 2]], -1).mul(rt[..., 2, 2, None]).numpy())


@pytest.mark.parametrize("fn", ["fully_fused_projection_2dgs", "rasterize_to_pixels_2dgs", "rasterization_2dgs"])
def test_same_parameters_as_reference(fn):
    with open(os.path.join(ROOT, "tests", "golden", "ref_signatures_2dgs.json")) as f:
        ref = json.load(f)["params"][fn]
    src = "rendering.py" if fn == "rasterization_2dgs" else "ops.py"
    tree = ast.parse(open(os.path.join(ROOT, "gsplat_b200", src)).read())
    node = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == fn)
    a = node.args
    assert [x.arg for x in a.posonlyargs + a.args + a.kwonlyargs] == ref["params"]
    assert len(a.defaults) == ref["n_defaults"]


def test_rasterization_2dgs_defaults_match_reference():
    import inspect

    import gsplat_b200

    p = inspect.signature(gsplat_b200.rasterization_2dgs).parameters
    assert (p["packed"].default, p["tile_size"].default, p["render_mode"].default, p["depth_mode"].default) == (False, 16, "RGB", "expected")
    assert gsplat_b200.has_2dgs()


def test_argument_checks_before_launch():
    import gsplat_b200 as gs

    z = torch.zeros
    N = 6
    proj = (z(N, 3), z(N, 4), z(N, 3), torch.eye(4)[None], torch.eye(3)[None], 32, 32)
    for kw in (dict(packed=True), dict(sparse_grad=True), dict(packed=True, sparse_grad=True)):
        with pytest.raises(NotImplementedError):
            gs.fully_fused_projection_2dgs(*proj, **kw)
        with pytest.raises(NotImplementedError):
            gs.rasterization_2dgs(z(N, 3), z(N, 4), z(N, 3), z(N), z(N, 3), torch.eye(4)[None], torch.eye(3)[None], 32, 32, **kw)
    with pytest.raises(ValueError):
        gs.fully_fused_projection_2dgs(z(N, 3), z(N + 1, 4), z(N, 3), *proj[3:])
    with pytest.raises(ValueError):
        gs.fully_fused_projection_2dgs(z(N, 3), z(N, 4), z(N, 3), torch.eye(4)[None], torch.eye(3)[None, :2], 32, 32)
    m2, rt, col, op, nrm, dens = z(1, N, 2), z(1, N, 3, 3), z(1, N, 3), z(1, N), z(1, N, 3), z(1, N, 2)
    off, fl = z(1, 2, 2, dtype=torch.int32), z(0, dtype=torch.int32)

    def rast(**kw):
        a = dict(means2d=m2, ray_transforms=rt, colors=col, opacities=op, normals=nrm, densify=dens, image_width=32,
                 image_height=32, tile_size=16, isect_offsets=off, flatten_ids=fl)
        a.update(kw)
        return gs.rasterize_to_pixels_2dgs(**a)

    with pytest.raises(NotImplementedError):
        rast(packed=True)
    with pytest.raises(NotImplementedError):  # 6 channels: not built, and depth is the last channel so no padding
        rast(colors=z(1, N, 6))
    for kw in (dict(ray_transforms=z(1, N, 9)), dict(opacities=z(1, N + 1)), dict(normals=z(1, N, 2)), dict(densify=z(1, N, 3)),
               dict(backgrounds=z(1, 4)), dict(masks=z(1, 3, 2, dtype=torch.bool)), dict(tile_size=8), dict(image_width=40),
               dict(means2d=z(2, N, 2))):
        with pytest.raises(ValueError):
            rast(**kw)
    args = (z(N, 3), z(N, 4), z(N, 3), z(N), z(N, 3), torch.eye(4)[None], torch.eye(3)[None], 32, 32)
    for kw in (dict(render_mode="bogus"), dict(depth_mode="mean"), dict(tile_size=8), dict(distloss=True)):
        with pytest.raises(ValueError):
            gs.rasterization_2dgs(*args, **kw)
    for mode in ("d", "Ed", "RGB-d", "RGB-Ed"):
        with pytest.raises(NotImplementedError):
            gs.rasterization_2dgs(*args, render_mode=mode)
    with pytest.raises(ValueError):
        gs.rasterization_2dgs(z(N, 3), z(N, 4), z(N, 3), z(N + 1), *args[4:])


_NAMES = ("fully_fused_projection_2dgs", "rasterize_to_pixels_2dgs")
_STUB = {
    "gsplat/__init__.py": """
        from .cuda._wrapper import *  # noqa
        from .rendering import rasterization, rasterization_2dgs
        """,
    "gsplat/cuda/__init__.py": "",
    "gsplat/cuda/_wrapper.py": """
        def _stock(name):
            def f(*a, **k):
                return ("stock", name)
            f.__name__ = name
            return f
        _NAMES = ["quat_scale_to_covar_preci", "fully_fused_projection", "spherical_harmonics", "isect_tiles",
                  "isect_offset_encode", "rasterize_to_pixels", "adam", "build_sparse_tile_layout", "isect_tiles_sparse",
                  "rasterize_to_pixels_sparse", "fully_fused_projection_2dgs", "rasterize_to_pixels_2dgs"]
        for _n in _NAMES:
            globals()[_n] = _stock(_n)
        __all__ = list(_NAMES)
        """,
    "gsplat/rendering.py": (
        "def rasterization(*a, **k):\n    return ('stock', 'rasterization')\n"
        "def rasterization_2dgs(*a, **k):\n    return ('stock', 'rasterization_2dgs')\n"
    ),
    "gsplat/relocation.py": "def compute_relocation(*a, **k):\n    return ('stock', 'compute_relocation')\n",
    "gsplat/strategy/__init__.py": "",
    "gsplat/strategy/ops.py": "from ..relocation import compute_relocation\ndef _cuda_fused_mcmc_perturb(*a, **k):\n    return False\n",
    "gsplat/optimizers/__init__.py": "class SelectiveAdam:\n    pass\n",
}


def test_dropin_rebinds_2dgs_names(tmp_path, monkeypatch):
    for rel, text in _STUB.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    monkeypatch.syspath_prepend(str(tmp_path))
    for m in [m for m in sys.modules if m == "gsplat" or m.startswith("gsplat.")]:
        monkeypatch.delitem(sys.modules, m)
    import gsplat_b200
    from gsplat_b200 import dropin

    G = importlib.import_module("gsplat")
    W = importlib.import_module("gsplat.cuda._wrapper")
    R = importlib.import_module("gsplat.rendering")
    stock = {n: getattr(W, n) for n in _NAMES}
    stock_r = R.rasterization_2dgs
    try:
        dropin.apply(losses=False)
        for n in _NAMES:
            for mod in (W, G):
                fn = getattr(mod, n)
                assert fn is not stock[n] and fn.__gsb200_ours__ is getattr(gsplat_b200, n)
        for mod in (R, G):
            assert mod.rasterization_2dgs.__gsb200_ours__ is gsplat_b200.rasterization_2dgs
        # packed calls are handed to the package's own implementation
        z = torch.zeros
        out = G.rasterization_2dgs(z(4, 3), z(4, 4), z(4, 3), z(4), z(4, 3), torch.eye(4)[None], torch.eye(3)[None], 32, 32, packed=True)
        assert out == ("stock", "rasterization_2dgs")
        out = W.fully_fused_projection_2dgs(z(4, 3), z(4, 4), z(4, 3), torch.eye(4)[None], torch.eye(3)[None], 32, 32, packed=True)
        assert out == ("stock", "fully_fused_projection_2dgs")
    finally:
        dropin.undo()
    for n in _NAMES:
        assert getattr(W, n) is stock[n] and getattr(G, n) is stock[n]
    assert R.rasterization_2dgs is stock_r and G.rasterization_2dgs is stock_r
