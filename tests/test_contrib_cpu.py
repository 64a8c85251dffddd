"""The per-pixel contributor queries without a GPU: the reference's signatures, every argument error raised on CPU
tensors before anything needs the device, the exports, the drop-in's rebinding and the top-K bound."""
import ast
import json
import os

import pytest
import torch

import gsplat_b200 as gs
from gsplat_b200 import _cabi, ops
from tests.test_indices_cpu import _BASE, _stub_package

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
NAMES = tuple(
    f"rasterize_{n}{s}"
    for n in ("num_contributing_gaussians", "contributing_gaussian_ids", "top_contributing_gaussian_ids")
    for s in ("", "_sparse")
)
I, N, W, H, AT, P = 2, 5, 40, 20, 3, 9


@pytest.mark.parametrize("fn", NAMES)
def test_same_parameters_as_reference(fn):
    with open(os.path.join(ROOT, "tests", "golden", "ref_signatures_contrib.json")) as f:
        ref = json.load(f)["params"][fn]
    tree = ast.parse(open(os.path.join(ROOT, "gsplat_b200", "ops.py")).read())
    node = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == fn)
    a = node.args
    assert [x.arg for x in a.posonlyargs + a.args + a.kwonlyargs] == ref["params"]
    assert len(a.defaults) == ref["n_defaults"]


def test_exported():
    for n in NAMES:
        assert n in gs.__all__ and callable(getattr(gs, n))


def _args(fn, packed=False):
    """well-formed CPU arguments of `fn` by parameter name"""
    z = torch.zeros
    lead = (7,) if packed else (I, N)
    a = dict(means2d=z(lead + (2,)), conics=z(lead + (3,)), opacities=z(lead), flatten_ids=z(11, dtype=torch.int32),
             image_width=W, image_height=H, tile_size=16, num_depth_samples=4)
    if fn.endswith("_sparse"):
        a.update(active_tiles=z(AT, dtype=torch.int32), tile_offsets=z(AT + 1, dtype=torch.int32),
                 tile_pixel_mask=z(AT, 4, dtype=torch.int64), tile_pixel_cumsum=z(AT, dtype=torch.int64),
                 pixel_map=z(P, dtype=torch.int64), tile_width=3, tile_height=2,
                 num_contributing_gaussians=z(P, dtype=torch.int32))
    else:
        a.update(tile_offsets=z(I, 2, 3, dtype=torch.int32), num_contributing_gaussians=z(I, H, W, dtype=torch.int32))
    return a


def _call(fn, **kw):
    a = _args(fn, kw.pop("packed", False))
    a.update(kw)
    f = getattr(gs, fn)
    params = [x.arg for x in next(n for n in ast.walk(ast.parse(open(os.path.join(ROOT, "gsplat_b200", "ops.py")).read()))
                                  if isinstance(n, ast.FunctionDef) and n.name == fn).args.args]
    return f(*(a[p] for p in params))


def _bad_values(fn):
    z = torch.zeros
    cases = [dict(tile_size=8), dict(means2d=z(I, N, 3)), dict(means2d=z(5)), dict(conics=z(I, N + 1, 3)),
             dict(conics=z(I, N, 2)), dict(opacities=z(I, N, 1)), dict(opacities=z(I, N - 1)),
             dict(flatten_ids=z(11, 1, dtype=torch.int32)), dict(image_width=W + 100)]
    if fn.endswith("_sparse"):
        cases += [dict(tile_offsets=z(AT, dtype=torch.int32)), dict(tile_pixel_mask=z(AT, 3, dtype=torch.int64)),
                  dict(tile_pixel_cumsum=z(AT + 1, dtype=torch.int64)), dict(active_tiles=z(AT, 1, dtype=torch.int32)),
                  dict(pixel_map=z(P, 1, dtype=torch.int64)), dict(tile_height=1)]
        if "_ids" in fn and "top" not in fn:
            cases += [dict(num_contributing_gaussians=z(P + 1, dtype=torch.int32))]
    else:
        cases += [dict(tile_offsets=z(I, 1, 3, dtype=torch.int32)), dict(tile_offsets=z(3, 2, 3, dtype=torch.int32)),
                  dict(tile_offsets=z(3, dtype=torch.int32)), dict(means2d=z(1, I, N, 2))]
        if "_ids" in fn and "top" not in fn:
            cases += [dict(num_contributing_gaussians=z(I, H, W + 1, dtype=torch.int32)),
                      dict(num_contributing_gaussians=z(H, W, dtype=torch.int32))]
    if "top" in fn:
        cases += [dict(num_depth_samples=0), dict(num_depth_samples=-3)]
    return cases


def _bad_types(fn):
    z = torch.zeros
    cases = [dict(means2d=z(I, N, 2, dtype=torch.float64)), dict(conics=z(I, N, 3, dtype=torch.float16)),
             dict(opacities=z(I, N, dtype=torch.float64)), dict(flatten_ids=z(11, dtype=torch.int64))]
    if fn.endswith("_sparse"):
        cases += [dict(tile_offsets=z(AT + 1, dtype=torch.int64)), dict(active_tiles=z(AT, dtype=torch.int64)),
                  dict(tile_pixel_mask=z(AT, 4, dtype=torch.float64)), dict(tile_pixel_cumsum=z(AT, dtype=torch.int32)),
                  dict(pixel_map=z(P, dtype=torch.int32))]
        if "_ids" in fn and "top" not in fn:
            cases += [dict(num_contributing_gaussians=z(P, dtype=torch.int64))]
    else:
        cases += [dict(tile_offsets=z(I, 2, 3, dtype=torch.int64))]
        if "_ids" in fn and "top" not in fn:
            cases += [dict(num_contributing_gaussians=z(I, H, W, dtype=torch.float32))]
    if "top" in fn:
        cases += [dict(num_depth_samples=2.0), dict(num_depth_samples="4")]
    return cases


@pytest.mark.parametrize("fn", NAMES)
def test_value_errors_before_the_device(fn):
    for kw in _bad_values(fn):
        with pytest.raises(ValueError):
            _call(fn, **kw)


@pytest.mark.parametrize("fn", NAMES)
def test_type_errors_before_the_device(fn):
    for kw in _bad_types(fn):
        with pytest.raises(TypeError):
            _call(fn, **kw)


@pytest.mark.parametrize("fn", NAMES)
def test_valid_cpu_call_reaches_the_device_check(fn):
    """well-formed dense and packed arguments pass every check and stop at the CUDA requirement"""
    for packed in (False, True):
        with pytest.raises(_cabi.GsplatB200Error):
            _call(fn, packed=packed)


def test_depth_sample_bound_drives_the_error(monkeypatch):
    """num_depth_samples up to the device's bound runs, one more is a ValueError before any launch"""
    if torch.cuda.is_available():
        bound = ops._max_depth_samples(torch.device("cuda", 0))
        assert bound == _cabi.lib().gsb200_contrib_max_samples() and bound >= 1
    else:
        # no device to ask: the C query says so, and the bound is only checked where the tensors live on a device
        assert _cabi.lib().gsb200_contrib_max_samples() == -3
    monkeypatch.setattr(ops, "_max_depth_samples", lambda dev: 6)
    monkeypatch.setattr(ops, "require_cuda", lambda *t: torch.device("cpu"))
    launched = []
    monkeypatch.setattr(ops, "_Ctx", lambda dev: launched.append(dev))
    for fn in ("rasterize_top_contributing_gaussian_ids", "rasterize_top_contributing_gaussian_ids_sparse"):
        with pytest.raises(ValueError, match="exceeds 6"):
            _call(fn, num_depth_samples=7)
        with pytest.raises(TypeError):  # K = 6 passes the bound and reaches the launch (here a stub)
            _call(fn, num_depth_samples=6)
    assert len(launched) == 2


def test_dropin_rebinds_the_contributor_queries(tmp_path, monkeypatch):
    from gsplat_b200 import dropin

    G, Wr = _stub_package(tmp_path, monkeypatch, _BASE + list(NAMES))
    stock = {n: getattr(Wr, n) for n in NAMES}
    try:
        out = dropin.apply(losses=False)
        for n in NAMES:
            assert n in out["ops"]
            for mod in (Wr, G):
                assert getattr(mod, n).__gsb200_ours__ is getattr(gs, n)
        # an argument the b200 path declines (tile_size 8) is the package's business
        a = _args("rasterize_num_contributing_gaussians")
        got = G.rasterize_num_contributing_gaussians(a["means2d"], a["conics"], a["opacities"], a["tile_offsets"],
                                                     a["flatten_ids"], W, H, 8)
        assert got == ("stock", "rasterize_num_contributing_gaussians")
    finally:
        dropin.undo()
    for n in NAMES:
        assert getattr(Wr, n) is stock[n] and getattr(G, n) is stock[n]


def test_dropin_leaves_a_package_without_them_alone(tmp_path, monkeypatch):
    from gsplat_b200 import dropin

    G, Wr = _stub_package(tmp_path, monkeypatch, list(_BASE))
    try:
        dropin.apply(losses=False)
        for n in NAMES:
            assert not hasattr(Wr, n) and not hasattr(G, n)
    finally:
        dropin.undo()
