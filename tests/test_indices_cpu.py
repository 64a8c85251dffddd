"""rasterize_to_indices_in_range / _2dgs without a GPU: the reference's signatures, every argument error raised on CPU
tensors before anything needs the device, the exports and the drop-in's rebinding."""
import ast
import importlib
import json
import os
import sys
import textwrap

import pytest
import torch

import gsplat_b200 as gs
from gsplat_b200 import _cabi

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
NAMES = ("rasterize_to_indices_in_range", "rasterize_to_indices_in_range_2dgs")


@pytest.mark.parametrize("fn", NAMES)
def test_same_parameters_as_reference(fn):
    with open(os.path.join(ROOT, "tests", "golden", "ref_signatures_indices.json")) as f:
        ref = json.load(f)["params"][fn]
    tree = ast.parse(open(os.path.join(ROOT, "gsplat_b200", "ops.py")).read())
    node = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == fn)
    a = node.args
    assert [x.arg for x in a.posonlyargs + a.args + a.kwonlyargs] == ref["params"]
    assert len(a.defaults) == ref["n_defaults"]


def test_exported():
    for n in NAMES:
        assert n in gs.__all__ and callable(getattr(gs, n))


def _args(two_d=False, I=2, N=5, W=40, H=20):
    z = torch.zeros
    rows = z(I, N, 3, 3) if two_d else z(I, N, 3)
    return dict(range_start=0, range_end=10, transmittances=torch.ones(I, H, W), means2d=z(I, N, 2), rows=rows,
                opacities=z(I, N), image_width=W, image_height=H, tile_size=16,
                isect_offsets=z(I, 2, 3, dtype=torch.int32), flatten_ids=z(7, dtype=torch.int32))


def _call(two_d=False, **kw):
    a = _args(two_d)
    a.update(kw)
    fn = gs.rasterize_to_indices_in_range_2dgs if two_d else gs.rasterize_to_indices_in_range
    return fn(a["range_start"], a["range_end"], a["transmittances"], a["means2d"], a["rows"], a["opacities"],
              a["image_width"], a["image_height"], a["tile_size"], a["isect_offsets"], a["flatten_ids"])


def _bad_value_cases(two_d):
    z = torch.zeros
    rows_bad = z(2, 5, 3) if two_d else z(2, 5, 3, 3)
    return [
        dict(tile_size=8),
        dict(range_start=-1),
        dict(range_end=-3),
        dict(range_end=2.5),
        dict(range_end=float("inf")),
        dict(means2d=z(2, 5, 3)),
        dict(means2d=z(5)),
        dict(rows=rows_bad),
        dict(rows=z(2, 6, 3, 3) if two_d else z(2, 6, 3)),
        dict(opacities=z(2, 4)),
        dict(opacities=z(2, 5, 1)),
        dict(transmittances=torch.ones(2, 20, 41)),
        dict(transmittances=torch.ones(1, 20, 40)),
        dict(transmittances=torch.ones(2, 1, 20, 40)),
        dict(isect_offsets=z(2, 1, 3, dtype=torch.int32)),  # 3 x 1 tiles do not cover 40 x 20
        dict(isect_offsets=z(3, 2, 3, dtype=torch.int32)),
        dict(isect_offsets=z(2, 3, dtype=torch.int32)),
        dict(flatten_ids=z(7, 1, dtype=torch.int32)),
    ]


@pytest.mark.parametrize("two_d", [False, True])
def test_value_errors_before_the_device(two_d):
    for kw in _bad_value_cases(two_d):
        with pytest.raises(ValueError):
            _call(two_d, **kw)


@pytest.mark.parametrize("two_d", [False, True])
def test_type_errors_before_the_device(two_d):
    z = torch.zeros
    cases = [
        dict(transmittances=torch.ones(2, 20, 40, dtype=torch.float64)),
        dict(means2d=z(2, 5, 2, dtype=torch.float16)),
        dict(rows=z(2, 5, 3, 3, dtype=torch.float64) if two_d else z(2, 5, 3, dtype=torch.float64)),
        dict(opacities=z(2, 5, dtype=torch.float64)),
        dict(isect_offsets=z(2, 2, 3, dtype=torch.int64)),
        dict(flatten_ids=z(7, dtype=torch.int64)),
        dict(range_start="0"),
        dict(range_end=None),
    ]
    for kw in cases:
        with pytest.raises(TypeError):
            _call(two_d, **kw)


@pytest.mark.parametrize("two_d", [False, True])
def test_valid_cpu_call_reaches_the_device_check(two_d):
    """well-formed arguments pass every check and stop at the CUDA requirement; so do an empty range and 1e10"""
    for kw in (dict(), dict(range_start=3, range_end=3), dict(range_end=1e10), dict(range_end=2**70)):
        with pytest.raises(_cabi.GsplatB200Error):
            _call(two_d, **kw)


_STUB = {
    "gsplat/__init__.py": """
        from .cuda._wrapper import *  # noqa
        from .rendering import rasterization
        """,
    "gsplat/cuda/__init__.py": "",
    "gsplat/rendering.py": "def rasterization(*a, **k):\n    return ('stock', 'rasterization')\n",
    "gsplat/relocation.py": "def compute_relocation(*a, **k):\n    return ('stock', 'compute_relocation')\n",
    "gsplat/strategy/__init__.py": "",
    "gsplat/strategy/ops.py": "from ..relocation import compute_relocation\ndef _cuda_fused_mcmc_perturb(*a, **k):\n    return False\n",
    "gsplat/optimizers/__init__.py": "class SelectiveAdam:\n    pass\n",
}
_WRAPPER = """
    def _stock(name):
        def f(*a, **k):
            return ("stock", name)
        f.__name__ = name
        return f
    _NAMES = {names!r}
    for _n in _NAMES:
        globals()[_n] = _stock(_n)
    __all__ = list(_NAMES)
    """
_BASE = ["quat_scale_to_covar_preci", "fully_fused_projection", "spherical_harmonics", "isect_tiles", "isect_offset_encode",
         "rasterize_to_pixels", "adam", "build_sparse_tile_layout", "isect_tiles_sparse", "rasterize_to_pixels_sparse"]


def _stub_package(tmp_path, monkeypatch, names):
    files = dict(_STUB)
    files["gsplat/cuda/_wrapper.py"] = _WRAPPER.format(names=names)
    for rel, text in files.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    monkeypatch.syspath_prepend(str(tmp_path))
    for m in [m for m in sys.modules if m == "gsplat" or m.startswith("gsplat.")]:
        monkeypatch.delitem(sys.modules, m)
    return importlib.import_module("gsplat"), importlib.import_module("gsplat.cuda._wrapper")


def test_dropin_rebinds_the_index_ops(tmp_path, monkeypatch):
    from gsplat_b200 import dropin

    G, W = _stub_package(tmp_path, monkeypatch, _BASE + list(NAMES))
    stock = {n: getattr(W, n) for n in NAMES}
    try:
        out = dropin.apply(losses=False)
        for n in NAMES:
            assert n in out["ops"]
            for mod in (W, G):
                assert getattr(mod, n).__gsb200_ours__ is getattr(gs, n)
        # an argument the b200 path declines (tile_size 8) is the package's business
        a = _args()
        got = G.rasterize_to_indices_in_range(0, 1, a["transmittances"], a["means2d"], a["rows"], a["opacities"], 40, 20, 8,
                                              a["isect_offsets"], a["flatten_ids"])
        assert got == ("stock", "rasterize_to_indices_in_range")
    finally:
        dropin.undo()
    for n in NAMES:
        assert getattr(W, n) is stock[n] and getattr(G, n) is stock[n]


def test_dropin_leaves_a_package_without_them_alone(tmp_path, monkeypatch):
    from gsplat_b200 import dropin

    G, W = _stub_package(tmp_path, monkeypatch, list(_BASE))
    try:
        dropin.apply(losses=False)
        for n in NAMES:
            assert not hasattr(W, n) and not hasattr(G, n)
    finally:
        dropin.undo()
    for n in NAMES:
        assert not hasattr(W, n) and not hasattr(G, n)
