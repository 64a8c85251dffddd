"""Sparse-pixel ops without a GPU: the public signatures against the reference's, the argument checks that run on the
host before anything is launched, and the drop-in rebinding of the three names on a stub ``gsplat`` package."""
import ast
import importlib
import json
import os
import sys
import textwrap

import pytest
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
NAMES = ("build_sparse_tile_layout", "isect_tiles_sparse", "rasterize_to_pixels_sparse")


@pytest.mark.parametrize("fn", NAMES)
def test_same_parameters_as_reference(fn):
    """tests/golden/ref_signatures_sparse.json holds the reference's parameter names and number of defaulted parameters
    of the three functions (gsplat/cuda/_wrapper.py), parsed from its sources with `ast` like ref_signatures.json."""
    with open(os.path.join(ROOT, "tests", "golden", "ref_signatures_sparse.json")) as f:
        ref = json.load(f)["params"][fn]
    tree = ast.parse(open(os.path.join(ROOT, "gsplat_b200", "ops.py")).read())
    node = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == fn)
    a = node.args
    assert [x.arg for x in a.posonlyargs + a.args + a.kwonlyargs] == ref["params"]
    assert len(a.defaults) == ref["n_defaults"]


def _layout(pixels, image_ids, n_images=1, tile_size=16, tw=20, th=13):
    import gsplat_b200

    return gsplat_b200.build_sparse_tile_layout(
        torch.tensor(pixels, dtype=torch.int32).reshape(-1, 2), torch.tensor(image_ids, dtype=torch.int32), n_images, tile_size, tw, th
    )


@pytest.mark.parametrize(
    "pixels,image_ids,n_images,match",
    [
        ([[0, 0], [208, 5]], [0, 0], 1, "tile grid"),  # row past the 13 tile rows
        ([[0, 320]], [0], 1, "tile grid"),  # col past the 20 tile columns
        ([[-1, 3]], [0], 1, "tile grid"),
        ([[0, 0], [1, 1]], [0, 2], 2, "image id"),
        ([[0, 0]], [-1], 1, "image id"),
    ],
)
def test_layout_rejects_out_of_range_before_launch(pixels, image_ids, n_images, match):
    """CPU tensors never reach the library: the ValueError comes from the host-side checks."""
    with pytest.raises(ValueError, match=match):
        _layout(pixels, image_ids, n_images)


def test_layout_rejects_other_tile_sizes():
    with pytest.raises(ValueError, match="tile_size"):
        _layout([[0, 0]], [0], 1, tile_size=8, tw=40, th=26)


def test_layout_shape_checks():
    import gsplat_b200

    with pytest.raises(ValueError, match="pixels"):
        gsplat_b200.build_sparse_tile_layout(torch.zeros(3, dtype=torch.int32), torch.zeros(3, dtype=torch.int32), 1, 16, 4, 4)
    with pytest.raises(ValueError, match="image_ids"):
        gsplat_b200.build_sparse_tile_layout(torch.zeros(3, 2, dtype=torch.int32), torch.zeros(2, dtype=torch.int32), 1, 16, 4, 4)


def test_rasterize_sparse_argument_checks():
    import gsplat_b200

    z = torch.zeros
    m2, con, op = z(1, 5, 2), z(1, 5, 3), z(1, 5)
    ids, pmap = z(4, dtype=torch.int32), z(4, dtype=torch.int64)
    active, toff, fl = z(2, dtype=torch.int32), z(3, dtype=torch.int32), z(0, dtype=torch.int32)
    words, cum = z(2, 4, dtype=torch.int64), z(2, dtype=torch.int64)

    def call(colors, tile_size=16, packed=False, tile_offsets=toff):
        return gsplat_b200.rasterize_to_pixels_sparse(
            m2, con, colors, op, ids, active, tile_offsets, fl, words, cum, pmap, 64, 48, tile_size, 4, 3, packed=packed
        )

    with pytest.raises(ValueError, match="channels"):
        call(z(1, 5, 33))
    with pytest.raises(ValueError, match="tile_size"):
        call(z(1, 5, 3), tile_size=8)
    with pytest.raises(ValueError, match="packed"):
        call(z(1, 5, 3), packed=True)
    with pytest.raises(ValueError, match="tile_offsets"):
        call(z(1, 5, 3), tile_offsets=z(2, dtype=torch.int32))


def test_isect_sparse_argument_checks():
    import gsplat_b200

    z = torch.zeros
    mask, active = z(2, 3, 4, dtype=torch.bool), z(0, dtype=torch.int32)
    with pytest.raises(ValueError, match="image_ids"):
        gsplat_b200.isect_tiles_sparse(z(5, 2), z(5, 2, dtype=torch.int32), z(5), mask, active, 2, 16, 4, 3)
    with pytest.raises(ValueError, match="n_images"):
        gsplat_b200.isect_tiles_sparse(z(1, 5, 2), z(1, 5, 2, dtype=torch.int32), z(1, 5), mask, active, 2, 16, 4, 3)
    with pytest.raises(ValueError, match="tile_mask"):
        gsplat_b200.isect_tiles_sparse(z(2, 5, 2), z(2, 5, 2, dtype=torch.int32), z(2, 5), mask[..., :3], active, 2, 16, 4, 3)


_STUB = {
    "gsplat/__init__.py": """
        from .cuda._wrapper import *  # noqa
        from .rendering import rasterization
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
                  "rasterize_to_pixels_sparse"]
        for _n in _NAMES:
            globals()[_n] = _stock(_n)
        __all__ = list(_NAMES)
        """,
    "gsplat/rendering.py": "def rasterization(*a, **k):\n    return ('stock', 'rasterization')\n",
    "gsplat/relocation.py": "def compute_relocation(*a, **k):\n    return ('stock', 'compute_relocation')\n",
    "gsplat/strategy/__init__.py": "",
    "gsplat/strategy/ops.py": "from ..relocation import compute_relocation\ndef _cuda_fused_mcmc_perturb(*a, **k):\n    return False\n",
    "gsplat/optimizers/__init__.py": "class SelectiveAdam:\n    pass\n",
}


def test_dropin_rebinds_sparse_names(tmp_path, monkeypatch):
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
    stock = {n: getattr(W, n) for n in NAMES}
    try:
        dropin.apply(losses=False)
        for n in NAMES:
            for mod in (W, G):
                fn = getattr(mod, n)
                assert fn is not stock[n] and fn.__gsb200_ours__ is getattr(gsplat_b200, n)
        # an argument the b200 path declines (tile_size 8) is handed to the package's own implementation
        out = W.build_sparse_tile_layout(torch.zeros(1, 2, dtype=torch.int32), torch.zeros(1, dtype=torch.int32), 1, 8, 4, 4)
        assert out == ("stock", "build_sparse_tile_layout")
    finally:
        dropin.undo()
    for n in NAMES:
        assert getattr(W, n) is stock[n] and getattr(G, n) is stock[n]
