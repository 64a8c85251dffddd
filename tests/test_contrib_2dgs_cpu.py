"""The 2DGS per-pixel contributor queries without a GPU: the six exported names and their parameters, every argument
error raised on CPU tensors before anything needs the device, the refusal of CPU tensors, the surfel walk's own top-K
bound, and the return codes of the four C entries (gsb200_surfel_contrib_*) for invalid and early-return arguments.
Every library call here returns before a kernel is launched or the device is touched: the pointers are fake and never
read."""
import ast
import os

import pytest
import torch

import gsplat_b200 as gs
from gsplat_b200 import _cabi, ops

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
OK, INVALID, UNSUPPORTED, CUDA = 0, -1, -2, -3
FAKE = 1 << 20  # 16-byte aligned, never dereferenced

NAMES = tuple(
    f"rasterize_{n}_2dgs{s}"
    for n in ("num_contributing_gaussians", "contributing_gaussian_ids", "top_contributing_gaussian_ids")
    for s in ("", "_sparse")
)
DENSE = ["means2d", "ray_transforms", "opacities", "tile_offsets", "flatten_ids", "image_width", "image_height", "tile_size"]
SPARSE = ["means2d", "ray_transforms", "opacities", "active_tiles", "tile_offsets", "flatten_ids", "tile_pixel_mask",
          "tile_pixel_cumsum", "pixel_map"]
GRID = ["image_width", "image_height", "tile_size", "tile_width", "tile_height"]
PARAMS = {
    "rasterize_num_contributing_gaussians_2dgs": DENSE,
    "rasterize_num_contributing_gaussians_2dgs_sparse": SPARSE + GRID,
    "rasterize_contributing_gaussian_ids_2dgs": DENSE + ["num_contributing_gaussians"],
    "rasterize_contributing_gaussian_ids_2dgs_sparse": SPARSE + ["num_contributing_gaussians"] + GRID,
    "rasterize_top_contributing_gaussian_ids_2dgs": DENSE + ["num_depth_samples"],
    "rasterize_top_contributing_gaussian_ids_2dgs_sparse": SPARSE + GRID + ["num_depth_samples"],
}
I, N, W, H, AT, P = 2, 5, 40, 20, 3, 9


def _node(fn):
    tree = ast.parse(open(os.path.join(ROOT, "gsplat_b200", "ops.py")).read())
    return next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == fn)


@pytest.mark.parametrize("fn", NAMES)
def test_parameters(fn):
    """the 3DGS twin's parameters in its order, with ray_transforms in place of conics, and no defaults"""
    a = _node(fn).args
    assert [x.arg for x in a.posonlyargs + a.args + a.kwonlyargs] == PARAMS[fn]
    assert not a.defaults and not a.kw_defaults
    twin = _node(fn.replace("_2dgs", "")).args
    assert [x.arg for x in twin.args] == ["conics" if p == "ray_transforms" else p for p in PARAMS[fn]]


def test_exported():
    for n in NAMES:
        assert n in gs.__all__ and getattr(gs, n) is getattr(ops, n)


def _args(fn):
    """well-formed CPU arguments of `fn` by parameter name: two images of N surfels"""
    z = torch.zeros
    a = dict(means2d=z(I, N, 2), ray_transforms=z(I, N, 3, 3), opacities=z(I, N), flatten_ids=z(11, dtype=torch.int32),
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
    a = _args(fn)
    a.update(kw)
    return getattr(gs, fn)(*(a[p] for p in PARAMS[fn]))


def _bad_values(fn):
    z = torch.zeros
    cases = [dict(tile_size=8), dict(means2d=z(I, N, 3)), dict(means2d=z(5)), dict(ray_transforms=z(I, N + 1, 3, 3)),
             dict(ray_transforms=z(I, N, 3)), dict(ray_transforms=z(I, N, 9)), dict(ray_transforms=z(I, N, 3, 2)),
             dict(opacities=z(I, N, 1)), dict(opacities=z(I, N - 1)), dict(flatten_ids=z(11, 1, dtype=torch.int32)),
             dict(image_width=W + 100)]
    if fn.endswith("_sparse"):
        cases += [dict(tile_offsets=z(AT, dtype=torch.int32)), dict(tile_pixel_mask=z(AT, 3, dtype=torch.int64)),
                  dict(tile_pixel_cumsum=z(AT + 1, dtype=torch.int64)), dict(active_tiles=z(AT, 1, dtype=torch.int32)),
                  dict(pixel_map=z(P, 1, dtype=torch.int64)), dict(tile_height=1),
                  # pixels but no active tile: nothing could hold them
                  dict(active_tiles=z(0, dtype=torch.int32), tile_offsets=z(1, dtype=torch.int32),
                       tile_pixel_mask=z(0, 4, dtype=torch.int64), tile_pixel_cumsum=z(1, dtype=torch.int64))]
        if "_ids" in fn and "top" not in fn:
            cases += [dict(num_contributing_gaussians=z(P + 1, dtype=torch.int32))]
    else:
        cases += [dict(tile_offsets=z(I, 1, 3, dtype=torch.int32)), dict(tile_offsets=z(3, 2, 3, dtype=torch.int32)),
                  dict(tile_offsets=z(3, dtype=torch.int32)), dict(means2d=z(1, I, N, 2)),
                  # packed rows [nnz, *]: the surfel rows are dense only
                  dict(means2d=z(7, 2), ray_transforms=z(7, 3, 3), opacities=z(7))]
        if "_ids" in fn and "top" not in fn:
            cases += [dict(num_contributing_gaussians=z(I, H, W + 1, dtype=torch.int32)),
                      dict(num_contributing_gaussians=z(H, W, dtype=torch.int32))]
    if "top" in fn:
        cases += [dict(num_depth_samples=0), dict(num_depth_samples=-3)]
    return cases


def _bad_types(fn):
    z = torch.zeros
    cases = [dict(means2d=z(I, N, 2, dtype=torch.float64)), dict(ray_transforms=z(I, N, 3, 3, dtype=torch.float16)),
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


def test_messages_name_the_surfel_rows():
    z = torch.zeros
    with pytest.raises(ValueError, match=r"ray_transforms"):
        _call("rasterize_num_contributing_gaussians_2dgs", ray_transforms=z(I, N, 3))
    with pytest.raises(ValueError, match=r"means2d must be \[\.\.\., N, 2\], got"):
        _call("rasterize_num_contributing_gaussians_2dgs", means2d=z(5))
    with pytest.raises(ValueError, match="to match tile_offsets"):
        _call("rasterize_num_contributing_gaussians_2dgs", means2d=z(7, 2), ray_transforms=z(7, 3, 3), opacities=z(7))
    with pytest.raises(TypeError, match="ray_transforms: expected float32"):
        _call("rasterize_top_contributing_gaussian_ids_2dgs_sparse", ray_transforms=z(I, N, 3, 3, dtype=torch.float64))


@pytest.mark.parametrize("fn", NAMES)
def test_type_errors_before_the_device(fn):
    for kw in _bad_types(fn):
        with pytest.raises(TypeError):
            _call(fn, **kw)


@pytest.mark.parametrize("fn", NAMES)
def test_cpu_tensors_raise(fn):
    """well-formed arguments pass every check and stop at the CUDA requirement, also a single image and a batch"""
    z = torch.zeros
    for kw in (dict(), dict(means2d=z(1, I, N, 2), ray_transforms=z(1, I, N, 3, 3), opacities=z(1, I, N),
                            tile_offsets=z(1, I, 2, 3, dtype=torch.int32),
                            num_contributing_gaussians=z(1, I, H, W, dtype=torch.int32))):
        if fn.endswith("_sparse"):
            kw.pop("tile_offsets", None)
            kw.pop("num_contributing_gaussians", None)
        with pytest.raises(_cabi.GsplatB200Error, match="CUDA"):
            _call(fn, **kw)


def test_surfel_bound_drives_the_error(monkeypatch):
    """the 2DGS top-K forms check num_depth_samples against the surfel walk's bound, the 3DGS forms against theirs"""
    if torch.cuda.is_available():
        bound = ops._max_depth_samples(torch.device("cuda", 0), "gsb200_surfel_contrib_max_samples")
        assert bound == _cabi.lib().gsb200_surfel_contrib_max_samples() and bound >= 1
    else:
        assert _cabi.lib().gsb200_surfel_contrib_max_samples() == CUDA
    bounds = {"gsb200_contrib_max_samples": 100, "gsb200_surfel_contrib_max_samples": 6}
    asked = []

    def fake_bound(dev, entry="gsb200_contrib_max_samples"):
        asked.append(entry)
        return bounds[entry]

    monkeypatch.setattr(ops, "_max_depth_samples", fake_bound)
    monkeypatch.setattr(ops, "require_cuda", lambda *t: torch.device("cpu"))
    launched = []
    monkeypatch.setattr(ops, "_Ctx", lambda dev: launched.append(dev))
    for fn in ("rasterize_top_contributing_gaussian_ids_2dgs", "rasterize_top_contributing_gaussian_ids_2dgs_sparse"):
        with pytest.raises(ValueError, match="exceeds 6"):
            _call(fn, num_depth_samples=7)
        with pytest.raises(TypeError):  # K = 6 passes the bound and reaches the launch (here a stub)
            _call(fn, num_depth_samples=6)
    assert len(launched) == 2 and set(asked) == {"gsb200_surfel_contrib_max_samples"}
    from tests.test_contrib_cpu import _call as call_3dgs

    with pytest.raises(TypeError):  # 7 is within the 3DGS bound
        call_3dgs("rasterize_top_contributing_gaussian_ids", num_depth_samples=7)
    assert len(launched) == 3 and asked[-1] == "gsb200_contrib_max_samples"


# ---------------------------------------------------------------------------------------------- C ABI return codes
HEAD = ("I N means2d rows opacities W H tile_size tw th offsets flatten_ids n_isects n_active active_tiles tile_pixel_mask "
        "tile_pixel_cumsum pixel_map")
ENTRY_PARAMS = {
    "count": f"{HEAD} counts alphas stream",
    "ids": f"{HEAD} max_samples ids weights stream",
    "top": f"{HEAD} num_samples ids weights stream",
}
# a 16 x 16 image of one tile, one intersection; every other pointer fake
BASE = dict(I=1, N=4, W=16, H=16, tile_size=16, tw=1, th=1, n_isects=1, n_active=0, active_tiles=None, alphas=None,
            max_samples=2, num_samples=2, stream=None)
SPARSE_ON = dict(active_tiles=FAKE, n_active=1)

# (query, arguments changed from BASE, expected code).  None of these reaches a launch, with or without a device.
CASES = [
    ("count", dict(I=-1), INVALID),
    ("count", dict(N=-1), INVALID),
    ("count", dict(n_isects=-1), INVALID),
    ("count", dict(n_active=-1), INVALID),
    ("count", dict(tile_size=8), UNSUPPORTED),
    ("count", dict(tile_size=8, I=-1), INVALID),
    ("count", dict(I=0), OK),
    ("count", dict(I=0, counts=None, offsets=None), OK),
    ("count", dict(W=0), OK),
    ("count", dict(H=0, means2d=None), OK),
    ("count", dict(active_tiles=FAKE, n_active=0, I=5), OK),
    ("count", dict(offsets=None), INVALID),
    ("count", dict(means2d=None), INVALID),
    ("count", dict(rows=None), INVALID),
    ("count", dict(opacities=None), INVALID),
    ("count", dict(flatten_ids=None), INVALID),
    ("count", dict(counts=None), INVALID),
    ("count", dict(W=17), INVALID),
    ("count", dict(SPARSE_ON, tile_pixel_mask=None), INVALID),
    ("count", dict(SPARSE_ON, tile_pixel_cumsum=None), INVALID),
    ("count", dict(SPARSE_ON, pixel_map=None), INVALID),
    ("count", dict(SPARSE_ON, W=17), INVALID),
    ("count", dict(tw=1 << 16, th=1 << 15), UNSUPPORTED),
    ("count", dict(n_isects=1 << 31), UNSUPPORTED),
    ("count", dict(SPARSE_ON, n_active=1 << 31), UNSUPPORTED),
    ("count", dict(n_isects=1 << 31, flatten_ids=None), INVALID),
    ("ids", dict(max_samples=-1), INVALID),
    ("ids", dict(N=1 << 31), INVALID),
    ("ids", dict(max_samples=0, ids=None, weights=None), OK),
    ("ids", dict(max_samples=0, I=-1), OK),
    ("ids", dict(I=-1), INVALID),
    ("ids", dict(tile_size=8), UNSUPPORTED),
    ("ids", dict(I=0), OK),
    ("ids", dict(ids=None), INVALID),
    ("ids", dict(weights=None), INVALID),
    ("ids", dict(SPARSE_ON, pixel_map=None), INVALID),
    ("ids", dict(n_isects=1 << 31), UNSUPPORTED),
    ("top", dict(num_samples=0), INVALID),
    ("top", dict(num_samples=-1), INVALID),
    ("top", dict(num_samples=0, tile_size=8), INVALID),
    ("top", dict(N=1 << 31), INVALID),
]


@pytest.mark.parametrize("walk", ["gsb200_surfel_contrib", "gsb200_contrib"])
@pytest.mark.parametrize("query", sorted(ENTRY_PARAMS))
def test_return_codes_before_launch(walk, query):
    """the surfel entries, and the 3DGS entries whose checks they share, in the same order with the same codes"""
    entry = f"{walk}_{query}"
    L = _cabi.lib()
    assert len(ENTRY_PARAMS[query].split()) == len(_cabi._SIGNATURES[entry][1])
    assert _cabi._SIGNATURES[entry] == _cabi._SIGNATURES[f"gsb200_contrib_{query}"]

    def call(changes):
        args = dict(BASE, **changes)
        return getattr(L, entry)(*[args.get(p, FAKE) for p in ENTRY_PARAMS[query].split()])

    got = [(changes, call(changes)) for q, changes, _ in CASES if q == query]
    want = [(changes, code) for q, changes, code in CASES if q == query]
    assert got == want


def test_max_samples_entry():
    """the surfel walk's bound: >= 1 with a device, GSB200_E_CUDA without one"""
    L = _cabi.lib()
    assert "gsb200_surfel_contrib_max_samples" in _cabi.EXPORTED_SYMBOLS
    rc = L.gsb200_surfel_contrib_max_samples()
    assert rc >= 1 if torch.cuda.is_available() else rc == CUDA
