"""rasterize_to_pixels_2dgs_sparse without a GPU: its public surface, the argument checks that run on the host before
anything is launched, the refusal of CPU tensors, and the return codes of its two C entries
(gsb200_surfel_raster_sparse_fwd / _bwd) for invalid or early-return arguments, including which check fires first.
Every library call here returns before a kernel is launched or the device is touched: the pointers are fake and never
read."""
import ast
import os

import pytest
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
OK, INVALID, UNSUPPORTED = 0, -1, -2
FAKE = 1 << 20  # 16-byte aligned, never dereferenced


def test_exported():
    import gsplat_b200

    assert "rasterize_to_pixels_2dgs_sparse" in gsplat_b200.__all__
    assert gsplat_b200.rasterize_to_pixels_2dgs_sparse is gsplat_b200.ops.rasterize_to_pixels_2dgs_sparse


def test_parameters():
    """The arguments of rasterize_to_pixels_sparse, with the 2DGS rows where rasterize_to_pixels_2dgs has them."""
    tree = ast.parse(open(os.path.join(ROOT, "gsplat_b200", "ops.py")).read())
    node = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == "rasterize_to_pixels_2dgs_sparse")
    assert [a.arg for a in node.args.args] == [
        "means2d", "ray_transforms", "colors", "opacities", "normals", "densify", "image_ids", "active_tiles", "tile_offsets",
        "flatten_ids", "tile_pixel_mask", "tile_pixel_cumsum", "pixel_map", "image_width", "image_height", "tile_size",
        "tile_width", "tile_height", "backgrounds", "masks", "absgrad", "distloss",
    ]
    assert [ast.literal_eval(d) for d in node.args.defaults] == [None, None, False, False]


# two images of N = 5 surfels, D = 3; a 64 x 48 image on a 4 x 3 tile grid; P = 4 pixels in AT = 2 active tiles
def _args(**changes):
    z = torch.zeros
    a = dict(
        means2d=z(2, 5, 2), ray_transforms=z(2, 5, 3, 3), colors=z(2, 5, 3), opacities=z(2, 5), normals=z(2, 5, 3),
        densify=z(2, 5, 2), image_ids=z(4, dtype=torch.int32), active_tiles=z(2, dtype=torch.int32),
        tile_offsets=z(3, dtype=torch.int32), flatten_ids=z(6, dtype=torch.int32), tile_pixel_mask=z(2, 4, dtype=torch.int64),
        tile_pixel_cumsum=z(2, dtype=torch.int64), pixel_map=z(4, dtype=torch.int64), image_width=64, image_height=48,
        tile_size=16, tile_width=4, tile_height=3,
    )
    a.update(changes)
    return a


def _call(**changes):
    import gsplat_b200

    return gsplat_b200.rasterize_to_pixels_2dgs_sparse(**_args(**changes))


z = torch.zeros
ARG_ERRORS = [
    (dict(tile_size=8), ValueError, "tile_size"),
    (dict(active_tiles=z(2, dtype=torch.int64)), ValueError, "active_tiles"),
    (dict(pixel_map=z(2, 2, dtype=torch.int64)), ValueError, "active_tiles"),
    (dict(tile_offsets=z(2, dtype=torch.int32)), ValueError, "tile_offsets"),
    (dict(flatten_ids=z(6, dtype=torch.int64)), ValueError, "tile_offsets"),
    (dict(flatten_ids=z(3, 2, dtype=torch.int32)), ValueError, "flatten_ids"),
    (dict(tile_pixel_mask=z(2, 3, dtype=torch.int64)), ValueError, "tile_pixel_mask"),
    (dict(tile_pixel_mask=z(2, 4, dtype=torch.int32)), ValueError, "tile_pixel_mask"),
    (dict(tile_pixel_cumsum=z(3, dtype=torch.int64)), ValueError, "tile_pixel_cumsum"),
    (dict(pixel_map=z(4, dtype=torch.int32)), ValueError, "tile_pixel_cumsum"),
    (dict(image_ids=z(3, dtype=torch.int32)), ValueError, "image_ids"),
    (dict(image_width=65), ValueError, "does not cover"),
    (dict(image_height=49), ValueError, "does not cover"),
    (dict(means2d=z(10, 2)), ValueError, "colors"),  # packed rows [nnz, 2]: 2DGS has dense rows only
    (dict(means2d=z(2, 5, 3)), ValueError, "means2d"),
    (dict(ray_transforms=z(2, 5, 9)), ValueError, "ray_transforms"),
    (dict(colors=z(5, 3)), ValueError, "colors"),
    (dict(colors=z(2, 4, 3)), ValueError, "colors"),
    (dict(opacities=z(2, 5, 1)), ValueError, "opacities"),
    (dict(normals=z(2, 5, 2)), ValueError, "normals"),
    (dict(densify=z(2, 5)), ValueError, "densify"),
    (dict(backgrounds=z(1, 3)), ValueError, "backgrounds"),
    (dict(backgrounds=z(2, 4)), ValueError, "backgrounds"),
    (dict(masks=z(2, 4, 3, dtype=torch.bool)), ValueError, "masks"),
    (dict(colors=z(2, 5, 6)), NotImplementedError, "channels"),
    (dict(colors=z(2, 5, 33)), NotImplementedError, "channels"),
]


@pytest.mark.parametrize("changes,exc,match", ARG_ERRORS, ids=[f"{i}-{m}" for i, (_, _, m) in enumerate(ARG_ERRORS)])
def test_argument_errors_before_launch(changes, exc, match):
    """CPU tensors never reach the library: each error comes from the host-side checks."""
    with pytest.raises(exc, match=match):
        _call(**changes)


@pytest.mark.parametrize(
    "changes",
    [
        dict(),
        dict(backgrounds=z(2, 3), masks=z(2, 3, 4, dtype=torch.bool), absgrad=True, distloss=True),
        dict(means2d=z(1, 2, 5, 2), ray_transforms=z(1, 2, 5, 3, 3), colors=z(1, 2, 5, 3), opacities=z(1, 2, 5),
             normals=z(1, 2, 5, 3), densify=z(1, 2, 5, 2)),  # a batch dimension: n_images = 1 * 2
        # the empty cases are refused as well: they launch nothing, but still only run on CUDA tensors
        dict(flatten_ids=z(0, dtype=torch.int32)),
        dict(image_ids=z(0, dtype=torch.int32), pixel_map=z(0, dtype=torch.int64), active_tiles=z(0, dtype=torch.int32),
             tile_offsets=z(1, dtype=torch.int32), tile_pixel_mask=z(0, 4, dtype=torch.int64),
             tile_pixel_cumsum=z(1, dtype=torch.int64), flatten_ids=z(0, dtype=torch.int32)),
    ],
    ids=["plain", "options", "batch", "no-lists", "no-pixels"],
)
def test_cpu_tensors_raise(changes):
    from gsplat_b200._cabi import GsplatB200Error

    with pytest.raises(GsplatB200Error, match="CUDA"):
        _call(**changes)


# ---------------------------------------------------------------------------------------------- C ABI return codes
LAYOUT = "W H tile_size tw th n_active active_tiles tile_offsets flatten_ids n_isects tile_pixel_mask tile_pixel_cumsum pixel_map"
PARAMS = {
    "gsb200_surfel_raster_sparse_fwd": f"n_rows D means2d ray_transforms colors opacities normals backgrounds masks {LAYOUT} "
    "render_colors render_alphas render_normals render_distort render_median last_ids median_ids stream",
    "gsb200_surfel_raster_sparse_bwd": f"n_rows D means2d ray_transforms colors opacities normals backgrounds masks {LAYOUT} "
    "render_colors render_alphas last_ids median_ids v_render_colors v_render_alphas v_render_normals v_render_distort "
    "v_render_median v_means2d v_ray_transforms v_colors v_opacities v_normals v_densify v_means2d_abs stream",
}
# a 16 x 16 image of one active tile, one intersection, D = 3; every other pointer fake and 16-byte aligned
BASE = dict(n_rows=4, D=3, W=16, H=16, tile_size=16, tw=1, th=1, n_active=1, n_isects=1, backgrounds=None, masks=None,
            v_render_alphas=None, v_render_normals=None, v_render_distort=None, v_render_median=None, v_means2d_abs=None,
            stream=None)
GRID_SMALL = dict(W=17)  # one 16-pixel tile column for a 17-pixel wide image
ROWS_MAX = dict(n_rows=(1 << 31) // 9 + 1)  # n_rows * 9 >= 2^31

# (entry, arguments changed from BASE, expected code).  None of these reaches a launch.
CASES = [
    ("gsb200_surfel_raster_sparse_fwd", dict(tile_size=8), UNSUPPORTED),
    ("gsb200_surfel_raster_sparse_fwd", dict(tile_size=8, n_rows=-1), UNSUPPORTED),
    ("gsb200_surfel_raster_sparse_fwd", dict(n_rows=-1), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(n_isects=-1), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(n_active=-1), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(n_active=1 << 31), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(active_tiles=None), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(tile_offsets=None), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(tile_pixel_mask=None), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(tile_pixel_cumsum=None), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(pixel_map=None), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(GRID_SMALL), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(GRID_SMALL, n_active=0), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(n_active=0), OK),
    ("gsb200_surfel_raster_sparse_fwd", dict(n_active=0, D=6, active_tiles=None, render_colors=None), OK),
    ("gsb200_surfel_raster_sparse_fwd", dict(n_active=0, **ROWS_MAX), OK),
    ("gsb200_surfel_raster_sparse_fwd", dict(render_colors=None), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(render_normals=None, D=6), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(median_ids=None), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(means2d=None), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(normals=None), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(flatten_ids=None, **ROWS_MAX), INVALID),
    ("gsb200_surfel_raster_sparse_fwd", dict(ROWS_MAX), UNSUPPORTED),
    ("gsb200_surfel_raster_sparse_fwd", dict(n_isects=0, means2d=None, flatten_ids=None, D=6), UNSUPPORTED),
    ("gsb200_surfel_raster_sparse_fwd", dict(D=6), UNSUPPORTED),
    ("gsb200_surfel_raster_sparse_fwd", dict(D=0), UNSUPPORTED),

    ("gsb200_surfel_raster_sparse_bwd", dict(tile_size=8), UNSUPPORTED),
    ("gsb200_surfel_raster_sparse_bwd", dict(tile_size=8, n_isects=0), UNSUPPORTED),
    ("gsb200_surfel_raster_sparse_bwd", dict(n_rows=-1), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(n_isects=-1), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(n_active=-1), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(pixel_map=None), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(pixel_map=None, n_isects=0), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(GRID_SMALL), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(GRID_SMALL, n_isects=0), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(n_isects=0), OK),
    ("gsb200_surfel_raster_sparse_bwd", dict(n_active=0, D=6), OK),
    ("gsb200_surfel_raster_sparse_bwd", dict(n_isects=0, v_densify=None, **ROWS_MAX), OK),
    ("gsb200_surfel_raster_sparse_bwd", dict(render_alphas=None), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(median_ids=None), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(v_render_colors=None), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(v_densify=None), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(v_densify=None, D=6), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(ray_transforms=None, **ROWS_MAX), INVALID),
    ("gsb200_surfel_raster_sparse_bwd", dict(ROWS_MAX), UNSUPPORTED),
    ("gsb200_surfel_raster_sparse_bwd", dict(D=6), UNSUPPORTED),
    ("gsb200_surfel_raster_sparse_bwd", dict(D=0), UNSUPPORTED),
]


@pytest.mark.parametrize("entry", sorted(PARAMS))
def test_return_codes_before_launch(entry):
    from gsplat_b200 import _cabi

    L = _cabi.lib()
    assert len(PARAMS[entry].split()) == len(_cabi._SIGNATURES[entry][1])

    def call(changes):
        args = dict(BASE, **changes)
        return getattr(L, entry)(*[args.get(p, FAKE) for p in PARAMS[entry].split()])

    got = [(changes, call(changes)) for e, changes, _ in CASES if e == entry]
    want = [(changes, code) for e, changes, code in CASES if e == entry]
    assert got == want
