"""rasterize_to_pixels_eval3d_sparse without a GPU: its public surface, the argument checks that run on the host before
anything is launched (the sparse layout, the 3DGUT geometry, colours and camera), the refusal of CPU tensors, and the
return codes of its two C entries (gsb200_eval3d_sparse_fwd / _bwd) for invalid or early-return arguments, including
which check fires first.  Every library call here returns before a kernel is launched or the device is touched: the
pointers are fake and never read."""
import ctypes
import inspect

import pytest
import torch

OK, INVALID, UNSUPPORTED = 0, -1, -2
FAKE = 1 << 20  # 16-byte aligned, never dereferenced


def test_exported():
    import gsplat_b200

    assert "rasterize_to_pixels_eval3d_sparse" in gsplat_b200.__all__
    assert gsplat_b200.rasterize_to_pixels_eval3d_sparse is gsplat_b200.ops.rasterize_to_pixels_eval3d_sparse


def test_parameters():
    """The geometry and camera of rasterize_to_pixels_eval3d, the layout of the other sparse ops."""
    import gsplat_b200

    sig = inspect.signature(gsplat_b200.rasterize_to_pixels_eval3d_sparse)
    assert list(sig.parameters) == [
        "means", "quats", "scales", "colors", "opacities", "viewmats", "Ks", "image_ids", "active_tiles", "tile_offsets",
        "flatten_ids", "tile_pixel_mask", "tile_pixel_cumsum", "pixel_map", "image_width", "image_height", "tile_size",
        "tile_width", "tile_height", "backgrounds", "masks", "camera_model", "ut_params", "radial_coeffs",
        "tangential_coeffs", "thin_prism_coeffs", "ftheta_coeffs", "rolling_shutter", "viewmats_rs",
    ]
    defaults = {k: p.default for k, p in sig.parameters.items() if p.default is not inspect.Parameter.empty}
    assert defaults == dict(backgrounds=None, masks=None, camera_model="pinhole", ut_params=None, radial_coeffs=None,
                            tangential_coeffs=None, thin_prism_coeffs=None, ftheta_coeffs=None,
                            rolling_shutter=gsplat_b200.RollingShutterType.GLOBAL, viewmats_rs=None)


z = torch.zeros


# two cameras of N = 5 gaussians, D = 3; a 64 x 48 image on a 4 x 3 tile grid; P = 4 pixels in AT = 2 active tiles
def _args(**changes):
    a = dict(
        means=z(5, 3), quats=z(5, 4), scales=z(5, 3), colors=z(2, 5, 3), opacities=z(2, 5), viewmats=z(2, 4, 4),
        Ks=z(2, 3, 3), image_ids=z(4, dtype=torch.int32), active_tiles=z(2, dtype=torch.int32),
        tile_offsets=z(3, dtype=torch.int32), flatten_ids=z(6, dtype=torch.int32), tile_pixel_mask=z(2, 4, dtype=torch.int64),
        tile_pixel_cumsum=z(2, dtype=torch.int64), pixel_map=z(4, dtype=torch.int64), image_width=64, image_height=48,
        tile_size=16, tile_width=4, tile_height=3,
    )
    a.update(changes)
    return a


def _call(**changes):
    import gsplat_b200

    return gsplat_b200.rasterize_to_pixels_eval3d_sparse(**_args(**changes))


def _ftheta(**changes):
    import gsplat_b200

    p = dict(reference_poly=0, pixeldist_to_angle_poly=[0.0, 0.01, 0.0, 0.0, 0.0, 0.0],
             angle_to_pixeldist_poly=[0.0, 100.0, 0.0, 0.0, 0.0, 0.0], max_angle=1.0, linear_cde=[1.0, 0.0, 0.0])
    p.update(changes)
    return gsplat_b200.FThetaCameraDistortionParameters(**p)


class _Ut:
    alpha, kappa = 0.0, 0.0


RS = 0  # RollingShutterType.ROLLING_TOP_TO_BOTTOM
ARG_ERRORS = [
    # the layout
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
    # the geometry
    (dict(means=z(5, 2)), ValueError, "means"),
    (dict(quats=z(5, 3)), ValueError, "quats"),
    (dict(scales=z(4, 3)), ValueError, "scales"),
    (dict(viewmats=z(2, 4, 3)), ValueError, "viewmats"),
    (dict(viewmats=z(1, 2, 4, 4)), ValueError, "viewmats"),
    (dict(Ks=z(2, 3, 4)), ValueError, "Ks"),
    (dict(means=z(5, 3, dtype=torch.float64)), TypeError, "means"),
    (dict(viewmats=z(2, 4, 4, dtype=torch.float64)), TypeError, "viewmats"),
    # colours, opacities, backgrounds, masks
    (dict(colors=z(2, 5)), ValueError, "colors"),
    (dict(colors=z(2, 4, 3)), ValueError, "colors"),
    (dict(colors=z(1, 5, 3)), ValueError, "colors"),
    (dict(opacities=z(2, 4)), ValueError, "opacities"),
    (dict(colors=z(2, 5, 3, dtype=torch.float64)), TypeError, "colors"),
    (dict(opacities=z(2, 5, dtype=torch.float64)), TypeError, "opacities"),
    (dict(backgrounds=z(1, 3)), ValueError, "backgrounds"),
    (dict(backgrounds=z(2, 4)), ValueError, "backgrounds"),
    (dict(backgrounds=z(2, 3, dtype=torch.float64)), TypeError, "backgrounds"),
    (dict(masks=z(2, 4, 3, dtype=torch.bool)), ValueError, "masks"),
    (dict(masks=z(1, 3, 4, dtype=torch.bool)), ValueError, "masks"),
    (dict(colors=z(2, 5, 6)), NotImplementedError, "channels"),
    (dict(colors=z(2, 5, 33)), NotImplementedError, "channels"),
    # the camera and the shutter (_ut_camera)
    (dict(camera_model="ortho"), NotImplementedError, "camera_model"),
    (dict(camera_model="lidar"), NotImplementedError, "camera_model"),
    (dict(camera_model="nope"), ValueError, "camera_model"),
    (dict(camera_model="ftheta"), NotImplementedError, "ftheta_coeffs"),
    (dict(ftheta_coeffs=_ftheta()), NotImplementedError, "ftheta_coeffs"),
    (dict(camera_model="ftheta", ftheta_coeffs=_ftheta(reference_poly=2)), ValueError, "reference_poly"),
    (dict(camera_model="ftheta", ftheta_coeffs=_ftheta(max_angle=float("nan"))), ValueError, "max_angle"),
    (dict(camera_model="ftheta", ftheta_coeffs=_ftheta(), radial_coeffs=z(2, 6)), ValueError, "radial_coeffs"),
    (dict(radial_coeffs=z(2, 5)), ValueError, "radial_coeffs"),
    (dict(camera_model="fisheye", radial_coeffs=z(2, 6)), ValueError, "radial_coeffs"),
    (dict(tangential_coeffs=z(1, 2)), ValueError, "tangential_coeffs"),
    (dict(thin_prism_coeffs=z(2, 3)), ValueError, "thin_prism_coeffs"),
    (dict(camera_model="fisheye", tangential_coeffs=z(2, 2)), ValueError, "tangential_coeffs"),
    (dict(camera_model="fisheye", thin_prism_coeffs=z(2, 4)), ValueError, "thin_prism_coeffs"),
    (dict(rolling_shutter=RS), NotImplementedError, "viewmats_rs"),
    (dict(viewmats_rs=z(2, 4, 4)), NotImplementedError, "viewmats_rs"),
    (dict(rolling_shutter=RS, viewmats_rs=z(1, 4, 4)), ValueError, "viewmats_rs"),
    (dict(rolling_shutter=RS, viewmats_rs=z(2, 4, 4, dtype=torch.float64)), TypeError, "viewmats_rs"),
    (dict(rolling_shutter=7), ValueError, "rolling_shutter"),
    (dict(rolling_shutter=RS, viewmats_rs=z(2, 4, 4), image_height=1, tile_height=1), ValueError, "rows"),
    (dict(ut_params=_Ut()), ValueError, "ut_params"),
]


@pytest.mark.parametrize("changes,exc,match", ARG_ERRORS, ids=[f"{i}-{m}" for i, (_, _, m) in enumerate(ARG_ERRORS)])
def test_argument_errors_before_launch(changes, exc, match):
    """CPU tensors never reach the library: each error comes from the host-side checks."""
    with pytest.raises(exc, match=match):
        _call(**changes)


VALID = {
    "plain": dict(),
    "options": dict(backgrounds=z(2, 3), masks=z(2, 3, 4, dtype=torch.bool)),
    # a batch dimension: n_images = 1 * 2
    "batch": dict(means=z(1, 5, 3), quats=z(1, 5, 4), scales=z(1, 5, 3), colors=z(1, 2, 5, 3), opacities=z(1, 2, 5),
                  viewmats=z(1, 2, 4, 4), Ks=z(1, 2, 3, 3)),
    "distorted": dict(radial_coeffs=z(2, 6), tangential_coeffs=z(2, 2), thin_prism_coeffs=z(2, 4)),
    "fisheye": dict(camera_model="fisheye", radial_coeffs=z(2, 4)),
    "ftheta": dict(camera_model="ftheta", ftheta_coeffs=_ftheta()),
    "rolling": dict(rolling_shutter=RS, viewmats_rs=z(2, 4, 4)),
    "channels": dict(colors=z(2, 5, 32), backgrounds=z(2, 32)),
    # the empty cases are refused as well: they launch nothing, but still only run on CUDA tensors
    "no-lists": dict(flatten_ids=z(0, dtype=torch.int32)),
    "no-pixels": dict(image_ids=z(0, dtype=torch.int32), pixel_map=z(0, dtype=torch.int64),
                      active_tiles=z(0, dtype=torch.int32), tile_offsets=z(1, dtype=torch.int32),
                      tile_pixel_mask=z(0, 4, dtype=torch.int64), tile_pixel_cumsum=z(1, dtype=torch.int64),
                      flatten_ids=z(0, dtype=torch.int32)),
}


@pytest.mark.parametrize("case", list(VALID))
def test_cpu_tensors_raise(case):
    from gsplat_b200._cabi import GsplatB200Error

    with pytest.raises(GsplatB200Error, match="CUDA"):
        _call(**VALID[case])


# ---------------------------------------------------------------------------------------------- C ABI return codes
CAMERA = "camera_model radial tangential thin ftheta viewmats_rs rolling_shutter"
LAYOUT = "W H tile_size tw th n_active active_tiles tile_offsets flatten_ids n_isects tile_pixel_mask tile_pixel_cumsum pixel_map"
GEOM = "B C N D means quats scales colors opacities backgrounds masks viewmats Ks"
PARAMS = {
    "gsb200_eval3d_sparse_fwd": f"{GEOM} {CAMERA} {LAYOUT} render_colors render_alphas last_ids stream",
    "gsb200_eval3d_sparse_bwd": f"{GEOM} {CAMERA} {LAYOUT} render_alphas last_ids v_render_colors v_render_alphas "
    "grad_records v_colors v_opacities v_means v_quats v_scales stream",
}
# one 16 x 16 image, N = 4, one active tile, one intersection, D = 3, the perfect pinhole under the global shutter; every
# other pointer fake and 16-byte aligned
BASE = dict(B=1, C=1, N=4, D=3, W=16, H=16, tile_size=16, tw=1, th=1, n_active=1, n_isects=1, camera_model=0,
            rolling_shutter=4, backgrounds=None, masks=None, radial=None, tangential=None, thin=None, ftheta=None,
            viewmats_rs=None, v_render_alphas=None, stream=None)
GRID_SMALL = dict(W=17)  # one 16-pixel tile column for a 17-pixel wide image
ROLLING = dict(rolling_shutter=0, viewmats_rs=FAKE)
FTHETA = "ftheta"  # replaced by the address of a valid gsb200_ftheta_params


def _cases(entry):
    fwd = entry.endswith("_fwd")
    common = [
        (dict(tile_size=8), UNSUPPORTED),
        (dict(tile_size=8, rolling_shutter=5), UNSUPPORTED),  # the size checks come first
        (dict(tile_size=8, n_active=-1), UNSUPPORTED),
        (dict(n_isects=-1), INVALID),
        (dict(n_isects=-1, camera_model=1), INVALID),
        (dict(B=-1), INVALID),
        (dict(N=-1), INVALID),
        (dict(GRID_SMALL), INVALID),
        (dict(B=1 << 16, C=1 << 15, n_active=0), UNSUPPORTED),  # B * C * tw * th >= 2^31
        (dict(camera_model=1), UNSUPPORTED),
        (dict(camera_model=1, n_active=-1), UNSUPPORTED),  # the camera comes before the layout
        (dict(camera_model=3), INVALID),
        (dict(ftheta=FTHETA), INVALID),
        (dict(camera_model=3, ftheta=FTHETA, radial=FAKE), INVALID),
        (dict(rolling_shutter=0), INVALID),
        (dict(rolling_shutter=5), INVALID),
        (dict(viewmats_rs=FAKE), INVALID),
        (dict(ROLLING, H=1), INVALID),
        (dict(rolling_shutter=1, viewmats_rs=FAKE, W=1), INVALID),
        (dict(n_active=-1), INVALID),
        (dict(n_active=1 << 31), INVALID),
        (dict(active_tiles=None), INVALID),
        (dict(tile_offsets=None), INVALID),
        (dict(tile_pixel_mask=None), INVALID),
        (dict(tile_pixel_cumsum=None), INVALID),
        (dict(pixel_map=None), INVALID),
        (dict(pixel_map=None, n_isects=0), INVALID),
        (dict(C=0), INVALID),  # active tiles of no image
        (dict(D=6), UNSUPPORTED),
        (dict(D=0), UNSUPPORTED),
        (dict(D=6, camera_model=3, ftheta=FTHETA), UNSUPPORTED),
        (dict(D=6, **ROLLING), UNSUPPORTED),
        (dict(means=None), INVALID),
        (dict(colors=None), INVALID),
        (dict(viewmats=None), INVALID),
        (dict(Ks=None), INVALID),
        (dict(flatten_ids=None), INVALID),
    ]
    if fwd:
        return common + [
            (dict(n_active=0), OK),
            (dict(n_active=0, D=6, active_tiles=None, render_colors=None), OK),
            (dict(n_active=0, C=0), OK),
            (dict(render_colors=None), INVALID),
            (dict(render_alphas=None), INVALID),
            (dict(last_ids=None), INVALID),
        ]
    return common + [
        (dict(N=0), OK),  # no gaussian has a gradient
        (dict(B=0, C=0), OK),
        (dict(grad_records=None), INVALID),
        (dict(v_means=None), INVALID),
        (dict(v_scales=None), INVALID),
        (dict(quats=None, n_isects=0), INVALID),
        (dict(D=6, n_isects=0), UNSUPPORTED),  # refused before the finish kernel too
        (dict(D=6, n_active=0), UNSUPPORTED),
        (dict(render_alphas=None), INVALID),
        (dict(last_ids=None), INVALID),
        (dict(v_render_colors=None), INVALID),
        (dict(v_colors=None), INVALID),
        (dict(v_opacities=None), INVALID),
    ]


@pytest.mark.parametrize("entry", sorted(PARAMS))
def test_return_codes_before_launch(entry):
    from gsplat_b200 import _cabi

    L = _cabi.lib()
    assert len(PARAMS[entry].split()) == len(_cabi._SIGNATURES[entry][1])
    ft = _cabi.FThetaParams()
    ft.reference_poly, ft.max_angle = 0, 1.0

    def call(changes):
        args = dict(BASE, **changes)
        if args["ftheta"] == FTHETA:
            args["ftheta"] = ctypes.addressof(ft)
        return getattr(L, entry)(*[args.get(p, FAKE) for p in PARAMS[entry].split()])

    cases = _cases(entry)
    got = [(changes, call(changes)) for changes, _ in cases]
    assert got == cases
