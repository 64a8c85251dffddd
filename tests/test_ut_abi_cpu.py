"""The return codes of the dense 3DGUT compositing entries (gsb200_eval3d_fwd / _bwd) for invalid or early-return
arguments, including which check fires first: the intersection count, the sizes, tile size, grid and 2^31 limits, every
rule of the camera and the shutter, the zero-size returns, each null pointer and the channel count.  Every call here
returns before a kernel is launched or the device is touched: the pointers are fake and never read."""
import ctypes
import math

import pytest

OK, INVALID, UNSUPPORTED = 0, -1, -2
FAKE = 1 << 20  # 16-byte aligned, never dereferenced

CAMERA = "camera_model radial tangential thin ftheta viewmats_rs rolling_shutter"
GEOM = "B C N D means quats scales colors opacities backgrounds masks viewmats Ks"
GRID = "W H tile_size tw th offsets flatten_ids n_isects"
PARAMS = {
    "gsb200_eval3d_fwd": f"{GEOM} {CAMERA} {GRID} render_colors render_alphas last_ids stream",
    "gsb200_eval3d_bwd": f"{GEOM} {CAMERA} {GRID} render_alphas last_ids v_render_colors v_render_alphas grad_records "
    "v_colors v_opacities v_means v_quats v_scales stream",
}
# one 16 x 16 image, N = 4, one intersection, D = 3, the perfect pinhole under the global shutter; every other pointer
# fake and 16-byte aligned
BASE = dict(B=1, C=1, N=4, D=3, W=16, H=16, tile_size=16, tw=1, th=1, n_isects=1, camera_model=0, rolling_shutter=4,
            backgrounds=None, masks=None, radial=None, tangential=None, thin=None, ftheta=None, viewmats_rs=None,
            v_render_alphas=None, stream=None)
ROLLING = dict(rolling_shutter=0, viewmats_rs=FAKE)
# FTheta parameters: valid, or with one field out of its domain (replaced by the address of a gsb200_ftheta_params)
FTHETA = {
    "ftheta": {},
    "ftheta_poly2": dict(reference_poly=2),
    "ftheta_poly-1": dict(reference_poly=-1),
    "ftheta_max_inf": dict(max_angle=math.inf),
    "ftheta_max_nan": dict(max_angle=math.nan),
    "ftheta_bw_nan": dict(pixeldist_to_angle_poly=(0, 1, 0, 0, 0, math.nan)),
    "ftheta_fw_inf": dict(angle_to_pixeldist_poly=(0, 1, 0, -math.inf, 0, 0)),
    "ftheta_cde_nan": dict(linear_cde=(1, math.nan, 0)),
}
FT = dict(camera_model=3, ftheta="ftheta")


def _cases(entry):
    fwd = entry.endswith("_fwd")
    common = [
        (dict(n_isects=-1), INVALID),
        (dict(n_isects=-1, B=-1), INVALID),
        (dict(n_isects=-1, tile_size=8), INVALID),  # the intersection count comes first
        (dict(n_isects=-1, camera_model=1), INVALID),
        (dict(B=-1), INVALID),
        (dict(C=-1), INVALID),
        (dict(N=-1), INVALID),
        (dict(B=-1, tile_size=8), INVALID),  # the sizes before the tile size
        (dict(tile_size=8), UNSUPPORTED),
        (dict(tile_size=8, W=17), UNSUPPORTED),  # the tile size before the grid
        (dict(tile_size=8, camera_model=1), UNSUPPORTED),
        (dict(W=17), INVALID),  # one 16-pixel tile column for a 17-pixel wide image
        (dict(H=17), INVALID),
        (dict(tw=0), INVALID),
        (dict(W=17, B=1 << 16, C=1 << 15), INVALID),  # the grid before the 2^31 limits
        (dict(W=17, camera_model=1), INVALID),
        (dict(N=1 << 31), UNSUPPORTED),  # B * C * N >= 2^31
        (dict(B=1 << 16, C=1 << 15), UNSUPPORTED),  # B * C * tw * th >= 2^31
        (dict(B=1, tw=1 << 16, th=1 << 15), UNSUPPORTED),
        (dict(B=1 << 16, C=1 << 15, camera_model=3), UNSUPPORTED),  # the sizes before the camera
        # camera_checks, rule by rule
        (dict(camera_model=1), UNSUPPORTED),
        (dict(camera_model=-1), UNSUPPORTED),
        (dict(camera_model=4), UNSUPPORTED),
        (dict(camera_model=1, rolling_shutter=5), UNSUPPORTED),  # the model before the shutter
        (dict(camera_model=3), INVALID),  # FTheta without its parameters
        (dict(ftheta="ftheta"), INVALID),  # parameters without FTheta
        (dict(camera_model=2, ftheta="ftheta"), INVALID),
        (dict(FT, radial=FAKE), INVALID),
        (dict(FT, tangential=FAKE), INVALID),
        (dict(FT, thin=FAKE), INVALID),
        (dict(FT, ftheta="ftheta_poly2"), INVALID),
        (dict(FT, ftheta="ftheta_poly-1"), INVALID),
        (dict(FT, ftheta="ftheta_max_inf"), INVALID),
        (dict(FT, ftheta="ftheta_max_nan"), INVALID),
        (dict(FT, ftheta="ftheta_bw_nan"), INVALID),
        (dict(FT, ftheta="ftheta_fw_inf"), INVALID),
        (dict(FT, ftheta="ftheta_cde_nan"), INVALID),
        (dict(FT, ftheta="ftheta_poly2", rolling_shutter=5), INVALID),
        (dict(rolling_shutter=-1), INVALID),
        (dict(rolling_shutter=5), INVALID),
        (dict(rolling_shutter=5, viewmats_rs=FAKE), INVALID),
        (dict(rolling_shutter=0), INVALID),  # a rolling shutter without its end pose
        (dict(rolling_shutter=3), INVALID),
        (dict(viewmats_rs=FAKE), INVALID),  # an end pose under the global shutter
        (dict(ROLLING, H=1), INVALID),  # top to bottom over one row
        (dict(rolling_shutter=2, viewmats_rs=FAKE, H=1), INVALID),
        (dict(rolling_shutter=1, viewmats_rs=FAKE, W=1), INVALID),  # left to right over one column
        (dict(rolling_shutter=3, viewmats_rs=FAKE, W=1), INVALID),
        (dict(rolling_shutter=1, viewmats_rs=FAKE, W=1, B=0), INVALID),  # the camera before the zero-size return
        (dict(camera_model=1, B=0), UNSUPPORTED),
        (dict(FT, ftheta="ftheta_cde_nan", N=0), INVALID),
        (dict(D=6, means=None), INVALID),  # the pointers before the channel count
        (dict(D=6), UNSUPPORTED),
        (dict(D=0), UNSUPPORTED),
        (dict(D=-3), UNSUPPORTED),
        (dict(D=6, **FT), UNSUPPORTED),
        (dict(D=6, **ROLLING), UNSUPPORTED),
        (dict(D=6, camera_model=3, ftheta="ftheta", **ROLLING), UNSUPPORTED),
        (dict(means=None), INVALID),
        (dict(colors=None), INVALID),
        (dict(opacities=None), INVALID),
        (dict(viewmats=None), INVALID),
        (dict(Ks=None), INVALID),
        (dict(offsets=None), INVALID),
        (dict(flatten_ids=None), INVALID),
        (dict(Ks=None, **ROLLING), INVALID),
        (dict(flatten_ids=None, **FT), INVALID),
    ]
    if fwd:
        return common + [
            (dict(B=0), OK),
            (dict(C=0), OK),
            (dict(W=0), OK),
            (dict(H=0), OK),
            (dict(W=0, tw=0), OK),
            (dict(B=0, W=17), OK),  # the grid is checked for images only
            (dict(C=0, D=6, viewmats=None, render_colors=None), OK),  # nothing is read for no image
            (dict(B=0, **FT), OK),
            (dict(ROLLING, C=0), OK),
            (dict(quats=None), INVALID),
            (dict(scales=None), INVALID),
            (dict(render_colors=None), INVALID),
            (dict(render_alphas=None), INVALID),
            (dict(last_ids=None), INVALID),
            (dict(render_colors=None, n_isects=0), INVALID),
            (dict(offsets=None, n_isects=0), INVALID),
            (dict(viewmats=None, n_isects=0), INVALID),
            (dict(Ks=None, n_isects=0), INVALID),
            (dict(D=6, render_alphas=None), INVALID),
        ]
    return common + [
        (dict(B=0), OK),  # no gaussian has a gradient
        (dict(N=0), OK),
        (dict(N=0, D=6, quats=None, grad_records=None), OK),
        (dict(B=0, W=17), OK),
        (dict(N=0, **FT), OK),
        (dict(N=0, **ROLLING), OK),
        (dict(quats=None), INVALID),
        (dict(scales=None), INVALID),
        (dict(grad_records=None), INVALID),
        (dict(v_means=None), INVALID),
        (dict(v_quats=None), INVALID),
        (dict(v_scales=None), INVALID),
        (dict(quats=None, n_isects=0), INVALID),  # the finish kernel's pointers, also without intersections
        (dict(v_scales=None, C=0), INVALID),
        (dict(grad_records=None, W=0), INVALID),
        (dict(v_means=None, D=6), INVALID),
        (dict(render_alphas=None), INVALID),
        (dict(last_ids=None), INVALID),
        (dict(v_render_colors=None), INVALID),
        (dict(v_colors=None), INVALID),
        (dict(v_opacities=None), INVALID),
        (dict(v_colors=None, D=6), INVALID),
    ]


@pytest.mark.parametrize("entry", sorted(PARAMS))
def test_return_codes_before_launch(entry):
    from gsplat_b200 import _cabi

    L = _cabi.lib()
    assert len(PARAMS[entry].split()) == len(_cabi._SIGNATURES[entry][1])
    fts = {}
    for name, fields in FTHETA.items():
        ft = _cabi.FThetaParams()
        ft.reference_poly, ft.max_angle = 0, 1.0
        ft.pixeldist_to_angle_poly[1] = ft.angle_to_pixeldist_poly[1] = ft.linear_cde[0] = 1.0
        for k, v in fields.items():
            if isinstance(v, tuple):
                getattr(ft, k)[:] = v
            else:
                setattr(ft, k, v)
        fts[name] = ft

    def call(changes):
        args = dict(BASE, **changes)
        if args["ftheta"] is not None:
            args["ftheta"] = ctypes.addressof(fts[args["ftheta"]])
        return getattr(L, entry)(*[args.get(p, FAKE) for p in PARAMS[entry].split()])

    cases = _cases(entry)
    got = [(changes, call(changes)) for changes, _ in cases]
    assert got == cases
