"""The 3DGUT pair query and per-pixel contributor queries without a GPU: the seven exported names and their exact
parameters, every argument error (shapes, dtypes, tile size, K, count tensors, cameras and shutters) raised on CPU
tensors before anything needs the device, the refusal of CPU tensors, the eval3d walk's own top-K bound, and the return
codes of the five C entries (gsb200_eval3d_indices, gsb200_eval3d_contrib_*) for invalid and early-return arguments.
Every library call here returns before a kernel is launched or the device is touched: the pointers are fake and never
read."""
import inspect

import pytest
import torch

import gsplat_b200 as gs
from gsplat_b200 import _cabi, ops

OK, INVALID, UNSUPPORTED, CUDA, WORKSPACE = 0, -1, -2, -3, -4
FAKE = 1 << 20  # 16-byte aligned, never dereferenced
RS = 0  # RollingShutterType.ROLLING_TOP_TO_BOTTOM

PAIR = "rasterize_to_indices_in_range_eval3d"
NAMES = tuple(
    f"rasterize_{n}_eval3d{s}"
    for n in ("num_contributing_gaussians", "contributing_gaussian_ids", "top_contributing_gaussian_ids")
    for s in ("", "_sparse")
)
GEOM = ["means", "quats", "scales", "opacities", "viewmats", "Ks"]
CAMERA = ["camera_model", "radial_coeffs", "tangential_coeffs", "thin_prism_coeffs", "ftheta_coeffs", "rolling_shutter",
          "viewmats_rs"]
DENSE = GEOM + ["tile_offsets", "flatten_ids", "image_width", "image_height", "tile_size"]
SPARSE = GEOM + ["active_tiles", "tile_offsets", "flatten_ids", "tile_pixel_mask", "tile_pixel_cumsum", "pixel_map"]
GRID = ["image_width", "image_height", "tile_size", "tile_width", "tile_height"]
PARAMS = {
    PAIR: ["range_start", "range_end", "transmittances"] + GEOM + ["image_width", "image_height", "tile_size",
                                                                  "isect_offsets", "flatten_ids"] + CAMERA,
    "rasterize_num_contributing_gaussians_eval3d": DENSE + CAMERA,
    "rasterize_num_contributing_gaussians_eval3d_sparse": SPARSE + GRID + CAMERA,
    "rasterize_contributing_gaussian_ids_eval3d": DENSE + ["num_contributing_gaussians"] + CAMERA,
    "rasterize_contributing_gaussian_ids_eval3d_sparse": SPARSE + ["num_contributing_gaussians"] + GRID + CAMERA,
    "rasterize_top_contributing_gaussian_ids_eval3d": DENSE + ["num_depth_samples"] + CAMERA,
    "rasterize_top_contributing_gaussian_ids_eval3d_sparse": SPARSE + GRID + ["num_depth_samples"] + CAMERA,
}
C, N, W, H, AT, P = 2, 5, 40, 20, 3, 9
z = torch.zeros


@pytest.mark.parametrize("fn", (PAIR,) + NAMES)
def test_parameters(fn):
    """the 3DGS twin's layout arguments with the geometry of rasterize_to_pixels_eval3d, then its camera keywords"""
    sig = inspect.signature(getattr(gs, fn))
    assert list(sig.parameters) == PARAMS[fn]
    defaults = {k: p.default for k, p in sig.parameters.items() if p.default is not inspect.Parameter.empty}
    assert defaults == dict(camera_model="pinhole", radial_coeffs=None, tangential_coeffs=None, thin_prism_coeffs=None,
                            ftheta_coeffs=None, rolling_shutter=gs.RollingShutterType.GLOBAL, viewmats_rs=None)
    twin = inspect.signature(getattr(gs, fn.replace("_eval3d", "")))
    layout = [p for p in twin.parameters if p not in ("means2d", "conics", "opacities")]
    assert [p for p in PARAMS[fn] if p not in GEOM + CAMERA] == layout


def test_exported():
    for n in (PAIR,) + NAMES:
        assert n in gs.__all__ and getattr(gs, n) is getattr(ops, n)
    assert gs.has_3dgut() is False


def _ftheta(**changes):
    p = dict(reference_poly=0, pixeldist_to_angle_poly=[0.0, 0.01, 0.0, 0.0, 0.0, 0.0],
             angle_to_pixeldist_poly=[0.0, 100.0, 0.0, 0.0, 0.0, 0.0], max_angle=1.0, linear_cde=[1.0, 0.0, 0.0])
    p.update(changes)
    return gs.FThetaCameraDistortionParameters(**p)


def _args(fn):
    """well-formed CPU arguments of `fn` by parameter name: two cameras of N Gaussians, a 40 x 20 image on 3 x 2 tiles"""
    a = dict(means=z(N, 3), quats=z(N, 4), scales=z(N, 3), opacities=z(C, N), viewmats=z(C, 4, 4), Ks=z(C, 3, 3),
             flatten_ids=z(11, dtype=torch.int32), image_width=W, image_height=H, tile_size=16, num_depth_samples=4,
             range_start=0, range_end=1e10, transmittances=torch.ones(C, H, W), isect_offsets=z(C, 2, 3, dtype=torch.int32))
    if fn.endswith("_sparse"):
        a.update(active_tiles=z(AT, dtype=torch.int32), tile_offsets=z(AT + 1, dtype=torch.int32),
                 tile_pixel_mask=z(AT, 4, dtype=torch.int64), tile_pixel_cumsum=z(AT, dtype=torch.int64),
                 pixel_map=z(P, dtype=torch.int64), tile_width=3, tile_height=2,
                 num_contributing_gaussians=z(P, dtype=torch.int32))
    else:
        a.update(tile_offsets=z(C, 2, 3, dtype=torch.int32), num_contributing_gaussians=z(C, H, W, dtype=torch.int32))
    return a


def _call(fn, **kw):
    a = _args(fn)
    a.update(kw)
    sig = inspect.signature(getattr(gs, fn))
    return getattr(gs, fn)(**{p: a[p] for p in sig.parameters if p in a})


def _value_errors(fn):
    cases = [dict(tile_size=8), dict(means=z(N, 2)), dict(means=z(5)), dict(quats=z(N, 3)), dict(scales=z(N + 1, 3)),
             dict(opacities=z(C, N + 1)), dict(opacities=z(N)), dict(viewmats=z(C, 4, 3)), dict(viewmats=z(1, C, 4, 4)),
             dict(Ks=z(C, 3, 4)), dict(flatten_ids=z(11, 1, dtype=torch.int32)), dict(image_width=W + 100),
             # malformed cameras
             dict(camera_model="nope"), dict(radial_coeffs=z(C, 5)), dict(tangential_coeffs=z(1, 2)),
             dict(camera_model="fisheye", radial_coeffs=z(C, 6)), dict(camera_model="fisheye", thin_prism_coeffs=z(C, 4)),
             dict(camera_model="ftheta", ftheta_coeffs=_ftheta(reference_poly=2)),
             dict(camera_model="ftheta", ftheta_coeffs=_ftheta(max_angle=float("nan"))),
             dict(camera_model="ftheta", ftheta_coeffs=_ftheta(), radial_coeffs=z(C, 6)),
             dict(rolling_shutter=RS, viewmats_rs=z(1, 4, 4)), dict(rolling_shutter=7)]
    if fn == PAIR:
        cases += [dict(range_start=-1), dict(range_end=1.5), dict(transmittances=z(C, H, W + 1)),
                  dict(transmittances=z(H, W)), dict(isect_offsets=z(C + 1, 2, 3, dtype=torch.int32)),
                  dict(isect_offsets=z(C, 1, 3, dtype=torch.int32)), dict(isect_offsets=z(3, dtype=torch.int32))]
    elif fn.endswith("_sparse"):
        cases += [dict(tile_offsets=z(AT, dtype=torch.int32)), dict(tile_pixel_mask=z(AT, 3, dtype=torch.int64)),
                  dict(tile_pixel_cumsum=z(AT + 1, dtype=torch.int64)), dict(active_tiles=z(AT, 1, dtype=torch.int32)),
                  dict(pixel_map=z(P, 1, dtype=torch.int64)), dict(tile_height=1),
                  dict(active_tiles=z(0, dtype=torch.int32), tile_offsets=z(1, dtype=torch.int32),
                       tile_pixel_mask=z(0, 4, dtype=torch.int64), tile_pixel_cumsum=z(1, dtype=torch.int64))]
        if "_ids" in fn and "top" not in fn:
            cases += [dict(num_contributing_gaussians=z(P + 1, dtype=torch.int32))]
    else:
        # images of the lists against the cameras, a grid that does not cover the image, no grid
        cases += [dict(tile_offsets=z(C + 1, 2, 3, dtype=torch.int32)), dict(tile_offsets=z(C, 1, 3, dtype=torch.int32)),
                  dict(tile_offsets=z(3, dtype=torch.int32)), dict(tile_offsets=z(1, C, 2, 3, dtype=torch.int32))]
        if "_ids" in fn and "top" not in fn:
            cases += [dict(num_contributing_gaussians=z(C, H, W + 1, dtype=torch.int32)),
                      dict(num_contributing_gaussians=z(H, W, dtype=torch.int32))]
    if "top" in fn:
        cases += [dict(num_depth_samples=0), dict(num_depth_samples=-3)]
    return cases


def _type_errors(fn):
    cases = [dict(means=z(N, 3, dtype=torch.float64)), dict(quats=z(N, 4, dtype=torch.float16)),
             dict(Ks=z(C, 3, 3, dtype=torch.float64)), dict(opacities=z(C, N, dtype=torch.float64)),
             dict(flatten_ids=z(11, dtype=torch.int64)),
             dict(rolling_shutter=RS, viewmats_rs=z(C, 4, 4, dtype=torch.float64))]
    if fn == PAIR:
        cases += [dict(transmittances=z(C, H, W, dtype=torch.float64)), dict(isect_offsets=z(C, 2, 3, dtype=torch.int64))]
    elif fn.endswith("_sparse"):
        cases += [dict(tile_offsets=z(AT + 1, dtype=torch.int64)), dict(active_tiles=z(AT, dtype=torch.int64)),
                  dict(tile_pixel_mask=z(AT, 4, dtype=torch.float64)), dict(tile_pixel_cumsum=z(AT, dtype=torch.int32)),
                  dict(pixel_map=z(P, dtype=torch.int32))]
        if "_ids" in fn and "top" not in fn:
            cases += [dict(num_contributing_gaussians=z(P, dtype=torch.int64))]
    else:
        cases += [dict(tile_offsets=z(C, 2, 3, dtype=torch.int64))]
        if "_ids" in fn and "top" not in fn:
            cases += [dict(num_contributing_gaussians=z(C, H, W, dtype=torch.float32))]
    if "top" in fn:
        cases += [dict(num_depth_samples=2.0), dict(num_depth_samples="4")]
    return cases


def _not_implemented(fn):
    return [dict(camera_model="ortho"), dict(camera_model="lidar"), dict(camera_model="ftheta"),
            dict(ftheta_coeffs=_ftheta()), dict(rolling_shutter=RS), dict(viewmats_rs=z(C, 4, 4))]


@pytest.mark.parametrize("fn", (PAIR,) + NAMES)
def test_value_errors_before_the_device(fn):
    for kw in _value_errors(fn):
        with pytest.raises(ValueError):
            _call(fn, **kw)


@pytest.mark.parametrize("fn", (PAIR,) + NAMES)
def test_type_errors_before_the_device(fn):
    for kw in _type_errors(fn):
        with pytest.raises(TypeError):
            _call(fn, **kw)


@pytest.mark.parametrize("fn", (PAIR,) + NAMES)
def test_unsupported_cameras_before_the_device(fn):
    """lidar, ortho, FTheta without its parameters, a rolling shutter without end poses: the messages of the 3DGUT
    compositing ops (_ut_camera), naming this op"""
    for kw in _not_implemented(fn):
        with pytest.raises(NotImplementedError, match=fn):
            _call(fn, **kw)


def test_messages_name_the_arguments():
    fn = "rasterize_num_contributing_gaussians_eval3d"
    with pytest.raises(ValueError, match="to match the cameras"):
        _call(fn, tile_offsets=z(C + 1, 2, 3, dtype=torch.int32))
    with pytest.raises(ValueError, match="opacities"):
        _call(fn, opacities=z(C, N + 1))
    with pytest.raises(TypeError, match="opacities: expected float32"):
        _call(fn + "_sparse", opacities=z(C, N, dtype=torch.float64))
    with pytest.raises(ValueError, match="needs at least two image rows"):
        _call(fn, rolling_shutter=RS, viewmats_rs=z(C, 4, 4), image_height=1)


@pytest.mark.parametrize("fn", (PAIR,) + NAMES)
def test_cpu_tensors_raise(fn):
    """well-formed arguments pass every check and stop at the CUDA requirement: one camera set, a batch dimension, and
    each camera model and shutter"""
    batch = dict(means=z(1, N, 3), quats=z(1, N, 4), scales=z(1, N, 3), opacities=z(1, C, N), viewmats=z(1, C, 4, 4),
                 Ks=z(1, C, 3, 3), transmittances=torch.ones(1, C, H, W), isect_offsets=z(1, C, 2, 3, dtype=torch.int32))
    if not fn.endswith("_sparse"):
        batch.update(tile_offsets=z(1, C, 2, 3, dtype=torch.int32),
                     num_contributing_gaussians=z(1, C, H, W, dtype=torch.int32))
    for kw in (dict(), batch, dict(radial_coeffs=z(C, 6), tangential_coeffs=z(C, 2), thin_prism_coeffs=z(C, 4)),
               dict(camera_model="fisheye", radial_coeffs=z(C, 4)), dict(camera_model="ftheta", ftheta_coeffs=_ftheta()),
               dict(rolling_shutter=RS, viewmats_rs=z(C, 4, 4))):
        with pytest.raises(_cabi.GsplatB200Error, match="CUDA"):
            _call(fn, **kw)


def test_eval3d_bound_drives_the_error(monkeypatch):
    """the eval3d top-K forms check num_depth_samples against the eval3d walk's bound, the 3DGS forms against theirs"""
    if torch.cuda.is_available():
        bound = ops._max_depth_samples(torch.device("cuda", 0), "gsb200_eval3d_contrib_max_samples")
        assert bound == _cabi.lib().gsb200_eval3d_contrib_max_samples() and bound >= 1
    else:
        assert _cabi.lib().gsb200_eval3d_contrib_max_samples() == CUDA
    bounds = {"gsb200_contrib_max_samples": 100, "gsb200_eval3d_contrib_max_samples": 6}
    asked = []

    def fake_bound(dev, entry="gsb200_contrib_max_samples"):
        asked.append(entry)
        return bounds[entry]

    monkeypatch.setattr(ops, "_max_depth_samples", fake_bound)
    monkeypatch.setattr(ops, "require_cuda", lambda *t: torch.device("cpu"))
    launched = []
    monkeypatch.setattr(ops, "_Ctx", lambda dev: launched.append(dev))
    for fn in ("rasterize_top_contributing_gaussian_ids_eval3d", "rasterize_top_contributing_gaussian_ids_eval3d_sparse"):
        with pytest.raises(ValueError, match="exceeds 6"):
            _call(fn, num_depth_samples=7)
        with pytest.raises(TypeError):  # K = 6 passes the bound and reaches the launch (here a stub)
            _call(fn, num_depth_samples=6)
    assert len(launched) == 2 and set(asked) == {"gsb200_eval3d_contrib_max_samples"}
    from tests.test_contrib_cpu import _call as call_3dgs

    with pytest.raises(TypeError):  # 7 is within the 3DGS bound
        call_3dgs("rasterize_top_contributing_gaussian_ids", num_depth_samples=7)
    assert len(launched) == 3 and asked[-1] == "gsb200_contrib_max_samples"


# ---------------------------------------------------------------------------------------------- C ABI return codes
GEOM_C = ("B C N means quats scales opacities viewmats Ks camera_model radial tangential thin ftheta viewmats_rs "
          "rolling_shutter")
LAYOUT = ("W H tile_size tw th offsets flatten_ids n_isects n_active active_tiles tile_pixel_mask tile_pixel_cumsum "
          "pixel_map")
ENTRY_PARAMS = {
    "gsb200_eval3d_indices": f"{GEOM_C} transmittances W H tile_size tw th offsets flatten_ids n_isects range_start "
                             "range_end emit workspace workspace_bytes total gaussian_ids pixel_ids image_ids stream",
    "gsb200_eval3d_contrib_count": f"{GEOM_C} {LAYOUT} counts alphas stream",
    "gsb200_eval3d_contrib_ids": f"{GEOM_C} {LAYOUT} max_samples ids weights stream",
    "gsb200_eval3d_contrib_top": f"{GEOM_C} {LAYOUT} num_samples ids weights stream",
}
# one camera, a 16 x 16 image of one tile, one intersection; every other pointer fake
BASE = dict(B=1, C=1, N=4, camera_model=0, radial=None, tangential=None, thin=None, ftheta=None, viewmats_rs=None,
            rolling_shutter=4, W=16, H=16, tile_size=16, tw=1, th=1, n_isects=1, n_active=0, active_tiles=None,
            alphas=None, max_samples=2, num_samples=2, range_start=0, range_end=1, emit=1, workspace_bytes=1 << 30,
            stream=None)
SPARSE_ON = dict(active_tiles=FAKE, n_active=1)

# (entry suffix, arguments changed from BASE, expected code).  None of these reaches a launch, with or without a device.
CASES = [
    # sizes first (gsb200_eval3d_fwd's checks), then the camera, then the layout, then the query's own
    ("count", dict(B=-1), INVALID),
    ("count", dict(C=-1), INVALID),
    ("count", dict(N=-1), INVALID),
    ("count", dict(tile_size=8), UNSUPPORTED),
    ("count", dict(tile_size=8, B=-1), INVALID),
    ("count", dict(W=17), INVALID),
    ("count", dict(tw=1 << 16, th=1 << 15), UNSUPPORTED),
    ("count", dict(camera_model=1), UNSUPPORTED),
    ("count", dict(camera_model=1, counts=None), UNSUPPORTED),
    ("count", dict(camera_model=3), INVALID),
    ("count", dict(ftheta=FAKE), INVALID),
    ("count", dict(rolling_shutter=RS), INVALID),
    ("count", dict(viewmats_rs=FAKE), INVALID),
    ("count", dict(rolling_shutter=9, viewmats_rs=FAKE), INVALID),
    ("count", dict(SPARSE_ON, tile_pixel_mask=None), INVALID),
    ("count", dict(SPARSE_ON, pixel_map=None), INVALID),
    ("count", dict(SPARSE_ON, n_active=1 << 31), INVALID),
    ("count", dict(SPARSE_ON, pixel_map=None, camera_model=1), UNSUPPORTED),
    ("count", dict(SPARSE_ON, pixel_map=None, W=17), INVALID),
    ("count", dict(n_isects=-1), INVALID),
    ("count", dict(n_active=-1), INVALID),
    # nothing to do
    ("count", dict(B=0), OK),
    ("count", dict(C=0, counts=None, offsets=None), OK),
    ("count", dict(W=0), OK),
    ("count", dict(H=0, means=None, viewmats=None), OK),
    ("count", dict(active_tiles=FAKE, n_active=0, B=5), OK),
    # missing inputs and outputs
    ("count", dict(offsets=None), INVALID),
    ("count", dict(means=None), INVALID),
    ("count", dict(quats=None), INVALID),
    ("count", dict(scales=None), INVALID),
    ("count", dict(opacities=None), INVALID),
    ("count", dict(viewmats=None), INVALID),
    ("count", dict(Ks=None), INVALID),
    ("count", dict(viewmats=None, n_isects=0), INVALID),  # every pixel's ray reads the camera
    ("count", dict(flatten_ids=None), INVALID),
    ("count", dict(counts=None), INVALID),
    ("count", dict(SPARSE_ON, B=0), INVALID),  # active tiles of no image
    ("count", dict(n_isects=1 << 31), UNSUPPORTED),
    ("count", dict(n_isects=1 << 31, flatten_ids=None), INVALID),
    ("ids", dict(max_samples=-1), INVALID),
    ("ids", dict(N=1 << 31), UNSUPPORTED),
    ("ids", dict(max_samples=0, ids=None, weights=None), OK),
    ("ids", dict(max_samples=0, B=-1), INVALID),
    ("ids", dict(tile_size=8), UNSUPPORTED),
    ("ids", dict(B=0), OK),
    ("ids", dict(ids=None), INVALID),
    ("ids", dict(weights=None), INVALID),
    ("ids", dict(SPARSE_ON, pixel_map=None), INVALID),
    ("ids", dict(n_isects=1 << 31), UNSUPPORTED),
    ("top", dict(num_samples=0), INVALID),
    ("top", dict(num_samples=-1), INVALID),
    ("top", dict(num_samples=0, tile_size=8), UNSUPPORTED),
    ("top", dict(num_samples=0, camera_model=1), UNSUPPORTED),
    ("top", dict(ids=None, B=-1), INVALID),
    ("indices", dict(B=-1), INVALID),
    ("indices", dict(tile_size=8), UNSUPPORTED),
    ("indices", dict(camera_model=1), UNSUPPORTED),
    ("indices", dict(rolling_shutter=RS), INVALID),
    ("indices", dict(range_start=-1), INVALID),
    ("indices", dict(emit=0, total=None), INVALID),
    ("indices", dict(range_end=0), OK),
    ("indices", dict(B=0), OK),
    ("indices", dict(n_isects=0), OK),
    ("indices", dict(transmittances=None), INVALID),
    ("indices", dict(means=None), INVALID),
    ("indices", dict(viewmats=None), INVALID),
    ("indices", dict(gaussian_ids=None), INVALID),
    ("indices", dict(W=17), INVALID),
    ("indices", dict(workspace=None), WORKSPACE),
    ("indices", dict(workspace_bytes=16), WORKSPACE),
]


@pytest.mark.parametrize("query", ["indices", "count", "ids", "top"])
def test_return_codes_before_launch(query):
    entry = "gsb200_eval3d_indices" if query == "indices" else f"gsb200_eval3d_contrib_{query}"
    L = _cabi.lib()
    assert len(ENTRY_PARAMS[entry].split()) == len(_cabi._SIGNATURES[entry][1])

    def call(changes):
        args = dict(BASE, **changes)
        return getattr(L, entry)(*[args.get(p, FAKE) for p in ENTRY_PARAMS[entry].split()])

    got = [(changes, call(changes)) for q, changes, _ in CASES if q == query]
    want = [(changes, code) for q, changes, code in CASES if q == query]
    assert got == want


def test_max_samples_entry():
    """the eval3d walk's bound: >= 1 with a device, GSB200_E_CUDA without one"""
    L = _cabi.lib()
    assert "gsb200_eval3d_contrib_max_samples" in _cabi.EXPORTED_SYMBOLS
    rc = L.gsb200_eval3d_contrib_max_samples()
    assert rc >= 1 if torch.cuda.is_available() else rc == CUDA
