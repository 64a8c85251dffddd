"""FTheta 3DGUT without a GPU: argument handling (what stays rejected, duck-typed parameters, malformed parameters), a
valid call reaching the library's device check, and the float64 oracle: forward-inverse round trips, the scaled
calibrations, and the reference's records (ref_ut_ftheta.npz, ref_ut_ftheta_rasterization.npz)."""
import math
import os
import re

import numpy as np
import pytest
import torch

import gsplat_b200 as gs
from gsplat_b200._cabi import GsplatB200Error
from oracle import ut as U
from tests import scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_NPZ = os.path.join(ROOT, "tests", "golden", "ref_ut_ftheta.npz")
REF_RASTER_NPZ = os.path.join(ROOT, "tests", "golden", "ref_ut_ftheta_rasterization.npz")
W, H = 96, 64


def _params(ref=0, **kw):
    params, _, _ = scene.scaled(scene.calibrations()["cross_left_120fov"], W)
    params = dict(params, reference_poly=ref)
    params.update(kw)
    return params


def _scene(N=4):
    means, quats, scales = torch.zeros(N, 3), torch.zeros(N, 4), torch.ones(N, 3)
    quats[:, 0] = 1
    K = torch.tensor([[1.0, 0, 48], [0, 1.0, 32], [0, 0, 1]])[None]
    return means, quats, scales, torch.eye(4)[None], K


def _proj(**kw):
    m, q, s, vm, K = _scene()
    return gs.fully_fused_projection_with_ut(m, q, s, None, vm, K, W, H, **kw)


def _eval(**kw):
    m, q, s, vm, K = _scene()
    offs, ids = torch.zeros(1, 4, 6, dtype=torch.int32), torch.zeros(0, dtype=torch.int32)
    return gs.rasterize_to_pixels_eval3d(m, q, s, torch.zeros(1, 4, 3), torch.ones(1, 4), vm, K, W, H, 16, offs, ids, **kw)


def _raster(**kw):
    m, q, s, vm, K = _scene(10)
    return gs.rasterization(m, q, s, torch.rand(10), torch.rand(10, 3), vm, K, W, H, packed=False, with_ut=True,
                            with_eval3d=True, **kw)


class _Duck:
    """The reference's torch class seen through its five attributes."""

    def __init__(self, **kw):
        for k, v in kw.items():
            setattr(self, k, v)


# ---- what stays rejected
@pytest.mark.parametrize("fn", [_proj, _eval, _raster])
def test_ftheta_without_coefficients_is_rejected(fn):
    with pytest.raises(NotImplementedError, match=re.escape("camera_model='ftheta'")) as e:
        fn(camera_model="ftheta")
    assert "ftheta_coeffs" in str(e.value)


@pytest.mark.parametrize("model", ["pinhole", "fisheye"])
@pytest.mark.parametrize("fn", [_proj, _eval, _raster])
def test_coefficients_with_another_model_are_rejected(fn, model):
    with pytest.raises(NotImplementedError, match="ftheta_coeffs"):
        fn(camera_model=model, ftheta_coeffs=gs.FThetaCameraDistortionParameters(**_params()))


@pytest.mark.parametrize("model", ["pinhole", "fisheye"])
@pytest.mark.parametrize("fn", [_proj, _raster])
def test_euclidean_order_stays_ftheta_only(fn, model):
    with pytest.raises(NotImplementedError, match="global_z_order"):
        fn(camera_model=model, global_z_order=False)


def test_ftheta_outside_3dgut_is_rejected():
    m, q, s, vm, K = _scene(10)
    args = (m, q, s, torch.rand(10), torch.rand(10, 3), vm, K, W, H)
    for kw in (dict(), dict(with_ut=True), dict(with_eval3d=True)):
        with pytest.raises(NotImplementedError):
            gs.rasterization(*args, packed=False, camera_model="ftheta",
                             ftheta_coeffs=gs.FThetaCameraDistortionParameters(**_params()), **kw)
    assert gs.has_3dgut() is False


# ---- accepted calls reach the device check
@pytest.mark.parametrize("ref", [0, 1])
@pytest.mark.parametrize("gzo", [True, False])
@pytest.mark.parametrize("fn", [_proj, _raster])
def test_valid_call_reaches_the_device_check(fn, gzo, ref):
    with pytest.raises(GsplatB200Error):
        fn(camera_model="ftheta", ftheta_coeffs=gs.FThetaCameraDistortionParameters(**_params(ref)), global_z_order=gzo)


@pytest.mark.parametrize("obj", [
    lambda p: gs.FThetaCameraDistortionParameters(**p),
    lambda p: _Duck(**p),
    lambda p: _Duck(**dict(p, reference_poly=gs.FThetaPolynomialType(p["reference_poly"]),
                           pixeldist_to_angle_poly=tuple(p["pixeldist_to_angle_poly"]),
                           angle_to_pixeldist_poly=np.float64(p["angle_to_pixeldist_poly"]))),
])
def test_duck_typed_parameters_are_accepted(obj):
    p = _params(1)
    with pytest.raises(GsplatB200Error):
        _eval(camera_model="ftheta", ftheta_coeffs=obj(p))
    with pytest.raises(GsplatB200Error):
        _proj(camera_model="ftheta", ftheta_coeffs=obj(p), global_z_order=False)


def test_parameters_defaults_and_types():
    d = gs.FThetaCameraDistortionParameters()
    assert d.reference_poly == 0 and d.max_angle == 0.0
    assert list(d.pixeldist_to_angle_poly) == [0.0] * 6 and list(d.angle_to_pixeldist_poly) == [0.0] * 6
    assert list(d.linear_cde) == [0.0] * 3
    assert int(gs.FThetaPolynomialType.PIXELDIST_TO_ANGLE) == 0 and int(gs.FThetaPolynomialType.ANGLE_TO_PIXELDIST) == 1
    assert "FThetaCameraDistortionParameters" in gs.__all__ and "FThetaPolynomialType" in gs.__all__


@pytest.mark.parametrize("bad", [
    dict(reference_poly=2), dict(reference_poly=0.5), dict(pixeldist_to_angle_poly=[0.0] * 5),
    dict(angle_to_pixeldist_poly=[0.0] * 7), dict(linear_cde=[1.0, 0.0]), dict(max_angle=math.nan),
    dict(linear_cde=[1.0, math.inf, 0.0]), dict(angle_to_pixeldist_poly=[0.0, math.nan, 0, 0, 0, 0]),
    dict(max_angle="wide"),
])
@pytest.mark.parametrize("fn", [_proj, _eval, _raster])
def test_malformed_parameters_raise_value_error(fn, bad):
    with pytest.raises(ValueError):
        fn(camera_model="ftheta", ftheta_coeffs=_Duck(**_params(**bad)))


@pytest.mark.parametrize("fn", [_proj, _eval, _raster])
def test_missing_attribute_raises_value_error(fn):
    p = _params()
    del p["linear_cde"]
    with pytest.raises(ValueError, match="linear_cde"):
        fn(camera_model="ftheta", ftheta_coeffs=_Duck(**p))


def test_coefficient_arrays_do_not_apply_to_ftheta():
    with pytest.raises(ValueError, match="radial_coeffs"):
        _proj(camera_model="ftheta", ftheta_coeffs=_Duck(**_params()), radial_coeffs=torch.zeros(1, 4))


# ---- the oracle
@pytest.mark.parametrize("ref", [0, 1])
@pytest.mark.parametrize("cname", list(scene.calibrations()))
def test_oracle_round_trip_at_pixel_centres(cname, ref):
    params, pp, _ = scene.scaled(scene.calibrations()[cname], W)
    cam = U.FThetaCamera(dict(params, reference_poly=ref), [[1, 0, pp[0]], [0, 1, pp[1]], [0, 0, 1]], W, H)
    jj, ii = torch.meshgrid(torch.arange(W, dtype=torch.float64), torch.arange(H, dtype=torch.float64), indexing="xy")
    u, v = jj.reshape(-1) + 0.5, ii.reshape(-1) + 0.5
    d, ok = cam.unproject(u, v)
    assert ok.all()
    np.testing.assert_allclose(d.norm(dim=-1).numpy(), 1.0, atol=1e-12)
    uv, valid = cam.project(d * 3.0, 0.1)
    inside = valid & ok
    assert inside.float().mean() > 0.8
    # three Newton steps from a consistent pair of polynomials invert to well below a thousandth of a pixel
    np.testing.assert_allclose(uv[inside].numpy(), torch.stack([u, v], -1)[inside].numpy(), atol=1e-3)


@pytest.mark.parametrize("cname", ["cross_left_120fov", "front_tele_30fov"])
def test_scaled_calibration_is_s_times_the_original(cname):
    cal = scene.calibrations()[cname]
    params, pp, (w, h) = scene.scaled(cal, W)
    s = W / cal["resolution"][0]
    assert (w, h) == (W, round(cal["resolution"][1] * s))
    np.testing.assert_allclose(pp, np.asarray(cal["principal_point"]) * s)
    th = torch.linspace(0.0, cal["max_angle"], 50, dtype=torch.float64)
    np.testing.assert_allclose(U.poly(params["angle_to_pixeldist_poly"], th).numpy(),
                               s * U.poly(cal["angle_to_pixeldist_poly"], th).numpy(), rtol=1e-12, atol=1e-12)
    delta = U.poly(cal["angle_to_pixeldist_poly"], th)
    np.testing.assert_allclose(U.poly(params["pixeldist_to_angle_poly"], s * delta).numpy(),
                               U.poly(cal["pixeldist_to_angle_poly"], delta).numpy(), rtol=1e-9, atol=1e-12)


def test_synthetic_calibration_sees_beyond_180_degrees():
    cal = scene.calibrations()["synthetic_wide_190"]
    assert cal["max_angle"] > math.pi / 2 + 0.2 and cal["reference_poly"] == 0
    cam = U.FThetaCamera(dict(scene.scaled(cal, W)[0], reference_poly=0), [[1, 0, 47.3], [0, 1, 31.6], [0, 0, 1]], W, H)
    pc = torch.tensor([[math.sin(1.75), 0.0, math.cos(1.75)]], dtype=torch.float64) * 2.0  # z < 0
    uv, valid = cam.project(pc, 0.1)
    assert bool(valid[0]) and 0 <= float(uv[0, 0]) < W


@pytest.mark.parametrize("cname", list(scene.calibrations()))
def test_oracle_reproduces_reference_records(cname):
    import sys

    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_ref_ut_ftheta_golden import ORDERS, POLYS

    z = np.load(REF_NPZ)
    params, _, _ = scene.scaled(scene.calibrations()[cname], W)
    K = z[f"{cname}/Ks"][0]
    for pname, ref in POLYS.items():
        for oname, gzo in ORDERS.items():
            for rolling in ((False, True) if (pname, oname) == ("ptoa", "dist") else (False,)):
                name = f"{cname}/{pname}/{oname}" + ("/rs" if rolling else "")
                cam = U.FThetaCamera(dict(params, reference_poly=ref), K, W, H)
                pose = U.ShutterPoses(z["viewmats"][0], z["viewmats_rs"][0], 0) if rolling else z["viewmats"][0]
                o = U.ut_projection(z["means"], z["quats"], z["scales"], z["opacities"], pose, cam, global_z_order=gzo)
                r, rr = o["radii"].numpy(), z[f"{name}/radii"][0]
                frac = o["radii_unrounded"].numpy()
                loose = (np.abs(frac - np.round(frac)) < 1e-3).any(-1) | o["rs_edge"].numpy()
                diff = (r != rr).any(-1)
                assert (diff & ~loose).sum() <= max(2, len(r) // 100), (name, (diff & ~loose).sum())
                ok = (r > 0).all(-1) & (rr > 0).all(-1) & ~loose
                assert ok.sum() > 20, name
                np.testing.assert_allclose(o["depths"].numpy()[ok], z[f"{name}/depths"][0][ok], rtol=1e-5)
                err = np.abs(o["means2d"].numpy()[ok] - z[f"{name}/means2d"][0][ok]).max(-1)
                assert (err > 5e-3).sum() <= max(1, ok.sum() // 100), name


def test_reference_rasterization_record():
    z = np.load(REF_RASTER_NPZ)
    N, C = z["means"].shape[0], z["viewmats"].shape[0]
    assert (int(z["width"]), int(z["height"])) == (W, H) and C == 2 and int(z["sh_degree"]) == 3
    shapes = dict(render_colors=(C, H, W, 4), render_alphas=(C, H, W, 1), radii=(C, N, 2), means2d=(C, N, 2),
                  depths=(C, N), v_means=(N, 3), v_quats=(N, 4), v_scales=(N, 3), v_opacities=(N,), v_sh=(N, 16, 3),
                  v_backgrounds=(C, 3))
    for k, s in shapes.items():
        assert z[k].shape == s, k
    # the two cameras share the FTheta parameters and differ in their principal points
    assert not np.array_equal(z["Ks"][0], z["Ks"][1])
    assert z["render_alphas"].mean() > 0.02
