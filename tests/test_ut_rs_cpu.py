"""Rolling-shutter 3DGUT without a GPU: the shutter type and its resolution, the float64 oracle's pose interpolation,
frame times and fixed-point projection (equal to the global shutter when the two poses coincide, and against the
reference's records in ref_ut_rs.npz), and the scope of the operators and of rasterization()."""
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
REF_NPZ = os.path.join(ROOT, "tests", "golden", "ref_ut_rs.npz")
REF_RASTER_NPZ = os.path.join(ROOT, "tests", "golden", "ref_ut_rs_rasterization.npz")
RS_CAMERAS = ["pinhole", "pinhole_distorted", "fisheye_radial"]
SHUTTERS = {"top_to_bottom": 0, "left_to_right": 1, "bottom_to_top": 2, "right_to_left": 3}
KEYS = {"radial": "radial_coeffs", "tangential": "tangential_coeffs", "thin": "thin_prism_coeffs"}
UT = dict(with_ut=True, with_eval3d=True)


class _Shutter:
    def __init__(self, name):
        self.name = name


# ---- the shutter type
def test_rolling_shutter_type():
    T = gs.RollingShutterType
    assert "RollingShutterType" in gs.__all__
    assert [(m.name, int(m)) for m in T] == [("ROLLING_TOP_TO_BOTTOM", 0), ("ROLLING_LEFT_TO_RIGHT", 1),
                                              ("ROLLING_BOTTOM_TO_TOP", 2), ("ROLLING_RIGHT_TO_LEFT", 3), ("GLOBAL", 4)]


@pytest.mark.parametrize("arg,want", [
    (None, 4), (4, 4), (0, 0), (3, 3), (gs.RollingShutterType.ROLLING_LEFT_TO_RIGHT, 1), (_Shutter("GLOBAL"), 4),
    (_Shutter("ROLLING_BOTTOM_TO_TOP"), 2), ("GLOBAL", 4), ("RollingShutterType.GLOBAL", 4),
    ("RollingShutterType.ROLLING_RIGHT_TO_LEFT", 3),
])
def test_shutter_resolution(arg, want):
    from gsplat_b200.ops import _shutter_type

    assert int(_shutter_type(arg)) == want


@pytest.mark.parametrize("arg", [5, -1, _Shutter("SIDEWAYS"), "NOPE"])
def test_unknown_shutter_raises(arg):
    from gsplat_b200.ops import _shutter_type

    with pytest.raises(ValueError, match="rolling_shutter"):
        _shutter_type(arg)


# ---- the oracle's pieces
def test_frame_time_at_pixel_centres():
    W, H = 7, 5
    jj, ii = np.meshgrid(np.arange(W), np.arange(H), indexing="xy")
    u, v = torch.from_numpy(jj + 0.5), torch.from_numpy(ii + 0.5)
    np.testing.assert_array_equal(U.frame_time(0, W, H, u, v).numpy(), ii / (H - 1))
    np.testing.assert_array_equal(U.frame_time(1, W, H, u, v).numpy(), jj / (W - 1))
    np.testing.assert_array_equal(U.frame_time(2, W, H, u, v).numpy(), (H - 1 - ii) / (H - 1))
    np.testing.assert_array_equal(U.frame_time(3, W, H, u, v).numpy(), (W - 1 - jj) / (W - 1))
    # not clamped: a point in the margin has a time outside [0, 1]
    assert float(U.frame_time(0, W, H, torch.tensor(0.0), torch.tensor(-2.5))) < 0
    assert float(U.frame_time(1, W, H, torch.tensor(W + 3.5), torch.tensor(0.0))) > 1


def _quat(axis, deg):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    h = math.radians(deg) / 2
    return torch.tensor([math.cos(h), *(math.sin(h) * axis)], dtype=torch.float64)


def test_slerp_ends_and_branches():
    q0, q1 = _quat([0, 0, 1], 10.0), _quat([1, 2, 0], 35.0)
    a = torch.tensor([0.0, 1.0], dtype=torch.float64)
    np.testing.assert_allclose(U.slerp(q0, q1, a).numpy(), torch.stack([q0, q1]).numpy(), atol=1e-15)
    # the short arc: -q1 is the same rotation
    np.testing.assert_allclose(U.slerp(q0, -q1, a).numpy(), torch.stack([q0, q1]).numpy(), atol=1e-15)
    # constant angular speed: halfway is half the angle
    mid = U.slerp(q0, q1, torch.tensor([0.5], dtype=torch.float64))[0]
    ang = lambda p, q: 2 * math.acos(min(1.0, abs(float((p * q).sum()))))  # noqa: E731
    assert abs(ang(q0, mid) - ang(mid, q1)) < 1e-12
    # near-parallel (cos > 1 - FLT_EPSILON): the normalised component-wise lerp
    q2 = _quat([1, 2, 0], 35.0 + 1e-3)
    assert float((q1 * q2).sum()) > 1 - U.FLT_EPS
    s = U.slerp(q1, q2, torch.tensor([0.25, 1.5], dtype=torch.float64))
    lerp = torch.stack([0.75 * q1 + 0.25 * q2, -0.5 * q1 + 1.5 * q2])
    np.testing.assert_allclose(s.numpy(), (lerp / lerp.norm(dim=-1, keepdim=True)).numpy(), atol=1e-15)


def test_quaternion_of_a_pose():
    for axis, deg in (([0, 0, 1], 10.0), ([1, -2, 3], 170.0), ([1, 0, 0], 179.0), ([0, 1, 0.1], -120.0)):
        q = _quat(axis, deg)
        got = U.quat_from_rotmat(U.quat_to_rotmat(q))
        np.testing.assert_allclose((got * torch.sign((got * q).sum())).numpy(), q.numpy(), atol=1e-14)


# ---- the oracle with both poses equal is the global shutter
def _small(n=200):
    sc = scene.make_scene(n_max=n, sh_degree=0, seed=0)
    W, H = 96, 64
    K = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[0]
    return sc, sc["viewmats"][0], K, W, H


@pytest.mark.parametrize("shutter", [0, 1, 2, 3])
@pytest.mark.parametrize("kind,coeffs", [("pinhole", {}), ("pinhole", dict(radial=[0.08, -0.03, 0.005, 0.01, 0, 0])),
                                         ("fisheye", dict(radial=[0.04, -0.01, 0.002, -0.0003]))])
def test_oracle_without_motion_is_global(shutter, kind, coeffs):
    sc, vm, K, W, H = _small()
    cam = U.Camera(kind, K, W, H, **coeffs)
    s = sc["scales"] * 4.0
    g = U.ut_projection(sc["means"], sc["quats"], s, sc["opacities"], vm, cam)
    r = U.ut_projection(sc["means"], sc["quats"], s, sc["opacities"], U.ShutterPoses(vm, vm, shutter), cam)
    assert g["valid"].sum() > 20
    assert torch.equal(g["valid"], r["valid"])
    # the float32 view matrix is orthonormal to ~1e-7 only; its quaternion is the nearest rotation
    for k in ("means2d", "depths", "conics", "compensations"):
        np.testing.assert_allclose(r[k].numpy(), g[k].numpy(), rtol=1e-5, atol=1e-6)
    o0, d0, ok0 = U.pixel_rays(vm, cam)
    o1, d1, ok1 = U.pixel_rays(U.ShutterPoses(vm, vm, shutter), cam)
    assert torch.equal(ok0, ok1)
    np.testing.assert_allclose(o1.numpy(), o0.numpy(), atol=1e-5)
    np.testing.assert_allclose(d1.numpy(), d0.numpy(), atol=1e-6)


def test_sh_camera_position_is_the_mean():
    _, vm, _, _, _ = _small(10)
    R = U.quat_to_rotmat(_quat([0, 1, 0], 20.0)).numpy()
    vm1 = vm.astype(np.float64).copy()
    vm1[:3, :3] = R @ vm1[:3, :3]
    vm1[:3, 3] += [0.1, -0.2, 0.05]
    avg = U.rs_sh_viewmat(vm, vm1).numpy()
    pos = lambda m: -m[:3, :3].T @ m[:3, 3]  # noqa: E731
    np.testing.assert_allclose(pos(avg), 0.5 * (pos(vm.astype(np.float64)) + pos(vm1)), atol=1e-12)


# ---- the oracle against the reference's records
def ref_case(z, cname):
    model = "fisheye" if cname.startswith("fisheye") else "pinhole"
    coeffs = {short: z[f"{cname}/{k}"][0] for short, k in KEYS.items() if f"{cname}/{k}" in z.files}
    return model, coeffs


@pytest.mark.parametrize("sname", list(SHUTTERS))
@pytest.mark.parametrize("cname", RS_CAMERAS)
def test_oracle_against_reference(cname, sname):
    z = np.load(REF_NPZ)
    W, H = int(z["width"]), int(z["height"])
    model, coeffs = ref_case(z, cname)
    cam = U.Camera(model, z["Ks"][0], W, H, **coeffs)
    o = U.ut_projection(z["means"], z["quats"], z["scales"], z["opacities"],
                        U.ShutterPoses(z["viewmats"][0], z["viewmats_rs"][0], SHUTTERS[sname]), cam)
    name = f"{cname}/{sname}"
    rr = z[f"{name}/radii"][0]
    ro = o["radii"].numpy()
    frac = o["radii_unrounded"].numpy()
    # a sigma point on a row (column) boundary may take the neighbouring row's pose in float32; a radius on an integer
    # may round apart
    loose = o["rs_edge"].numpy() | (np.abs(frac - np.round(frac)) < 1e-3).any(-1)
    diff = (rr != ro).any(-1)
    assert (diff & ~loose).sum() <= max(1, len(rr) // 200), (diff & ~loose).sum()
    ok = (rr > 0).all(-1) & (ro > 0).all(-1) & ~loose
    assert ok.sum() > 50
    np.testing.assert_allclose(o["means2d"].numpy()[ok], z[f"{name}/means2d"][0][ok], rtol=1e-4, atol=5e-3)
    np.testing.assert_allclose(o["depths"].numpy()[ok], z[f"{name}/depths"][0][ok], rtol=1e-5)
    cref = z[f"{name}/conics"][0][ok]
    np.testing.assert_allclose(o["conics"].numpy()[ok], cref, rtol=5e-3, atol=5e-3 * np.abs(cref).max())


def test_reference_records_have_motion_and_shapes():
    z = np.load(REF_NPZ)
    W, H = int(z["width"]), int(z["height"])
    assert (W, H) == (96, 64)
    N = len(z["means"])
    assert z["viewmats_rs"].shape == (1, 4, 4) and not np.allclose(z["viewmats_rs"], z["viewmats"])
    for cname in RS_CAMERAS:
        for sname in SHUTTERS:
            name = f"{cname}/{sname}"
            assert z[f"{name}/radii"].shape == (1, N, 2) and z[f"{name}/render_colors"].shape == (1, H, W, 1)
            assert z[f"{name}/flatten_ids"].dtype == np.int32 and len(z[f"{name}/flatten_ids"]) > 100
            assert z[f"{name}/render_alphas"].mean() > 0.02
    assert z["colors"].shape == (N, 1) and int(z["cotangent_seed"]) >= 0
    r = np.load(REF_RASTER_NPZ)
    C = r["viewmats"].shape[0]
    assert C == 2 and r["render_colors"].shape == (C, H, W, 4) and int(r["sh_degree"]) == 3
    assert r["viewmats_rs"].shape == (C, 4, 4) and r["v_viewmats_rs"].shape == (C, 4, 4)
    assert np.abs(r["v_viewmats_rs"]).sum() > 0


# ---- scope
def _scene(C=1, N=4, B=()):
    means, quats, scales = torch.zeros(B + (N, 3)), torch.zeros(B + (N, 4)), torch.ones(B + (N, 3))
    quats[..., 0] = 1
    vm = torch.eye(4).expand(B + (C, 4, 4)).clone()
    K = torch.tensor([[50.0, 0, 16], [0, 50.0, 16], [0, 0, 1]]).expand(B + (C, 3, 3)).clone()
    return means, quats, scales, vm, K


def _proj(width=32, height=32, **kw):
    m, q, s, vm, K = _scene()
    return gs.fully_fused_projection_with_ut(m, q, s, None, vm, K, width, height, **kw)


def _eval(width=32, height=32, **kw):
    m, q, s, vm, K = _scene()
    args = dict(means=m, quats=q, scales=s, colors=torch.zeros(1, 4, 3), opacities=torch.ones(1, 4), viewmats=vm, Ks=K,
                image_width=width, image_height=height, tile_size=16,
                isect_offsets=torch.zeros(1, (height + 15) // 16, (width + 15) // 16, dtype=torch.int32),
                flatten_ids=torch.zeros(0, dtype=torch.int32))
    args.update(kw)
    return gs.rasterize_to_pixels_eval3d(**args)


def _raster(width=64, height=64, **kw):
    N = 10
    quats = torch.zeros(N, 4)
    quats[:, 0] = 1
    K = torch.tensor([[50.0, 0, 32], [0, 50.0, 32], [0, 0, 1]])[None]
    return gs.rasterization(torch.rand(N, 3), quats, torch.rand(N, 3), torch.rand(N), torch.rand(N, 3), torch.eye(4)[None], K,
                            width, height, packed=False, **UT, **kw)


RS = torch.eye(4)[None]
OPS = {"projection": _proj, "eval3d": _eval, "rasterization": _raster}


@pytest.mark.parametrize("shutter", [0, 1, 2, 3, gs.RollingShutterType.ROLLING_TOP_TO_BOTTOM, _Shutter("ROLLING_RIGHT_TO_LEFT")])
@pytest.mark.parametrize("op", list(OPS))
def test_accepted_call_reaches_the_device_check(op, shutter):
    with pytest.raises(GsplatB200Error):
        OPS[op](rolling_shutter=shutter, viewmats_rs=RS)


def test_accepted_sh_and_fisheye_calls_reach_the_device_check():
    with pytest.raises(GsplatB200Error):
        _raster(rolling_shutter=2, viewmats_rs=RS, camera_model="fisheye", radial_coeffs=torch.zeros(1, 4),
                render_mode="RGB+ED", backgrounds=torch.rand(1, 3))
    with pytest.raises(GsplatB200Error):
        gs.rasterization(torch.rand(2, 10, 3), torch.nn.functional.normalize(torch.rand(2, 10, 4), dim=-1), torch.rand(2, 10, 3),
                         torch.rand(2, 10), torch.rand(10, 16, 3), torch.eye(4).expand(2, 3, 4, 4), torch.eye(3).expand(2, 3, 3, 3),
                         64, 64, sh_degree=3, packed=False, rolling_shutter=0, viewmats_rs=torch.eye(4).expand(2, 3, 4, 4), **UT)
    with pytest.raises(GsplatB200Error):
        gs.spherical_harmonics(3, torch.rand(1, 10, 3), torch.eye(4)[None], torch.rand(10, 16, 3), viewmats_rs=torch.eye(4)[None])


# (keyword arguments, exception, text the message names)
REJECTED = [
    (dict(rolling_shutter=0), NotImplementedError, "rolling_shutter"),
    (dict(rolling_shutter=_Shutter("ROLLING_TOP_TO_BOTTOM")), NotImplementedError, "rolling_shutter"),
    (dict(viewmats_rs=RS), NotImplementedError, "viewmats_rs"),
    (dict(rolling_shutter=4, viewmats_rs=RS), NotImplementedError, "viewmats_rs"),
    (dict(rolling_shutter=9, viewmats_rs=RS), ValueError, "rolling_shutter"),
    (dict(rolling_shutter=0, viewmats_rs=torch.eye(4)[None].expand(2, 4, 4)), ValueError, "viewmats_rs"),
    (dict(rolling_shutter=0, viewmats_rs=RS, ftheta_coeffs=object()), NotImplementedError, "ftheta_coeffs"),
    (dict(rolling_shutter=0, viewmats_rs=RS, camera_model="ftheta"), NotImplementedError, "camera_model='ftheta'"),
    (dict(rolling_shutter=0, viewmats_rs=RS, camera_model="lidar"), NotImplementedError, "camera_model='lidar'"),
    (dict(rolling_shutter=0, viewmats_rs=RS, external_distortion_coeffs=object()), NotImplementedError, "external_distortion_coeffs"),
]


@pytest.mark.parametrize("kw,exc,names", REJECTED, ids=[f"{e.__name__}-{n}-{i}" for i, (_, e, n) in enumerate(REJECTED)])
@pytest.mark.parametrize("op", list(OPS))
def test_rejected_combinations(op, kw, exc, names):
    with pytest.raises(exc, match=re.escape(names)):
        OPS[op](**kw)


@pytest.mark.parametrize("kw,exc,names", [
    (dict(packed=True), ValueError, "Packed mode"),
    (dict(tile_size=8), ValueError, "tile_size"),
    (dict(distributed=True), ValueError, "distributed"),
    (dict(rays=torch.zeros(1, 64, 64, 6)), NotImplementedError, "rays"),
    (dict(render_mode="RGB-Ed"), NotImplementedError, "render_mode='RGB-Ed'"),
    (dict(return_normals=True), NotImplementedError, "return_normals"),
])
def test_rolling_rasterization_keeps_the_3dgut_scope(kw, exc, names):
    N = 10
    quats = torch.zeros(N, 4)
    quats[:, 0] = 1
    args = (torch.rand(N, 3), quats, torch.rand(N, 3), torch.rand(N), torch.rand(N, 3), torch.eye(4)[None], torch.eye(3)[None], 64, 64)
    kw = dict(dict(packed=False), **kw)
    with pytest.raises(exc, match=re.escape(names)):
        gs.rasterization(*args, **UT, rolling_shutter=0, viewmats_rs=RS, **kw)


@pytest.mark.parametrize("kw", [dict(with_ut=True), dict(with_eval3d=True), dict()])
def test_rolling_shutter_without_3dgut_is_rejected(kw):
    N = 10
    quats = torch.zeros(N, 4)
    quats[:, 0] = 1
    args = (torch.rand(N, 3), quats, torch.rand(N, 3), torch.rand(N), torch.rand(N, 3), torch.eye(4)[None], torch.eye(3)[None], 64, 64)
    with pytest.raises(NotImplementedError):
        gs.rasterization(*args, packed=False, rolling_shutter=0, viewmats_rs=RS, **kw)
    with pytest.raises(NotImplementedError, match="rolling_shutter"):
        gs.rasterization(*args, packed=False, rolling_shutter=gs.RollingShutterType.ROLLING_LEFT_TO_RIGHT)


@pytest.mark.parametrize("shutter,size", [(0, (32, 1)), (2, (32, 1)), (1, (1, 32)), (3, (1, 32))])
@pytest.mark.parametrize("op", list(OPS))
def test_single_row_or_column_raises(op, shutter, size):
    w, h = size
    with pytest.raises(ValueError, match="two image"):
        OPS[op](width=w, height=h, rolling_shutter=shutter, viewmats_rs=RS)


def test_sh_rejects_a_mismatched_end_pose():
    with pytest.raises(ValueError, match="viewmats_rs"):
        gs.spherical_harmonics(0, torch.rand(1, 10, 3), torch.eye(4)[None], torch.rand(10, 1, 3), viewmats_rs=torch.eye(4)[None].expand(2, 4, 4))
