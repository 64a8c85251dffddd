"""rasterization(with_ut=True, with_eval3d=True) without a GPU: every argument outside the 3DGUT scope raises its
exception, naming the argument, before anything touches the device; a valid call fails only at the library's device
check; and the reference orchestrator's golden file has the expected keys and shapes."""
import os
import re

import numpy as np
import pytest
import torch

import gsplat_b200 as gs
from gsplat_b200._cabi import GsplatB200Error

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_NPZ = os.path.join(ROOT, "tests", "golden", "ref_ut_rasterization.npz")
REF_RASTER_CAMERAS = ["pinhole", "pinhole_distorted", "fisheye_radial"]
N = 10
UT = dict(with_ut=True, with_eval3d=True)


def _args():
    quats = torch.zeros(N, 4)
    quats[:, 0] = 1
    K = torch.tensor([[50.0, 0, 32], [0, 50.0, 32], [0, 0, 1]])[None]
    return (torch.rand(N, 3), quats, torch.rand(N, 3), torch.rand(N), torch.rand(N, 3), torch.eye(4)[None], K, 64, 64)


class _Config:
    pass


def _config(name):
    return type(name, (_Config,), {})()


class _Shutter:
    def __init__(self, name):
        self.name = name


# (keyword arguments, exception, text the message names)
SCOPE = [
    (dict(), ValueError, "Packed mode"),  # packed=True is the signature's default
    (dict(packed=True), ValueError, "Packed mode"),
    (dict(packed=False, rasterize_mode="antialiased"), ValueError, "rasterize_mode"),
    (dict(packed=False, covars=torch.eye(3).expand(N, 3, 3)), ValueError, "covars"),
    (dict(packed=False, distributed=True), ValueError, "distributed"),
    (dict(packed=False, tile_size=8), ValueError, "tile_size"),
    (dict(packed=False, sparse_grad=True), ValueError, "Sparse grad"),
    (dict(packed=False, render_mode="d"), NotImplementedError, "render_mode='d'"),
    (dict(packed=False, render_mode="Ed"), NotImplementedError, "render_mode='Ed'"),
    (dict(packed=False, render_mode="RGB-d"), NotImplementedError, "render_mode='RGB-d'"),
    (dict(packed=False, render_mode="RGB-Ed"), NotImplementedError, "render_mode='RGB-Ed'"),
    (dict(packed=False, return_normals=True), NotImplementedError, "return_normals"),
    (dict(packed=False, rays=torch.zeros(1, 64, 64, 6)), NotImplementedError, "rays"),
    (dict(packed=False, camera_model="ftheta"), NotImplementedError, "camera_model='ftheta'"),
    (dict(packed=False, camera_model="lidar"), NotImplementedError, "camera_model='lidar'"),
    (dict(packed=False, camera_model="ortho"), NotImplementedError, "camera_model='ortho'"),
    (dict(packed=False, ftheta_coeffs=object()), NotImplementedError, "ftheta_coeffs"),
    (dict(packed=False, lidar_coeffs=object()), NotImplementedError, "lidar_coeffs"),
    (dict(packed=False, external_distortion_coeffs=object()), NotImplementedError, "external_distortion_coeffs"),
    (dict(packed=False, rolling_shutter=0), NotImplementedError, "rolling_shutter"),
    (dict(packed=False, rolling_shutter=_Shutter("ROLLING_TOP_TO_BOTTOM")), NotImplementedError, "rolling_shutter"),
    (dict(packed=False, viewmats_rs=torch.eye(4)[None]), NotImplementedError, "viewmats_rs"),
    (dict(packed=False, global_z_order=False), NotImplementedError, "global_z_order"),
    (dict(packed=False, renderer_config=_config("RendererConfig_ParallelBatch")), NotImplementedError, "renderer_config"),
    (dict(packed=False, extra_signals=torch.zeros(N, 2)), NotImplementedError, "extra_signals"),
]


@pytest.mark.parametrize("kw,exc,names", SCOPE, ids=[f"{e.__name__}-{n}" for _, e, n in SCOPE])
def test_3dgut_scope(kw, exc, names):
    with pytest.raises(exc, match=re.escape(names)):
        gs.rasterization(*_args(), **UT, **kw)


@pytest.mark.parametrize("kw", [dict(with_ut=True), dict(with_eval3d=True), dict(with_ut=True, packed=False),
                                dict(with_eval3d=True, packed=False)])
def test_one_flag_alone_is_not_built(kw):
    with pytest.raises(NotImplementedError, match="with_ut/with_eval3d"):
        gs.rasterization(*_args(), **kw)


@pytest.mark.parametrize("name,val", [
    ("radial_coeffs", torch.zeros(1, 6)), ("tangential_coeffs", torch.zeros(1, 2)), ("thin_prism_coeffs", torch.zeros(1, 4)),
    ("ut_params", object()),
])
def test_camera_arguments_without_the_pair(name, val):
    for packed in (True, False):
        with pytest.raises(NotImplementedError, match=name):
            gs.rasterization(*_args(), packed=packed, **{name: val})


@pytest.mark.parametrize("kw", [
    dict(),
    dict(render_mode="RGB+ED", backgrounds=torch.rand(1, 3), radial_coeffs=torch.zeros(1, 6),
         tangential_coeffs=torch.zeros(1, 2), thin_prism_coeffs=torch.zeros(1, 4)),
    dict(camera_model="fisheye", radial_coeffs=torch.zeros(1, 4), render_mode="D"),
    dict(renderer_config=_config("RendererConfig_MixedBatch"), rolling_shutter=_Shutter("GLOBAL"), absgrad=True,
         tile_size=16, channel_chunk=4, render_mode="ED"),
    dict(rolling_shutter=4, global_z_order=True, ut_params=type("P", (), {"alpha": 0.5})()),
])
def test_valid_call_reaches_the_device_check(kw):
    with pytest.raises(GsplatB200Error):
        gs.rasterization(*_args(), packed=False, **UT, **kw)


def test_valid_call_with_sh_and_batch_dims_reaches_the_device_check():
    m, q, s, o, _, vm, K, w, h = _args()
    B = 2
    with pytest.raises(GsplatB200Error):
        gs.rasterization(m.expand(B, N, 3), q.expand(B, N, 4), s.expand(B, N, 3), o.expand(B, N), torch.rand(N, 16, 3),
                         vm.expand(B, 2, 4, 4), K.expand(B, 2, 3, 3), w, h, sh_degree=3, packed=False,
                         radial_coeffs=torch.zeros(B, 2, 6), **UT)


def test_malformed_arguments():
    args = _args()
    with pytest.raises(ValueError):  # opacities of the wrong length
        gs.rasterization(*args[:3], torch.rand(N + 1), *args[4:], packed=False, **UT)
    with pytest.raises(ValueError):  # backgrounds of the wrong width
        gs.rasterization(*args, packed=False, backgrounds=torch.rand(1, 4), **UT)
    with pytest.raises(ValueError):  # radial coefficients of the wrong width
        gs.rasterization(*args, packed=False, radial_coeffs=torch.zeros(1, 5), **UT)
    with pytest.raises(ValueError):  # a chunk wider than the compositing kernels take
        gs.rasterization(*args[:4], torch.rand(N, 40), *args[5:], packed=False, channel_chunk=64, **UT)
    with pytest.raises(ValueError):
        gs.rasterization(*args, packed=False, camera_model="nope", **UT)
    with pytest.raises(TypeError):
        gs.rasterization(*args[:4], args[4].double(), *args[5:], packed=False, **UT)
    assert gs.has_3dgut() is False


def test_reference_orchestrator_golden_file():
    z = np.load(REF_NPZ)
    W, H = int(z["width"]), int(z["height"])
    assert (W, H) == (96, 64) and int(z["sh_degree"]) == 3
    N, C = z["means"].shape[0], z["viewmats"].shape[0]
    assert C == 2
    shapes = dict(means=(N, 3), quats=(N, 4), scales=(N, 3), opacities=(N,), sh=(N, 16, 3), viewmats=(C, 4, 4),
                  Ks=(C, 3, 3), backgrounds=(C, 3), v_render_colors=(C, H, W, 4), v_render_alphas=(C, H, W, 1))
    for k, s in shapes.items():
        assert z[k].shape == s and z[k].dtype == np.float32, k
    th, tw = (H + 15) // 16, (W + 15) // 16
    coeff_width = {"pinhole_distorted": {"radial_coeffs": 6, "tangential_coeffs": 2, "thin_prism_coeffs": 4},
                   "fisheye_radial": {"radial_coeffs": 4}, "pinhole": {}}
    for name in REF_RASTER_CAMERAS:
        per = dict(render_colors=(C, H, W, 4), render_alphas=(C, H, W, 1), radii=(C, N, 2), means2d=(C, N, 2), depths=(C, N),
                   isect_offsets=(C, th, tw))
        per.update({f"v_{k}": shapes[k] for k in ("means", "quats", "scales", "opacities", "sh", "backgrounds")})
        per.update({k: (C, w) for k, w in coeff_width[name].items()})
        for k, s in per.items():
            assert z[f"{name}/{k}"].shape == s, (name, k)
        present = {k for k in ("radial_coeffs", "tangential_coeffs", "thin_prism_coeffs") if f"{name}/{k}" in z.files}
        assert present == set(coeff_width[name]), name
        fl = z[f"{name}/flatten_ids"]
        assert fl.ndim == 1 and fl.dtype == np.int32 and len(fl) > 100 and z[f"{name}/radii"].dtype == np.int32
        assert fl.min() >= 0 and fl.max() < C * N
        assert (np.diff(z[f"{name}/isect_offsets"].reshape(-1)) >= 0).all()
        assert z[f"{name}/render_alphas"].mean() > 0.02
