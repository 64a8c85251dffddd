"""numpy front-end of the CPU oracle (oracle/libgs_oracle.so).

TEST INFRASTRUCTURE ONLY.  Importable from tests/, ``__graft_entry__.smoke()`` and
``bench.py``'s cpu_baseline / ``--impl reference`` legs -- never from ``gsplat_b200``.

Function names and argument meaning follow the reference's Python operator surface
(/root/reference/gsplat/cuda/_wrapper.py): ``fully_fused_projection`` (:819),
``spherical_harmonics`` (:436), ``isect_tiles`` (:1196), ``isect_offset_encode`` (:1328),
``rasterize_to_pixels`` (:1497), ``quat_scale_to_covar_preci`` (:657).  All arrays are
numpy; the float dtype of ``means``/``means2d`` (float32 or float64) selects the
``_f32`` / ``_f64`` instantiation of the C code.
"""
from __future__ import annotations

import ctypes
import math
import os
import subprocess
from typing import Optional, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libgs_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    """Compile the C restatement (gcc) if needed; returns the .so path."""
    src = [os.path.join(_HERE, f) for f in ("gs_oracle.c", "gso_impl.h")]
    stale = (not os.path.exists(_LIB_PATH)) or any(
        os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in src
    )
    if force or stale:
        subprocess.check_call(["make", "-C", _HERE, "-B", "libgs_oracle.so"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_LIB_PATH)
        _lib.gso_bits_for_count.restype = ctypes.c_uint32
        _lib.gso_bits_for_count.argtypes = [ctypes.c_int64]
        for suf in ("_f32", "_f64"):
            getattr(_lib, "gso_isect_count" + suf).restype = ctypes.c_int64
    return _lib


def _p(a: Optional[np.ndarray]):
    if a is None:
        return ctypes.c_void_p(0)
    assert a.flags["C_CONTIGUOUS"], "oracle expects contiguous arrays"
    return ctypes.c_void_p(a.ctypes.data)


def _suf(a: np.ndarray) -> Tuple[str, type, type]:
    if a.dtype == np.float32:
        return "_f32", np.float32, ctypes.c_float
    if a.dtype == np.float64:
        return "_f64", np.float64, ctypes.c_double
    raise TypeError(f"unsupported dtype {a.dtype}")


def _c(a, dt):
    return None if a is None else np.ascontiguousarray(a, dtype=dt)


def bits_for_count(count: int) -> int:
    return int(lib().gso_bits_for_count(int(count)))


# --------------------------------------------------------------------------
def quat_scale_to_covar_preci(quats, scales, compute_covar=True, compute_preci=True, triu=False):
    suf, dt, _ = _suf(quats)
    quats, scales = _c(quats, dt), _c(scales, dt)
    lead = quats.shape[:-1]
    N = int(np.prod(lead)) if lead else 1
    shp = lead + ((6,) if triu else (3, 3))
    cov = np.empty(shp, dt) if compute_covar else None
    pre = np.empty(shp, dt) if compute_preci else None
    rc = getattr(lib(), "gso_quat_scale_to_covar_preci" + suf)(
        ctypes.c_int64(N), _p(quats), _p(scales), ctypes.c_int(int(triu)), _p(cov), _p(pre)
    )
    assert rc == 0
    return cov, pre


def quat_scale_to_covar_preci_bwd(quats, scales, triu, v_covars, v_precis):
    suf, dt, _ = _suf(quats)
    quats, scales = _c(quats, dt), _c(scales, dt)
    v_covars, v_precis = _c(v_covars, dt), _c(v_precis, dt)
    N = int(np.prod(quats.shape[:-1]))
    v_q, v_s = np.empty_like(quats), np.empty_like(scales)
    rc = getattr(lib(), "gso_quat_scale_to_covar_preci_bwd" + suf)(
        ctypes.c_int64(N), _p(quats), _p(scales), ctypes.c_int(int(triu)), _p(v_covars), _p(v_precis), _p(v_q), _p(v_s)
    )
    assert rc == 0
    return v_q, v_s


# --------------------------------------------------------------------------
def _bcn(means, viewmats):
    batch = means.shape[:-2]
    B = int(np.prod(batch)) if batch else 1
    return batch, B, viewmats.shape[-3], means.shape[-2]


CAMERA_MODELS = {"pinhole": 0, "ortho": 1, "fisheye": 2}  # reference CameraModelType, ext.cpp:58-64


def fully_fused_projection(
    means, covars, quats, scales, viewmats, Ks, width, height, eps2d=0.3, near_plane=0.01, far_plane=1e10,
    radius_clip=0.0, calc_compensations=False, camera_model="pinhole", opacities=None,
):
    """Dense (packed=False) projection.  covars: [..., N, 6] triu or None."""
    cam_id = CAMERA_MODELS[camera_model]
    suf, dt, cr = _suf(means)
    batch, B, C, N = _bcn(means, viewmats)
    means, covars, quats, scales = _c(means, dt), _c(covars, dt), _c(quats, dt), _c(scales, dt)
    opacities, viewmats, Ks = _c(opacities, dt), _c(viewmats, dt), _c(Ks, dt)
    radii = np.zeros(batch + (C, N, 2), np.int32)
    means2d = np.zeros(batch + (C, N, 2), dt)
    depths = np.zeros(batch + (C, N), dt)
    conics = np.zeros(batch + (C, N, 3), dt)
    comps = np.zeros(batch + (C, N), dt) if calc_compensations else None
    rc = getattr(lib(), "gso_projection_fwd" + suf)(
        ctypes.c_int64(B), ctypes.c_int64(C), ctypes.c_int64(N), _p(means), _p(covars), _p(quats), _p(scales),
        _p(opacities), _p(viewmats), _p(Ks), ctypes.c_uint32(width), ctypes.c_uint32(height), cr(eps2d),
        cr(near_plane), cr(far_plane), cr(radius_clip), ctypes.c_int(cam_id), _p(radii), _p(means2d), _p(depths),
        _p(conics), _p(comps),
    )
    assert rc == 0
    return radii, means2d, depths, conics, comps


def fully_fused_projection_bwd(
    means, covars, quats, scales, viewmats, Ks, width, height, eps2d, radii, conics, compensations,
    v_means2d, v_depths, v_conics, v_compensations=None, viewmats_requires_grad=False, camera_model="pinhole",
):
    suf, dt, cr = _suf(means)
    batch, B, C, N = _bcn(means, viewmats)
    means, covars, quats, scales = _c(means, dt), _c(covars, dt), _c(quats, dt), _c(scales, dt)
    viewmats, Ks, conics = _c(viewmats, dt), _c(Ks, dt), _c(conics, dt)
    compensations, v_compensations = _c(compensations, dt), _c(v_compensations, dt)
    v_means2d, v_depths, v_conics = _c(v_means2d, dt), _c(v_depths, dt), _c(v_conics, dt)
    radii = np.ascontiguousarray(radii, np.int32)
    v_means = np.empty_like(means)
    v_covars = np.empty_like(covars) if covars is not None else None
    v_quats = np.empty_like(quats) if covars is None else None
    v_scales = np.empty_like(scales) if covars is None else None
    v_viewmats = np.empty_like(viewmats) if viewmats_requires_grad else None
    rc = getattr(lib(), "gso_projection_bwd" + suf)(
        ctypes.c_int64(B), ctypes.c_int64(C), ctypes.c_int64(N), _p(means), _p(covars), _p(quats), _p(scales),
        _p(viewmats), _p(Ks), ctypes.c_uint32(width), ctypes.c_uint32(height), cr(eps2d),
        ctypes.c_int(CAMERA_MODELS[camera_model]), _p(radii),
        _p(conics), _p(compensations), _p(v_means2d), _p(v_depths), _p(v_conics), _p(v_compensations), _p(v_means),
        _p(v_covars), _p(v_quats), _p(v_scales), _p(v_viewmats),
    )
    assert rc == 0
    return v_means, v_covars, v_quats, v_scales, v_viewmats


# --------------------------------------------------------------------------
def spherical_harmonics(degrees_to_use, means, viewmats, coeffs, masks=None):
    """means [..., N, 3], viewmats [..., C, 4, 4], coeffs [N, K, D] -> [..., C, N, D]."""
    suf, dt, _ = _suf(means)
    batch, B, C, N = _bcn(means, viewmats)
    means, viewmats, coeffs = _c(means, dt), _c(viewmats, dt), _c(coeffs, dt)
    K, D = coeffs.shape[-2:]
    m = None if masks is None else np.ascontiguousarray(masks, np.uint8)
    out = np.zeros(batch + (C, N, D), dt)
    rc = getattr(lib(), "gso_sh_fwd" + suf)(
        ctypes.c_int64(B), ctypes.c_int64(C), ctypes.c_int64(N), ctypes.c_int64(K), ctypes.c_int64(D),
        ctypes.c_int(degrees_to_use), _p(means), _p(viewmats), _p(coeffs), _p(m), _p(out),
    )
    assert rc == 0, "bad SH degree / K"
    return out


def spherical_harmonics_bwd(degrees_to_use, means, viewmats, coeffs, masks, v_colors, compute_v_means=True):
    suf, dt, _ = _suf(means)
    batch, B, C, N = _bcn(means, viewmats)
    means, viewmats, coeffs, v_colors = _c(means, dt), _c(viewmats, dt), _c(coeffs, dt), _c(v_colors, dt)
    K, D = coeffs.shape[-2:]
    m = None if masks is None else np.ascontiguousarray(masks, np.uint8)
    v_coeffs = np.empty_like(coeffs)
    v_means = np.empty_like(means) if compute_v_means else None
    rc = getattr(lib(), "gso_sh_bwd" + suf)(
        ctypes.c_int64(B), ctypes.c_int64(C), ctypes.c_int64(N), ctypes.c_int64(K), ctypes.c_int64(D),
        ctypes.c_int(degrees_to_use), _p(means), _p(viewmats), _p(coeffs), _p(m), _p(v_colors), _p(v_coeffs),
        _p(v_means),
    )
    assert rc == 0
    return v_coeffs, v_means


# --------------------------------------------------------------------------
def isect_tiles(
    means2d, radii, depths, tile_size, tile_width, tile_height, sort=True, conics=None, opacities=None,
):
    """Dense layout [..., N, *].  Returns tiles_per_gauss, isect_ids (int64), flatten_ids (int32)."""
    suf, dt, _ = _suf(means2d)
    image_dims = means2d.shape[:-2]
    I = int(np.prod(image_dims)) if image_dims else 1
    N = means2d.shape[-2]
    means2d, depths = _c(means2d, dt), _c(depths, dt)
    conics, opacities = _c(conics, dt), _c(opacities, dt)
    radii = np.ascontiguousarray(radii, np.int32)
    image_bits = bits_for_count(I)
    tile_bits = bits_for_count(tile_width * tile_height)
    if image_bits + tile_bits > 32:
        raise RuntimeError("intersect_tile: (image, tile) id packing needs more than 32 bits")
    tpg = np.zeros(image_dims + (N,), np.int32)
    L = lib()
    total = getattr(L, "gso_isect_count" + suf)(
        ctypes.c_int64(I), ctypes.c_int64(N), _p(means2d), _p(radii), _p(conics), _p(opacities),
        ctypes.c_uint32(tile_size), ctypes.c_uint32(tile_width), ctypes.c_uint32(tile_height), _p(tpg),
    )
    isect_ids = np.empty((total,), np.int64)
    flatten_ids = np.empty((total,), np.int32)
    if total:
        rc = getattr(L, "gso_isect_emit" + suf)(
            ctypes.c_int64(I), ctypes.c_int64(N), _p(means2d), _p(radii), _p(depths), _p(conics), _p(opacities),
            ctypes.c_uint32(tile_size), ctypes.c_uint32(tile_width), ctypes.c_uint32(tile_height),
            ctypes.c_uint32(tile_bits), _p(isect_ids), _p(flatten_ids),
        )
        assert rc == 0
        if sort:
            ks, vs = np.empty_like(isect_ids), np.empty_like(flatten_ids)
            rc = L.gso_sort_pairs(
                ctypes.c_int64(total), ctypes.c_int(32 + tile_bits + image_bits), _p(isect_ids), _p(flatten_ids),
                _p(ks), _p(vs),
            )
            assert rc == 0
            isect_ids, flatten_ids = ks, vs
    return tpg, isect_ids, flatten_ids


def isect_offset_encode(isect_ids, n_images, tile_width, tile_height):
    isect_ids = np.ascontiguousarray(isect_ids, np.int64)
    off = np.zeros((n_images, tile_height, tile_width), np.int32)
    rc = lib().gso_isect_offsets(
        ctypes.c_int64(isect_ids.shape[0]), _p(isect_ids), ctypes.c_int64(n_images), ctypes.c_uint32(tile_width),
        ctypes.c_uint32(tile_height), _p(off),
    )
    assert rc == 0
    return off


# --------------------------------------------------------------------------
def rasterize_to_pixels(
    means2d, conics, colors, opacities, image_width, image_height, tile_size, isect_offsets, flatten_ids,
    backgrounds=None, masks=None, return_aux=False,
):
    """Dense layout [..., N, *]; returns (render_colors [...,H,W,D], render_alphas [...,H,W,1])
    and, with return_aux, also (last_ids [...,H,W] int32, margins [...,H,W] float32)."""
    suf, dt, _ = _suf(means2d)
    image_dims = means2d.shape[:-2]
    I = int(np.prod(image_dims)) if image_dims else 1
    N, D = means2d.shape[-2], colors.shape[-1]
    th, tw = isect_offsets.shape[-2:]
    means2d, conics, colors, opacities = _c(means2d, dt), _c(conics, dt), _c(colors, dt), _c(opacities, dt)
    backgrounds = _c(backgrounds, dt)
    m = None if masks is None else np.ascontiguousarray(masks, np.uint8)
    off = np.ascontiguousarray(isect_offsets, np.int32)
    fl = np.ascontiguousarray(flatten_ids, np.int32)
    rc_ = np.zeros(image_dims + (image_height, image_width, D), dt)
    ra_ = np.zeros(image_dims + (image_height, image_width, 1), dt)
    li_ = np.zeros(image_dims + (image_height, image_width), np.int32)
    mg_ = np.ones(image_dims + (image_height, image_width), np.float32)
    rc = getattr(lib(), "gso_raster_fwd" + suf)(
        ctypes.c_int64(I), ctypes.c_int64(N), ctypes.c_int64(D), _p(means2d), _p(conics), _p(colors), _p(opacities),
        _p(backgrounds), _p(m), ctypes.c_uint32(image_width), ctypes.c_uint32(image_height), ctypes.c_uint32(tile_size),
        ctypes.c_uint32(tw), ctypes.c_uint32(th), _p(off), _p(fl), ctypes.c_int64(fl.shape[0]), _p(rc_), _p(ra_),
        _p(li_), _p(mg_),
    )
    assert rc == 0
    if return_aux:
        return rc_, ra_, li_, mg_
    return rc_, ra_


def rasterize_to_pixels_bwd(
    means2d, conics, colors, opacities, image_width, image_height, tile_size, isect_offsets, flatten_ids,
    render_alphas, last_ids, v_render_colors, v_render_alphas, backgrounds=None, masks=None, absgrad=False,
):
    """Returns dict of float64 gradients: v_means2d, v_conics, v_colors, v_opacities,
    (v_means2d_abs), mag [...,N,4] (sum of |terms| for xy / conic / opacity / colors) and
    v_backgrounds (reference: csrc/Rasterization.cpp:567-577)."""
    suf, dt, _ = _suf(means2d)
    image_dims = means2d.shape[:-2]
    I = int(np.prod(image_dims)) if image_dims else 1
    N, D = means2d.shape[-2], colors.shape[-1]
    th, tw = isect_offsets.shape[-2:]
    means2d, conics, colors, opacities = _c(means2d, dt), _c(conics, dt), _c(colors, dt), _c(opacities, dt)
    backgrounds = _c(backgrounds, dt)
    render_alphas, v_render_colors, v_render_alphas = _c(render_alphas, dt), _c(v_render_colors, dt), _c(v_render_alphas, dt)
    m = None if masks is None else np.ascontiguousarray(masks, np.uint8)
    off = np.ascontiguousarray(isect_offsets, np.int32)
    fl = np.ascontiguousarray(flatten_ids, np.int32)
    li = np.ascontiguousarray(last_ids, np.int32)
    f8 = np.float64
    out = dict(
        v_means2d=np.zeros(image_dims + (N, 2), f8), v_conics=np.zeros(image_dims + (N, 3), f8),
        v_colors=np.zeros(image_dims + (N, D), f8), v_opacities=np.zeros(image_dims + (N,), f8),
        mag=np.zeros(image_dims + (N, 4), f8),
    )
    out["v_means2d_abs"] = np.zeros(image_dims + (N, 2), f8) if absgrad else None
    rc = getattr(lib(), "gso_raster_bwd" + suf)(
        ctypes.c_int64(I), ctypes.c_int64(N), ctypes.c_int64(D), _p(means2d), _p(conics), _p(colors), _p(opacities),
        _p(backgrounds), _p(m), ctypes.c_uint32(image_width), ctypes.c_uint32(image_height), ctypes.c_uint32(tile_size),
        ctypes.c_uint32(tw), ctypes.c_uint32(th), _p(off), _p(fl), ctypes.c_int64(fl.shape[0]), _p(render_alphas),
        _p(li), _p(v_render_colors), _p(v_render_alphas), _p(out["v_means2d"]), _p(out["v_conics"]),
        _p(out["v_colors"]), _p(out["v_opacities"]), _p(out["v_means2d_abs"]), _p(out["mag"]),
    )
    assert rc == 0
    if backgrounds is not None:
        vb = (v_render_colors.astype(f8) * (1.0 - render_alphas.astype(f8))).sum(axis=(-3, -2))
        out["v_backgrounds"] = vb
    return out


# --------------------------------------------------------------------------
RENDER_MODES = ("RGB", "D", "ED", "RGB+D", "RGB+ED")


def rasterization_fwd_bwd(
    means, quats, scales, opacities, sh_coeffs, viewmats, Ks, width, height, sh_degree, v_render_colors,
    v_render_alphas, near_plane=0.01, far_plane=1e10, radius_clip=0.0, eps2d=0.3, tile_size=16, backgrounds=None,
    *, covars=None, rasterize_mode="classic", render_mode="RGB", camera_model="pinhole", viewmats_requires_grad=False,
):
    """The whole hot path on the CPU, dense layout: projection -> colours -> isect -> offsets -> raster fwd ->
    raster bwd -> colour bwd -> projection bwd.  Orchestration follows rendering._rasterization
    (/root/reference/gsplat/rendering.py:722-1106) and gsplat_b200.rendering.rasterization.

    means [..., N, 3] with optional leading batch dimensions, viewmats / Ks [..., C, 4, 4] / [..., C, 3, 3].
    ``sh_coeffs`` is the SH table [N, K, 3] when ``sh_degree`` is set, else post-activation colours [..., N, D] or
    [..., C, N, D]; None for ``render_mode`` "D" / "ED".  ``covars`` [..., N, 6] (triu) replaces quats / scales.
    ``rasterize_mode="antialiased"`` composites ``opacities * compensations``; the depth modes append the depth channel
    after the colours (background 0); "ED" / "RGB+ED" divide it by max(alpha, 1e-10).  ``v_render_colors`` is the
    cotangent of the returned render (so of the normalised depth in the ED modes).  Returns (fwd dict, grads dict)."""
    if render_mode not in RENDER_MODES:
        raise ValueError(f"render_mode {render_mode!r}")
    dt = means.dtype
    batch = means.shape[:-2]
    C, N = viewmats.shape[-3], means.shape[-2]
    I = int(np.prod(batch)) * C
    has_color = render_mode in ("RGB", "RGB+D", "RGB+ED")
    has_depth = render_mode != "RGB"
    expected = render_mode in ("ED", "RGB+ED")
    antialiased = rasterize_mode == "antialiased"
    radii, means2d, depths, conics, comps = fully_fused_projection(
        means, covars, quats, scales, viewmats, Ks, width, height, eps2d, near_plane, far_plane, radius_clip,
        antialiased, camera_model, opacities,
    )
    op_in = np.ascontiguousarray(np.broadcast_to(opacities[..., None, :], batch + (C, N)))
    op_cn = op_in * comps if antialiased else op_in
    tw, th = math.ceil(width / tile_size), math.ceil(height / tile_size)
    tpg, isect_ids, flatten_ids = isect_tiles(
        means2d, radii, depths, tile_size, tw, th, True, conics, op_cn
    )
    offsets = isect_offset_encode(isect_ids, I, tw, th).reshape(batch + (C, th, tw))
    valid = (radii > 0).all(-1)
    raw = None
    if not has_color:
        colors = depths[..., None]
    elif sh_degree is not None:
        raw = spherical_harmonics(sh_degree, means, viewmats, sh_coeffs, valid)
        colors = np.maximum(raw + dt.type(0.5), dt.type(0.0))
    else:
        per_gauss = sh_coeffs.ndim == means.ndim  # [..., N, D] shared by the cameras, else [..., C, N, D]
        colors = np.broadcast_to(sh_coeffs[..., None, :, :] if per_gauss else sh_coeffs, batch + (C, N, sh_coeffs.shape[-1]))
    if has_color and has_depth:
        colors = np.concatenate([colors, depths[..., None]], -1)
    bg = backgrounds
    if backgrounds is not None and has_depth:
        bg = np.zeros(batch + (C, 1), dt)
        if has_color:
            bg = np.concatenate([backgrounds, bg], -1)
    acc, ra, li, mg = rasterize_to_pixels(
        means2d, conics, colors, op_cn, width, height, tile_size, offsets, flatten_ids, bg, None, True
    )
    rc = acc
    if expected:
        rc = np.concatenate([acc[..., :-1], acc[..., -1:] / np.maximum(ra, 1e-10)], -1)
    fwd = dict(
        radii=radii, means2d=means2d, depths=depths, conics=conics, colors=colors, tiles_per_gauss=tpg,
        isect_ids=isect_ids, flatten_ids=flatten_ids, isect_offsets=offsets, render_colors=rc, render_alphas=ra,
        last_ids=li, margins=mg, sh_raw=raw, compensations=comps, opacities=op_cn,
    )
    if v_render_colors is None:
        return fwd, None
    v_acc, v_ra = v_render_colors, v_render_alphas
    if expected:
        # d = acc / max(alpha, 1e-10): v_acc = v_d / max(alpha, 1e-10), v_alpha += -v_d acc / alpha^2 where alpha > 1e-10
        v_d = v_render_colors[..., -1:]
        live = ra > 1e-10
        v_acc = np.concatenate([v_render_colors[..., :-1], v_d / np.maximum(ra, 1e-10)], -1)
        v_ra = v_render_alphas - np.where(live, v_d * acc[..., -1:] / np.where(live, ra, 1.0) ** 2, 0.0)
    g = rasterize_to_pixels_bwd(
        means2d, conics, colors, op_cn, width, height, tile_size, offsets, flatten_ids, ra, li, v_acc,
        v_ra, bg,
    )
    grads = dict(raster=g)
    v_feat = g["v_colors"]
    v_depths = np.zeros_like(depths)
    if has_depth:
        v_depths = v_feat[..., -1].astype(dt)
        v_feat = v_feat[..., :-1]
    v_means_sh = 0
    if has_color and sh_degree is not None:
        v_colors = (v_feat * ((raw + dt.type(0.5)) >= 0)).astype(dt)
        v_coeffs, v_means_sh = spherical_harmonics_bwd(sh_degree, means, viewmats, sh_coeffs, valid, v_colors)
        grads["v_sh"] = v_coeffs
    elif has_color:
        grads["v_colors"] = (v_feat.sum(-3) if per_gauss else v_feat).astype(dt)
    v_op = g["v_opacities"]
    v_comps = None
    if antialiased:
        v_comps = (v_op * op_in).astype(dt)
        v_op = v_op * comps
    v_means, v_covars, v_quats, v_scales, v_vm = fully_fused_projection_bwd(
        means, covars, quats, scales, viewmats, Ks, width, height, eps2d, radii, conics, comps,
        g["v_means2d"].astype(dt), v_depths, g["v_conics"].astype(dt), v_comps, viewmats_requires_grad, camera_model,
    )
    if viewmats_requires_grad and has_color and sh_degree is not None and sh_degree > 0:
        # SH view direction dir = mean + R^T t: dL/dR = t S^T, dL/dt = R S with S = sum_n dL/ddir_n per image
        mb, vmb = means.reshape((-1, N, 3)), viewmats.reshape((-1, C, 4, 4))
        vcb, vab = v_colors.reshape((-1, C, N, 3)), valid.reshape((-1, C, N))
        v_vm = v_vm.reshape((-1, C, 4, 4))
        for b in range(vmb.shape[0]):
            for c in range(C):
                _, v_dir = spherical_harmonics_bwd(
                    sh_degree, mb[b], vmb[b, c : c + 1], sh_coeffs, vab[b, c : c + 1], vcb[b, c : c + 1]
                )
                S = v_dir.sum(0)
                R, t = vmb[b, c, :3, :3], vmb[b, c, :3, 3]
                v_vm[b, c, :3, :3] += t[:, None] * S[None, :]
                v_vm[b, c, :3, 3] += R @ S
        v_vm = v_vm.reshape(viewmats.shape)
    grads.update(
        v_means=v_means + v_means_sh, v_quats=v_quats, v_scales=v_scales, v_covars=v_covars, v_viewmats=v_vm,
        v_opacities=v_op.sum(-2).astype(dt), v_compensations=v_comps,
    )
    if backgrounds is not None and has_color:
        grads["v_backgrounds"] = g["v_backgrounds"][..., : backgrounds.shape[-1]].astype(dt)
    return fwd, grads


# --------------------------------------------------------------------------
# MCMC strategy ops ("next" row): plain numpy restatements
def compute_relocation(opacities, scales, ratios, binoms, min_opacity=0.005):
    """Eq. 9 of the 3DGS-MCMC paper.  Reference: csrc/RelocationCUDA.cu:36-80 (kernel) and the reference's own
    Python restatement tests/test_relocation.py:42-76.  ratios already clamped to [1, n_max]."""
    dt = opacities.dtype
    eps = np.finfo(dt).eps
    N = opacities.shape[0]
    new_o = np.empty_like(opacities)
    new_s = np.empty_like(scales)
    for i in range(N):
        n = int(ratios[i])
        o = dt.type(1.0) - (dt.type(1.0) - opacities[i]) ** dt.type(1.0 / n)
        o = min(max(o, dt.type(min_opacity)), dt.type(1.0 - eps))
        new_o[i] = o
        denom = 0.0
        for r in range(1, n + 1):
            for k in range(r):
                denom += float(binoms[r - 1, k]) * ((-1.0) ** k) * (float(o) ** (k + 1)) / math.sqrt(k + 1)
        new_s[i] = scales[i] * dt.type(float(opacities[i]) / denom)
    return new_o, new_s


def mcmc_perturb_positions(positions, quats, scales_log, opacities_logit, noise, noise_scale, t=0.005, k=100.0):
    """positions + Sigma @ (noise * sigmoid(-k (sigmoid(o) - t)) * noise_scale).  Reference:
    csrc/MCMCPerturbCUDA.cu:28-60; PyTorch fallback gsplat/strategy/ops.py:494-512."""
    dt = positions.dtype
    cov, _ = quat_scale_to_covar_preci(quats.astype(dt), np.exp(scales_log.astype(dt)), True, False, False)
    dens = 1.0 / (1.0 + np.exp(-opacities_logit.astype(dt)))
    w = (1.0 / (1.0 + np.exp(k * (dens - t)))) * noise_scale
    nz = noise.astype(dt) * w[:, None]
    return positions + np.einsum("nij,nj->ni", cov, nz)


def adam(param, grad, exp_avg, exp_avg_sq, valid, lr, b1, b2, eps):
    """Selective Adam step without bias correction; returns the new (param, exp_avg, exp_avg_sq).
    Reference: csrc/AdamCUDA.cu:34-70 (m = b1 m + (1-b1) g; v = b2 v + (1-b2) g g; p += -lr m / (sqrt(v) + eps);
    rows with valid == False untouched).  Every operation is carried out in the array dtype, in the kernel's order."""
    dt = param.dtype.type
    lr, b1, b2, eps = dt(lr), dt(b1), dt(b2), dt(eps)
    m = b1 * exp_avg + (dt(1.0) - b1) * grad
    v = b2 * exp_avg_sq + (dt(1.0) - b2) * grad * grad
    p = param + (-lr * m / (np.sqrt(v) + eps))
    if valid is not None:
        keep = ~np.asarray(valid, bool).reshape((-1,) + (1,) * (param.ndim - 1))
        p, m, v = np.where(keep, param, p), np.where(keep, exp_avg, m), np.where(keep, exp_avg_sq, v)
    return p.astype(param.dtype), m.astype(param.dtype), v.astype(param.dtype)


def l1_loss(a, b):
    """mean |a - b| and d loss / d a = sign(a - b) / n  (the trainer's F.l1_loss; sign(0) = 0 like torch.abs)."""
    d = a.astype(np.float64) - b.astype(np.float64)
    return float(np.abs(d).mean()), (np.sign(d) / d.size).astype(a.dtype)


def fully_fused_projection_packed(*args, **kwargs):
    """packed=True bookkeeping over the dense projection (reference csrc/Projection.cpp:858-1060): the visible
    (batch, camera, gaussian) rows in ascending order.  Returns (batch_ids, camera_ids, gaussian_ids int64 [nnz],
    indptr int32 [B*C+1], radii, means2d, depths, conics, compensations) with [nnz, ...] rows."""
    radii, means2d, depths, conics, comps = fully_fused_projection(*args, **kwargs)
    C, N = radii.shape[-3], radii.shape[-2]
    vis = (radii > 0).all(-1).reshape(-1, C, N)
    b, c, n = np.nonzero(vis)
    indptr = np.concatenate([[0], np.cumsum(vis.reshape(-1, N).sum(-1))]).astype(np.int32)
    sel = vis.reshape(radii.shape[:-1])
    return (b.astype(np.int64), c.astype(np.int64), n.astype(np.int64), indptr, radii[sel], means2d[sel], depths[sel],
            conics[sel], None if comps is None else comps[sel])
