"""Operator surface: the Python functions the reference exposes in gsplat/cuda/_wrapper.py, with the
same names, argument meaning and error behaviour, implemented as torch.autograd.Function wrappers
around the C ABI of libgsplat_b200.so (include/gsplat_b200.h).

Reference wrappers mirrored here (file:line in /root/reference/gsplat/cuda/_wrapper.py):
  quat_scale_to_covar_preci :657   fully_fused_projection :819   spherical_harmonics :436
  isect_tiles :1196                isect_offset_encode :1328     rasterize_to_pixels :1497
and their autograd registrations (:559-716, :966-1191, :2010-2117).

PyTorch is plumbing here (device memory, streams, autograd graph); every number is produced by the
hand-written sm_90a kernels.
"""
from __future__ import annotations

import enum
import math
import operator
from typing import NamedTuple, Optional, Tuple

import torch
from torch import Tensor

from . import _cabi
from ._cabi import check, f32c, lib, ptr, require_cuda, stream

# --------------------------------------------------------------------------------------------
# helpers


def _prod(shape) -> int:
    return int(math.prod(shape)) if len(shape) else 1


def _rows(t: Optional[Tensor], width: int, name: str) -> Tuple[Optional[Tensor], int]:
    """Return (tensor, row_stride_in_floats) for a gradient the kernels address as ptr[row * stride + k],
    row being the C-order flattened index over the leading dims.  ``width`` > 1: t is [..., width] with a
    unit inner stride; ``width`` == 1: t is [...] (no trailing dim).  Accepts any layout whose rows sit at
    one uniform stride (e.g. views into a packed per-gaussian record); copies otherwise."""
    if t is None:
        return None, 0
    if t.dtype != torch.float32:
        raise TypeError(f"{name}: expected a float32 gradient, got {t.dtype}")
    has_inner = width > 1
    lead_shape = t.shape[:-1] if has_inner else t.shape
    lead_strides = t.stride()[:-1] if has_inner else t.stride()
    ok = (not has_inner) or (t.shape[-1] == width and t.stride(-1) == 1)
    if ok:
        row, expect = None, None
        for size, st in zip(reversed(lead_shape), reversed(lead_strides)):
            if size == 1:
                continue
            if expect is None:
                row, expect = st, st * size
            elif st != expect:
                ok = False
                break
            else:
                expect *= size
        if row is None:
            row = width
        if ok and row >= width:
            return t, int(row)
    return t.contiguous(), width


def _mask_u8(masks: Optional[Tensor]) -> Optional[Tensor]:
    """masks as the uint8 array the kernels read (a bool tensor is reinterpreted, not copied), or None"""
    if masks is None:
        return None
    return masks.contiguous().view(torch.uint8) if masks.dtype == torch.bool else masks.to(torch.uint8).contiguous()


class _Ctx:
    """device guard + stream fetch for one operator call"""

    __slots__ = ("dev", "_g")

    def __init__(self, dev: torch.device):
        self.dev = dev

    def __enter__(self):
        idx = self.dev.index
        if idx is None or torch._C._cuda_getDevice() != idx:  # not the current device: switch for the launches
            self._g = torch.cuda.device(self.dev)
            self._g.__enter__()
            return stream()
        self._g = None
        return stream(idx)

    def __exit__(self, *a):
        return self._g.__exit__(*a) if self._g is not None else None


def _camera_model_id(camera_model: str) -> int:
    table = {"pinhole": 0, "ortho": 1, "fisheye": 2, "ftheta": 3, "lidar": 4}
    if camera_model not in table:
        raise ValueError(f"unknown camera_model {camera_model!r}")
    if camera_model not in ("pinhole", "ortho", "fisheye"):
        raise NotImplementedError(
            f"camera_model={camera_model!r}: the EWA projection is built for pinhole / ortho / fisheye "
            "(reference: csrc/ProjectionEWA3DGSFused.cu:135-147); ftheta and lidar belong to the 3DGUT pipeline"
        )
    return table[camera_model]


# --------------------------------------------------------------------------------------------
# quat_scale_to_covar_preci


class _QuatScaleToCovarPreci(torch.autograd.Function):
    @staticmethod
    def forward(ctx, quats, scales, compute_covar: bool, compute_preci: bool, triu: bool):
        dev = require_cuda(quats, scales)
        q, s = f32c(quats, "quats"), f32c(scales, "scales")
        lead = q.shape[:-1]
        N = _prod(lead)
        shp = tuple(lead) + ((6,) if triu else (3, 3))
        covars = torch.empty(shp, device=dev, dtype=torch.float32) if compute_covar else None
        precis = torch.empty(shp, device=dev, dtype=torch.float32) if compute_preci else None
        with _Ctx(dev) as st:
            check(
                lib().gsb200_quat_scale_to_covar_preci_fwd(N, ptr(q), ptr(s), int(triu), ptr(covars), ptr(precis), st),
                "quat_scale_to_covar_preci",
            )
        ctx.save_for_backward(q, s)
        ctx.triu = triu
        return covars, precis

    @staticmethod
    def backward(ctx, v_covars, v_precis):
        q, s = ctx.saved_tensors
        N = _prod(q.shape[:-1])
        vc = None if v_covars is None else v_covars.contiguous()
        vp = None if v_precis is None else v_precis.contiguous()
        v_q, v_s = torch.empty_like(q), torch.empty_like(s)
        with _Ctx(q.device) as st:
            check(
                lib().gsb200_quat_scale_to_covar_preci_bwd(
                    N, ptr(q), ptr(s), int(ctx.triu), ptr(vc), ptr(vp), ptr(v_q), ptr(v_s), st
                ),
                "quat_scale_to_covar_preci_bwd",
            )
        return v_q, v_s, None, None, None


def quat_scale_to_covar_preci(
    quats: Tensor, scales: Tensor, compute_covar: bool = True, compute_preci: bool = True, triu: bool = False
) -> Tuple[Optional[Tensor], Optional[Tensor]]:
    """Quaternions (wxyz, need not be normalised) and scales -> covariance / precision matrices.
    Shapes: quats [..., 4], scales [..., 3] -> [..., 3, 3] or [..., 6] when ``triu``."""
    if quats.shape[-1] != 4 or scales.shape[-1] != 3 or quats.shape[:-1] != scales.shape[:-1]:
        raise ValueError(f"bad shapes quats {tuple(quats.shape)} scales {tuple(scales.shape)}")
    return _QuatScaleToCovarPreci.apply(quats, scales, compute_covar, compute_preci, triu)


# --------------------------------------------------------------------------------------------
# fully_fused_projection (dense)


class _FullyFusedProjection(torch.autograd.Function):
    @staticmethod
    def forward(
        ctx, means, covars, quats, scales, opacities, viewmats, Ks, width, height, eps2d, near_plane, far_plane,
        radius_clip, calc_compensations, camera_model_id,
    ):
        dev = require_cuda(means, viewmats, Ks)
        means, covars, quats, scales = f32c(means, "means"), f32c(covars, "covars"), f32c(quats, "quats"), f32c(scales, "scales")
        opacities, viewmats, Ks = f32c(opacities, "opacities"), f32c(viewmats, "viewmats"), f32c(Ks, "Ks")
        batch = tuple(means.shape[:-2])
        B, N, C = _prod(batch), means.shape[-2], viewmats.shape[-3]
        o = dict(device=dev, dtype=torch.float32)
        radii = torch.empty(batch + (C, N, 2), device=dev, dtype=torch.int32)
        means2d = torch.empty(batch + (C, N, 2), **o)
        depths = torch.empty(batch + (C, N), **o)
        conics = torch.empty(batch + (C, N, 3), **o)
        comps = torch.empty(batch + (C, N), **o) if calc_compensations else None
        with _Ctx(dev) as st:
            check(
                lib().gsb200_projection_fwd(
                    B, C, N, ptr(means), ptr(covars), ptr(quats), ptr(scales), ptr(opacities), ptr(viewmats), ptr(Ks),
                    width, height, eps2d, near_plane, far_plane, radius_clip, camera_model_id, ptr(radii), ptr(means2d),
                    ptr(depths), ptr(conics), ptr(comps), st,
                ),
                "projection_ewa_3dgs_fused",
            )
        ctx.save_for_backward(means, covars, quats, scales, viewmats, Ks, radii, conics, comps)
        ctx.meta = (width, height, eps2d, camera_model_id)
        ctx.mark_non_differentiable(radii)
        return radii, means2d, depths, conics, comps

    @staticmethod
    def backward(ctx, v_radii, v_means2d, v_depths, v_conics, v_comps):
        means, covars, quats, scales, viewmats, Ks, radii, conics, comps = ctx.saved_tensors
        width, height, eps2d, cam_id = ctx.meta
        batch = tuple(means.shape[:-2])
        B, N, C = _prod(batch), means.shape[-2], viewmats.shape[-3]
        dev = means.device
        z = lambda shape: torch.zeros(shape, device=dev, dtype=torch.float32)  # noqa: E731
        if v_means2d is None:
            v_means2d = z(batch + (C, N, 2))
        if v_depths is None:
            v_depths = z(batch + (C, N))
        if v_conics is None:
            v_conics = z(batch + (C, N, 3))
        v_means2d, s_m2 = _rows(v_means2d, 2, "v_means2d")
        v_depths, s_d = _rows(v_depths, 1, "v_depths")
        v_conics, s_c = _rows(v_conics, 3, "v_conics")
        v_comps = None if (v_comps is None or comps is None) else v_comps.contiguous()
        need_vm = ctx.needs_input_grad[5]
        v_means = torch.empty_like(means)
        v_covars = torch.empty_like(covars) if covars is not None else None
        v_quats = torch.empty_like(quats) if covars is None else None
        v_scales = torch.empty_like(scales) if covars is None else None
        v_viewmats = torch.empty_like(viewmats) if need_vm else None
        with _Ctx(dev) as st:
            check(
                lib().gsb200_projection_bwd(
                    B, C, N, ptr(means), ptr(covars), ptr(quats), ptr(scales), ptr(viewmats), ptr(Ks), width, height,
                    eps2d, cam_id, ptr(radii), ptr(conics), ptr(comps), ptr(v_means2d), s_m2, ptr(v_depths), s_d,
                    ptr(v_conics), s_c, ptr(v_comps), ptr(v_means), ptr(v_covars), ptr(v_quats), ptr(v_scales),
                    ptr(v_viewmats), st,
                ),
                "projection_ewa_3dgs_fused_bwd",
            )
        return (v_means, v_covars, v_quats, v_scales, None, v_viewmats) + (None,) * 9


class _FullyFusedProjectionPacked(torch.autograd.Function):
    """projection_ewa_3dgs_packed (/root/reference/gsplat/cuda/_wrapper.py:1065-1191): two-pass compacting
    projection; outputs are the nnz visible (batch, camera, gaussian) rows in ascending order."""

    @staticmethod
    def forward(
        ctx, means, covars, quats, scales, opacities, viewmats, Ks, width, height, eps2d, near_plane, far_plane,
        radius_clip, sparse_grad, calc_compensations, camera_model_id,
    ):
        dev = require_cuda(means, viewmats, Ks)
        means, covars, quats, scales = f32c(means, "means"), f32c(covars, "covars"), f32c(quats, "quats"), f32c(scales, "scales")
        opacities, viewmats, Ks = f32c(opacities, "opacities"), f32c(viewmats, "viewmats"), f32c(Ks, "Ks")
        batch = tuple(means.shape[:-2])
        if sparse_grad and len(batch) != 0:
            raise ValueError("sparse_grad does not support batch dimensions")
        B, N, C = _prod(batch), means.shape[-2], viewmats.shape[-3]
        if B * C > 65535:
            # same launch geometry limit as the reference's packed kernel (ProjectionEWA3DGSPacked.cu:325-333): B*C on grid.y
            raise RuntimeError(f"projection_ewa_3dgs_packed: B * C = {B * C} exceeds the CUDA grid.y limit of 65535")
        L = lib()
        o = dict(device=dev, dtype=torch.float32)
        nnz_dev = torch.empty(1, device=dev, dtype=torch.int32)
        args = (
            B, C, N, ptr(means), ptr(covars), ptr(quats), ptr(scales), ptr(opacities), ptr(viewmats), ptr(Ks), width, height,
            eps2d, near_plane, far_plane, radius_clip,
        )
        with _Ctx(dev) as st:
            ws = torch.empty(max(L.gsb200_projection_packed_workspace_bytes(B, C, N), 256), device=dev, dtype=torch.uint8)
            check(
                L.gsb200_projection_packed_count(*args, int(calc_compensations), camera_model_id, ptr(ws), ws.numel(), ptr(nnz_dev), st),
                "projection_ewa_3dgs_packed (count)",
            )
            nnz = int(nnz_dev.item())  # the host sync of the packed path (reference: Projection.cpp:924)
            ids = torch.empty((3, nnz), device=dev, dtype=torch.int64)
            indptr = torch.empty(B * C + 1, device=dev, dtype=torch.int32)
            radii = torch.empty((nnz, 2), device=dev, dtype=torch.int32)
            means2d, depths, conics = torch.empty((nnz, 2), **o), torch.empty((nnz,), **o), torch.empty((nnz, 3), **o)
            comps = torch.zeros((nnz,), **o) if calc_compensations else None
            check(
                L.gsb200_projection_packed_emit(
                    *args, camera_model_id, ptr(ws), ptr(indptr), ptr(ids[0]), ptr(ids[1]), ptr(ids[2]), ptr(radii), ptr(means2d),
                    ptr(depths), ptr(conics), ptr(comps), st,
                ),
                "projection_ewa_3dgs_packed (emit)",
            )
        batch_ids, camera_ids, gaussian_ids = ids[0], ids[1], ids[2]
        ctx.save_for_backward(means, covars, quats, scales, viewmats, Ks, batch_ids, camera_ids, gaussian_ids, conics, comps)
        ctx.meta = (width, height, eps2d, camera_model_id, bool(sparse_grad))
        ctx.mark_non_differentiable(batch_ids, camera_ids, gaussian_ids, indptr, radii)
        return batch_ids, camera_ids, gaussian_ids, indptr, radii, means2d, depths, conics, comps

    @staticmethod
    def backward(ctx, _vb, _vc, _vg, _vi, _vr, v_means2d, v_depths, v_conics, v_comps):
        means, covars, quats, scales, viewmats, Ks, batch_ids, camera_ids, gaussian_ids, conics, comps = ctx.saved_tensors
        width, height, eps2d, cam_id, sparse_grad = ctx.meta
        batch = tuple(means.shape[:-2])
        B, N, C = _prod(batch), means.shape[-2], viewmats.shape[-3]
        nnz = conics.shape[0]
        dev = means.device
        z = lambda shape: torch.zeros(shape, device=dev, dtype=torch.float32)  # noqa: E731
        v_means2d = z((nnz, 2)) if v_means2d is None else v_means2d
        v_depths = z((nnz,)) if v_depths is None else v_depths
        v_conics = z((nnz, 3)) if v_conics is None else v_conics
        v_means2d, s_m2 = _rows(v_means2d, 2, "v_means2d")
        v_depths, s_d = _rows(v_depths, 1, "v_depths")
        v_conics, s_c = _rows(v_conics, 3, "v_conics")
        v_comps = None if (v_comps is None or comps is None) else v_comps.contiguous()
        need_vm = ctx.needs_input_grad[5]
        lead = (nnz,) if sparse_grad else tuple(means.shape[:-1])
        e = lambda w: torch.empty(lead + (w,), device=dev, dtype=torch.float32)  # noqa: E731
        v_means = e(3)
        v_covars = e(6) if covars is not None else None
        v_quats = e(4) if covars is None else None
        v_scales = e(3) if covars is None else None
        v_viewmats = torch.empty_like(viewmats) if need_vm else None
        with _Ctx(dev) as st:
            check(
                lib().gsb200_projection_packed_bwd(
                    B, C, N, nnz, ptr(means), ptr(covars), ptr(quats), ptr(scales), ptr(viewmats), ptr(Ks), width, height, eps2d,
                    cam_id, ptr(batch_ids), ptr(camera_ids), ptr(gaussian_ids), ptr(conics), ptr(comps), ptr(v_means2d), s_m2,
                    ptr(v_depths), s_d, ptr(v_conics), s_c, ptr(v_comps), int(sparse_grad), ptr(v_means), ptr(v_covars),
                    ptr(v_quats), ptr(v_scales), ptr(v_viewmats), st,
                ),
                "projection_ewa_3dgs_packed_bwd",
            )
        if sparse_grad:
            # per-row gradients wrapped as COO over the gaussian index (reference Projection.cpp:1188-1206);
            # coalesced when there is a single camera (every gaussian id then appears at most once)
            idx = gaussian_ids[None]

            def coo(rows, like):
                return None if rows is None else torch.sparse_coo_tensor(idx, rows, size=like.shape, is_coalesced=(C == 1))

            v_means, v_covars = coo(v_means, means), coo(v_covars, covars)
            v_quats, v_scales = coo(v_quats, quats), coo(v_scales, scales)
        return (v_means, v_covars, v_quats, v_scales, None, v_viewmats) + (None,) * 10


def fully_fused_projection(
    means: Tensor,  # [..., N, 3]
    covars: Optional[Tensor],  # [..., N, 6] or None
    quats: Optional[Tensor],  # [..., N, 4] or None
    scales: Optional[Tensor],  # [..., N, 3] or None
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    width: int,
    height: int,
    eps2d: float = 0.3,
    near_plane: float = 0.01,
    far_plane: float = 1e10,
    radius_clip: float = 0.0,
    packed: bool = False,
    sparse_grad: bool = False,
    calc_compensations: bool = False,
    camera_model: str = "pinhole",
    opacities: Optional[Tensor] = None,  # [..., N] or None
):
    """Projects Gaussians to 2D (EWA).  Returns (radii int32 [..., C, N, 2], means2d [..., C, N, 2],
    depths [..., C, N], conics [..., C, N, 3], compensations [..., C, N] | None).  ``radii == 0`` marks
    culled entries; their float outputs are zero."""
    if sparse_grad and not packed:
        raise AssertionError("sparse_grad is only supported when packed is True")
    if covars is None and (quats is None or scales is None):
        raise ValueError("either covars or (quats, scales) must be given")
    if covars is not None:
        quats = scales = None
    cam = _camera_model_id(camera_model)
    if packed:
        # (batch_ids, camera_ids, gaussian_ids int64 [nnz], indptr int32 [B*C+1], radii [nnz,2], means2d [nnz,2],
        #  depths [nnz], conics [nnz,3], compensations [nnz] | None), rows in ascending (b, c, n) order
        return _FullyFusedProjectionPacked.apply(
            means, covars, quats, scales, opacities, viewmats, Ks, int(width), int(height), float(eps2d), float(near_plane),
            float(far_plane), float(radius_clip), bool(sparse_grad), bool(calc_compensations), cam,
        )
    return _FullyFusedProjection.apply(
        means, covars, quats, scales, opacities, viewmats, Ks, int(width), int(height), float(eps2d), float(near_plane),
        float(far_plane), float(radius_clip), bool(calc_compensations), cam,
    )


# --------------------------------------------------------------------------------------------
# spherical_harmonics (dense)


def _v_viewmats_from_dirsum(viewmats: Tensor, v_dirsum: Tensor) -> Tensor:
    """Pose gradient of the SH view directions.  dir = mean + R^T t  =>  dL/dR[i][j] = t[i] S[j],  dL/dt = R S, with
    S = v_dirsum, the sum of dL/ddir over the camera's gaussians."""
    R, t = viewmats[..., :3, :3], viewmats[..., :3, 3]
    v_viewmats = torch.zeros_like(viewmats)
    v_viewmats[..., :3, :3] = t[..., :, None] * v_dirsum[..., None, :]
    v_viewmats[..., :3, 3] = torch.einsum("...ij,...j->...i", R, v_dirsum)
    return v_viewmats


class _SphericalHarmonics(torch.autograd.Function):
    @staticmethod
    def forward(ctx, degrees_to_use, means, viewmats, coeffs, masks):
        dev = require_cuda(means, viewmats, coeffs)
        means, viewmats, coeffs = f32c(means, "means"), f32c(viewmats, "viewmats"), f32c(coeffs, "coeffs")
        batch = tuple(means.shape[:-2])
        B, N, C = _prod(batch), means.shape[-2], viewmats.shape[-3]
        K, D = coeffs.shape[-2:]
        m8 = _mask_u8(masks)
        colors = torch.empty(batch + (C, N, D), device=dev, dtype=torch.float32)
        with _Ctx(dev) as st:
            check(
                lib().gsb200_sh_fwd(B, C, N, K, D, degrees_to_use, ptr(means), ptr(viewmats), ptr(coeffs), ptr(m8), ptr(colors), st),
                "spherical_harmonics",
            )
        ctx.save_for_backward(means, viewmats, coeffs, m8)
        ctx.deg = degrees_to_use
        return colors

    @staticmethod
    def backward(ctx, v_colors):
        means, viewmats, coeffs, m8 = ctx.saved_tensors
        batch = tuple(means.shape[:-2])
        B, N, C = _prod(batch), means.shape[-2], viewmats.shape[-3]
        K, D = coeffs.shape[-2:]
        v_colors = v_colors.contiguous()
        v_coeffs = torch.empty_like(coeffs)
        v_means = torch.empty_like(means) if ctx.needs_input_grad[1] else None
        need_vm = ctx.needs_input_grad[2]
        v_dirsum = torch.empty(batch + (C, 3), device=means.device, dtype=torch.float32) if need_vm else None
        with _Ctx(means.device) as st:
            check(
                lib().gsb200_sh_bwd(
                    B, C, N, K, D, ctx.deg, ptr(means), ptr(viewmats), ptr(coeffs), ptr(m8), ptr(v_colors), ptr(v_coeffs),
                    ptr(v_means), ptr(v_dirsum), st,
                ),
                "spherical_harmonics_bwd",
            )
        v_viewmats = _v_viewmats_from_dirsum(viewmats, v_dirsum) if need_vm else None
        return None, v_means, v_viewmats, v_coeffs, None


class _SphericalHarmonicsRows(torch.autograd.Function):
    """SH colours of packed rows (batch_ids, camera_ids, gaussian_ids) with the coefficient table [N, K, D] indexed
    inside the kernel -- what rasterization(packed=True) uses instead of gathering [nnz, K, D] rows first."""

    @staticmethod
    def forward(ctx, degrees_to_use, means, viewmats, coeffs, batch_ids, camera_ids, gaussian_ids):
        dev = require_cuda(means, viewmats, coeffs)
        means, viewmats, coeffs = f32c(means, "means"), f32c(viewmats, "viewmats"), f32c(coeffs, "coeffs")
        ids = [t.to(torch.int64).contiguous() for t in (batch_ids, camera_ids, gaussian_ids)]
        batch = tuple(means.shape[:-2])
        B, N, C = _prod(batch), means.shape[-2], viewmats.shape[-3]
        K, D = coeffs.shape[-2:]
        nnz = ids[0].shape[0]
        colors = torch.empty((nnz, D), device=dev, dtype=torch.float32)
        with _Ctx(dev) as st:
            check(
                lib().gsb200_sh_rows_fwd(
                    nnz, B, C, N, K, D, degrees_to_use, ptr(means), ptr(viewmats), ptr(coeffs), ptr(ids[0]), ptr(ids[1]),
                    ptr(ids[2]), ptr(colors), st,
                ),
                "spherical_harmonics (rows)",
            )
        ctx.save_for_backward(means, viewmats, coeffs, *ids)
        ctx.deg = degrees_to_use
        return colors

    @staticmethod
    def backward(ctx, v_colors):
        means, viewmats, coeffs, b_ids, c_ids, g_ids = ctx.saved_tensors
        batch = tuple(means.shape[:-2])
        B, N, C = _prod(batch), means.shape[-2], viewmats.shape[-3]
        K, D = coeffs.shape[-2:]
        v_colors = v_colors.contiguous()
        v_coeffs = torch.empty_like(coeffs)
        v_means = torch.empty_like(means) if ctx.needs_input_grad[1] else None
        need_vm = ctx.needs_input_grad[2]
        v_dirsum = torch.empty(batch + (C, 3), device=means.device, dtype=torch.float32) if need_vm else None
        with _Ctx(means.device) as st:
            check(
                lib().gsb200_sh_rows_bwd(
                    b_ids.shape[0], B, C, N, K, D, ctx.deg, ptr(means), ptr(viewmats), ptr(coeffs), ptr(b_ids), ptr(c_ids),
                    ptr(g_ids), ptr(v_colors), ptr(v_coeffs), ptr(v_means), ptr(v_dirsum), st,
                ),
                "spherical_harmonics_bwd (rows)",
            )
        v_viewmats = _v_viewmats_from_dirsum(viewmats, v_dirsum) if need_vm else None
        return None, v_means, v_viewmats, v_coeffs, None, None, None


def _mid_position_viewmats(viewmats: Tensor, viewmats_rs: Tensor) -> Tensor:
    """View matrices [I | -c] whose camera position -R^T t is c, the mean of the positions of the two poses
    (differentiable in both): the SH view direction of a rolling-shutter camera."""
    def position(vm):
        return -torch.einsum("...ji,...j->...i", vm[..., :3, :3], vm[..., :3, 3])

    c = 0.5 * (position(viewmats) + position(viewmats_rs))
    eye = torch.eye(3, device=viewmats.device, dtype=viewmats.dtype).expand(viewmats.shape[:-2] + (3, 3))
    top = torch.cat([eye, -c[..., None]], dim=-1)
    return torch.cat([top, viewmats[..., 3:, :].detach()], dim=-2)


def spherical_harmonics_rows(
    degrees_to_use: int, means: Tensor, viewmats: Tensor, coeffs: Tensor, batch_ids: Tensor, camera_ids: Tensor,
    gaussian_ids: Tensor,
) -> Tensor:
    """SH colours [nnz, D] of the packed rows (batch_ids, camera_ids, gaussian_ids); ``coeffs`` is the full
    [N, K, D] table (NOT pre-gathered).  Same values as ``spherical_harmonics(..., coeffs[gaussian_ids], ids)``."""
    if coeffs.dim() != 3 or coeffs.shape[0] != means.shape[-2]:
        raise ValueError(f"coeffs must be [N, K, D]; got {tuple(coeffs.shape)} for N={means.shape[-2]}")
    if not (0 <= degrees_to_use <= 4) or (degrees_to_use + 1) ** 2 > coeffs.shape[-2]:
        raise ValueError(f"degrees_to_use={degrees_to_use} needs K >= {(degrees_to_use + 1) ** 2}, got {coeffs.shape[-2]}")
    return _SphericalHarmonicsRows.apply(int(degrees_to_use), means, viewmats, coeffs, batch_ids, camera_ids, gaussian_ids)


def spherical_harmonics(
    degrees_to_use: int,
    means: Tensor,  # [..., N, 3]
    viewmats: Tensor,  # [..., C, 4, 4]
    coeffs: Tensor,  # [N, K, D]
    masks: Optional[Tensor] = None,  # [..., C, N]
    batch_ids: Optional[Tensor] = None,
    camera_ids: Optional[Tensor] = None,
    gaussian_ids: Optional[Tensor] = None,
    viewmats_rs: Optional[Tensor] = None,  # [..., C, 4, 4]
) -> Tensor:
    """Evaluates SH colours for view directions ``mean - camera_position`` (camera position recovered as
    ``-R^T t``).  Returns [..., C, N, D]; masked-off rows are 0.  With ``viewmats_rs`` (a rolling shutter's end-of-frame
    poses) the camera position is the mean of the two poses' positions, and each pose gets half of its gradient."""
    if viewmats_rs is not None:
        if tuple(viewmats_rs.shape) != tuple(viewmats.shape):
            raise ValueError(f"viewmats_rs must be shaped like viewmats {tuple(viewmats.shape)}, got {tuple(viewmats_rs.shape)}")
        viewmats = _mid_position_viewmats(viewmats, viewmats_rs)
    # the reference rejects these with TORCH_CHECK (RuntimeError), csrc/SphericalHarmonics.cpp
    if not (0 <= degrees_to_use <= 4):
        raise RuntimeError(f"degrees_to_use must be between 0 and 4, got {degrees_to_use}")
    if coeffs.dim() == 3 and coeffs.shape[-1] == 0:
        raise RuntimeError("spherical_harmonics: coeffs must have at least one channel (D > 0)")
    if coeffs.dtype in (torch.float16, torch.bfloat16):
        # half-precision coefficient storage (the trainer's sh_fp16 option): evaluated in fp32 like the reference
        # kernel; the cast is differentiable, so v_coeffs comes back in the storage dtype
        coeffs = coeffs.float()
    if batch_ids is not None or camera_ids is not None or gaussian_ids is not None:
        # packed mode: coeffs [nnz, K, D] pre-gathered, one (batch, camera, gaussian) triple per row.  The view
        # direction mean + R^T t is formed per row (torch, differentiable) and evaluated by the dense kernel
        # with an identity view matrix, one "gaussian" per row.
        if batch_ids is None or camera_ids is None or gaussian_ids is None:
            raise ValueError("batch_ids, camera_ids and gaussian_ids must be given together")
        nb = means.dim() - 2
        N, C = means.shape[-2], viewmats.shape[-3]
        m = means.reshape(-1, N, 3)[batch_ids.long(), gaussian_ids.long()]  # [nnz, 3]
        vm = viewmats.reshape(-1, C, 4, 4)[batch_ids.long(), camera_ids.long()]  # [nnz, 4, 4]
        dirs = m + torch.einsum("nij,ni->nj", vm[:, :3, :3], vm[:, :3, 3])
        if coeffs.dim() != 3 or coeffs.shape[0] != dirs.shape[0]:
            raise ValueError(f"packed coeffs must be [nnz, K, D]; got {tuple(coeffs.shape)} for nnz={dirs.shape[0]}")
        if not (0 <= degrees_to_use <= 4) or (degrees_to_use + 1) ** 2 > coeffs.shape[-2]:
            raise ValueError(f"degrees_to_use={degrees_to_use} needs K >= {(degrees_to_use + 1) ** 2}")
        eye = torch.eye(4, device=dirs.device, dtype=dirs.dtype)[None]
        out = _SphericalHarmonics.apply(int(degrees_to_use), dirs, eye, coeffs, None if masks is None else masks[None])
        return out[0]
    if coeffs.dim() != 3 or coeffs.shape[0] != means.shape[-2]:
        raise ValueError(f"coeffs must be [N, K, D]; got {tuple(coeffs.shape)} for N={means.shape[-2]}")
    if not (0 <= degrees_to_use <= 4) or (degrees_to_use + 1) ** 2 > coeffs.shape[-2]:
        raise ValueError(f"degrees_to_use={degrees_to_use} needs K >= {(degrees_to_use + 1) ** 2}, got {coeffs.shape[-2]}")
    return _SphericalHarmonics.apply(int(degrees_to_use), means, viewmats, coeffs, masks)


# --------------------------------------------------------------------------------------------
# fused projection + conic + SH -> RGB (the rasterization() default path)


# Where the fused backward puts the parameter gradients.  The view-parallel trainer registers the segments of its
# symmetric (NVLS multicast) gradient buffer here, so that the backward kernel writes straight into the memory
# the all-reduce kernel works on (gsplat_b200.distributed.NvlsGradArena) -- no staging copy.
_grad_allocator = None


def set_gradient_allocator(fn) -> None:
    """fn(name, like) -> Tensor | None with name in {"means", "quats", "scales", "sh"}; None = default.
    The fused backward also asks for ``fn("seen_bits", None)``: an int32 [ceil(N / 32)] tensor that receives the
    row bitmap of the row-sparse all-reduce, or None."""
    global _grad_allocator
    _grad_allocator = fn


def _alloc_grad(name: str, like: Tensor) -> Tensor:
    if _grad_allocator is not None:
        t = _grad_allocator(name, like)
        if t is not None:
            # 16-byte aligned: the fused backward stores quaternion and SH gradient rows with 128-bit stores
            if (t.shape != like.shape or t.dtype != like.dtype or t.device != like.device or not t.is_contiguous()
                    or t.data_ptr() % 16):
                raise RuntimeError(f"gradient allocator returned a mismatching tensor for {name!r}")
            return t
    return torch.empty_like(like)


class _ProjectSH(torch.autograd.Function):
    @staticmethod
    def forward(
        ctx, means, quats, scales, opacities, sh_coeffs, viewmats, Ks, width, height, eps2d, near_plane, far_plane,
        radius_clip, sh_degree, calc_compensations, rows_out=None,
    ):
        dev = require_cuda(means, quats, scales, opacities, sh_coeffs, viewmats, Ks)
        means, quats, scales = f32c(means, "means"), f32c(quats, "quats"), f32c(scales, "scales")
        opacities, sh_coeffs = f32c(opacities, "opacities"), f32c(sh_coeffs, "colors")
        viewmats, Ks = f32c(viewmats, "viewmats"), f32c(Ks, "Ks")
        # the kernels read quaternions and SH rows with 128-bit loads: a contiguous VIEW with a storage offset (a
        # parameter carved from a flat buffer) may be only 4-byte aligned
        if quats.data_ptr() % 16:
            quats = quats.clone()
        if sh_coeffs.data_ptr() % 16:
            sh_coeffs = sh_coeffs.clone()
        N, C, K = means.shape[0], viewmats.shape[0], sh_coeffs.shape[1]
        o = dict(device=dev, dtype=torch.float32)
        radii = torch.empty((C, N, 2), device=dev, dtype=torch.int32)
        means2d, depths, conics = torch.empty((C, N, 2), **o), torch.empty((C, N), **o), torch.empty((C, N, 3), **o)
        colors = torch.empty((C, N, 3), **o)
        comps = torch.empty((C, N), **o) if calc_compensations else None
        with _Ctx(dev) as st:
            if rows_out is not None and not calc_compensations:
                # + per-row tile counts / totals and the 64-byte compositing row records (see RowSideOutputs)
                rows_out.rows = torch.empty((C, N, 16), **o)
                rows_out.tiles_per_gauss = torch.empty((C, N), device=dev, dtype=torch.int32)
                rows_out.totals = torch.empty(3, device=dev, dtype=torch.int64)
                check(
                    lib().gsb200_project_sh_fwd_rows(
                        C, N, K, sh_degree, ptr(means), ptr(quats), ptr(scales), ptr(opacities), ptr(sh_coeffs),
                        ptr(viewmats), ptr(Ks), width, height, eps2d, near_plane, far_plane, radius_clip, rows_out.tile_size,
                        rows_out.tile_width, rows_out.tile_height, ptr(radii), ptr(means2d), ptr(depths), ptr(conics),
                        ptr(colors), ptr(rows_out.rows), ptr(rows_out.tiles_per_gauss), ptr(rows_out.totals), st,
                    ),
                    "project_sh_fwd_rows",
                )
            else:
                check(
                    lib().gsb200_project_sh_fwd(
                        C, N, K, sh_degree, ptr(means), ptr(quats), ptr(scales), ptr(opacities), ptr(sh_coeffs),
                        ptr(viewmats), ptr(Ks), width, height, eps2d, near_plane, far_plane, radius_clip,
                        int(calc_compensations), ptr(radii), ptr(means2d), ptr(depths), ptr(conics), ptr(comps), ptr(colors), st,
                    ),
                    "project_sh_fwd",
                )
        ctx.save_for_backward(means, quats, scales, sh_coeffs, viewmats, Ks, radii, conics, comps, colors)
        ctx.meta = (width, height, eps2d, sh_degree)
        ctx.mark_non_differentiable(radii)
        ctx.set_materialize_grads(False)  # no zero tensors for radii / depths / compensations nobody differentiated
        return radii, means2d, depths, conics, colors, comps

    @staticmethod
    def backward(ctx, v_radii, v_means2d, v_depths, v_conics, v_colors, v_comps):
        means, quats, scales, sh_coeffs, viewmats, Ks, radii, conics, comps, colors = ctx.saved_tensors
        width, height, eps2d, sh_degree = ctx.meta
        if ctx.needs_input_grad[5]:
            raise NotImplementedError("fused project+SH path does not produce viewmats gradients")
        N, C, K = means.shape[0], viewmats.shape[0], sh_coeffs.shape[1]
        dev = means.device
        z = lambda shape: torch.zeros(shape, device=dev, dtype=torch.float32)  # noqa: E731
        if v_means2d is None:
            v_means2d = z((C, N, 2))
        if v_conics is None:
            v_conics = z((C, N, 3))
        if v_colors is None:
            v_colors = z((C, N, 3))
        v_means2d, s_m2 = _rows(v_means2d, 2, "v_means2d")
        v_depths, s_d = _rows(v_depths, 1, "v_depths")
        v_conics, s_c = _rows(v_conics, 3, "v_conics")
        v_colors, s_col = _rows(v_colors, 3, "v_colors")
        v_comps = None if (v_comps is None or comps is None) else v_comps.contiguous()
        v_means, v_quats, v_scales = _alloc_grad("means", means), _alloc_grad("quats", quats), _alloc_grad("scales", scales)
        v_sh = _alloc_grad("sh", sh_coeffs)
        # optional row bitmap for the row-sparse gradient all-reduce (distributed.NvlsGradArena): int32 [ceil(N / 32)]
        seen_bits = _grad_allocator("seen_bits", None) if _grad_allocator is not None else None
        if seen_bits is not None and (seen_bits.dtype != torch.int32 or seen_bits.numel() < (N + 31) // 32 or not seen_bits.is_contiguous()):
            raise RuntimeError("gradient allocator returned a mismatching tensor for 'seen_bits'")
        with _Ctx(dev) as st:
            check(
                lib().gsb200_project_sh_bwd(
                    C, N, K, sh_degree, ptr(means), ptr(quats), ptr(scales), ptr(sh_coeffs), ptr(viewmats), ptr(Ks),
                    width, height, eps2d, ptr(radii), ptr(conics), ptr(comps), ptr(colors), ptr(v_means2d), s_m2,
                    ptr(v_depths), s_d, ptr(v_conics), s_c, ptr(v_colors), s_col, ptr(v_comps), ptr(v_means),
                    ptr(v_quats), ptr(v_scales), ptr(v_sh), ptr(seen_bits), st,
                ),
                "project_sh_bwd",
            )
        # opacities only steer culling / radius (non-differentiable there)
        return (v_means, v_quats, v_scales, None, v_sh, None, None) + (None,) * 9


class RowSideOutputs:
    """Side outputs of the fused projection for the two stages that follow it in rasterization(): per-row tile counts
    and their totals (what gsb200_isect_count_totals would compute) and the 64-byte compositing row records
    {cull | axis | geom | rgb0} that make the pack pass a pure gather.  Valid only while the compositing runs on exactly
    the projection's means2d / conics / colours and the INPUT opacities (no antialiasing compensation, 3 channels)."""

    __slots__ = ("tile_size", "tile_width", "tile_height", "rows", "tiles_per_gauss", "totals")

    def __init__(self, tile_size: int, tile_width: int, tile_height: int):
        self.tile_size, self.tile_width, self.tile_height = int(tile_size), int(tile_width), int(tile_height)
        self.rows = self.tiles_per_gauss = self.totals = None


def fused_project_sh(
    means, quats, scales, opacities, sh_coeffs, viewmats, Ks, width, height, sh_degree, eps2d=0.3, near_plane=0.01,
    far_plane=1e10, radius_clip=0.0, calc_compensations=False, rows_out: Optional[RowSideOutputs] = None,
):
    """One pass over the gaussians: world->camera, covariance->conic, SH->RGB (+0.5, clamped at 0).
    means [N,3] quats [N,4] scales [N,3] opacities [N] sh_coeffs [N,K,3] viewmats [C,4,4] Ks [C,3,3].
    Returns (radii, means2d, depths, conics, colors [C,N,3], compensations|None)."""
    if sh_coeffs.dim() != 3 or sh_coeffs.shape[-1] != 3:
        raise ValueError("fused_project_sh needs SH coefficients [N, K, 3]")
    if not (0 <= sh_degree <= 4) or (sh_degree + 1) ** 2 > sh_coeffs.shape[1]:
        raise ValueError(f"sh_degree={sh_degree} needs K >= {(sh_degree + 1) ** 2}")
    return _ProjectSH.apply(
        means, quats, scales, opacities, sh_coeffs, viewmats, Ks, int(width), int(height), float(eps2d),
        float(near_plane), float(far_plane), float(radius_clip), int(sh_degree), bool(calc_compensations), rows_out,
    )


# --------------------------------------------------------------------------------------------
# isect_tiles / isect_offset_encode

_scratch = {}


def _scratch_buffer(dev: torch.device, tag: str, nbytes: int) -> Tensor:
    """Grow-only per-device scratch (CUB temp storage).  Stream-ordered use only."""
    key = (dev, tag, stream(dev.index))
    buf = _scratch.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 1 << 16), device=dev, dtype=torch.uint8)
        _scratch[key] = buf
    return buf


def _isect_rows(means2d, radii, depths, conics, opacities, tile_width, tile_height, n_images, image_ids):
    """The projected rows as the intersection entry points take them: contiguous float32 / int32 tensors, the int64 image
    id of each packed row (``image_ids`` given: [nnz, 2] means2d over ``n_images`` images) or None (dense
    [..., N, 2]), and (image_dims, I, N, I_count, total, packed): I images of N rows, ``total`` = I_count * N rows for
    the count, which sees packed rows as one flat list."""
    means2d, depths = f32c(means2d, "means2d"), f32c(depths, "depths")
    conics, opacities = f32c(conics, "conics"), f32c(opacities, "opacities")
    if radii.dtype != torch.int32:
        raise TypeError("radii must be int32")
    radii = radii.contiguous()
    packed = image_ids is not None
    if packed:
        image_dims, I, N, I_count = (), int(n_images), means2d.shape[0], 1
        image_ids = image_ids.to(torch.int64).contiguous()
    else:
        image_dims = tuple(means2d.shape[:-2])
        I, N = _prod(image_dims), means2d.shape[-2]
        I_count = I
    n_tiles = tile_width * tile_height
    image_bits, tile_bits = _cabi.bits_for_count(I), _cabi.bits_for_count(n_tiles)
    if image_bits + tile_bits > 32:
        raise RuntimeError(
            f"intersect_tile: (image, tile) id packing needs {image_bits + tile_bits} bits but only 32 are "
            f"available (I={I}, n_tiles={n_tiles})."
        )
    return means2d, radii, depths, conics, opacities, image_ids, (image_dims, I, N, I_count, I_count * N, packed)


@torch.no_grad()
def isect_tiles(
    means2d: Tensor,  # [..., N, 2]
    radii: Tensor,  # [..., N, 2]
    depths: Tensor,  # [..., N]
    tile_size: int,
    tile_width: int,
    tile_height: int,
    sort: bool = True,
    segmented: bool = False,
    packed: bool = False,
    n_images: Optional[int] = None,
    image_ids: Optional[Tensor] = None,
    gaussian_ids: Optional[Tensor] = None,
    conics: Optional[Tensor] = None,
    opacities: Optional[Tensor] = None,
) -> Tuple[Tensor, Tensor, Tensor]:
    """Maps projected Gaussians to the tiles they touch.  With ``conics`` and ``opacities`` the
    conservative ellipse test (AccuTile / SNUGBOX) is used, otherwise the radius AABB.
    Returns (tiles_per_gauss int32 [..., N], isect_ids int64 [n_isects], flatten_ids int32 [n_isects])."""
    dev = require_cuda(means2d, radii, depths)
    if packed:
        if n_images is None or image_ids is None:
            raise ValueError("n_images and image_ids are required when means2d is packed ([nnz, 2]).")
        if segmented:
            raise ValueError("segmented sort is not supported for packed inputs")
        if means2d.dim() != 2:
            raise ValueError(f"packed means2d must be [nnz, 2], got {tuple(means2d.shape)}")
    means2d, radii, depths, conics, opacities, img_ids, (image_dims, I, N, I_count, total, _) = _isect_rows(
        means2d, radii, depths, conics, opacities, tile_width, tile_height, n_images, image_ids if packed else None
    )
    L = lib()
    tiles_per_gauss = torch.empty(image_dims + (N,), device=dev, dtype=torch.int32)
    if total == 0:
        return (tiles_per_gauss, torch.empty(0, device=dev, dtype=torch.int64), torch.empty(0, device=dev, dtype=torch.int32))
    if sort:
        hits = isect_tiles_sorted(
            means2d, radii, depths, tile_size, tile_width, tile_height, conics=conics, opacities=opacities,
            n_images=I if packed else None, image_ids=img_ids, _exact=True,
        )
        return hits.tiles_per_gauss, hits.isect_ids(), hits.flatten_ids
    # unsorted (the reference's sort=False output): row-order count, scan, emission
    accu = conics is not None and opacities is not None
    cum = torch.empty(total, device=dev, dtype=torch.int64)
    with _Ctx(dev) as st:
        ws = _scratch_buffer(dev, "scan", L.gsb200_isect_scan_workspace_bytes(total))
        check(
            L.gsb200_isect_count(
                I_count, N, ptr(means2d), ptr(radii), ptr(conics) if accu else None, ptr(opacities) if accu else None,
                tile_size, tile_width, tile_height, ptr(tiles_per_gauss), ptr(cum), ptr(ws), ws.numel(), st,
            ),
            "intersect_tile (count)",
        )
        n_isects = int(cum[-1].item())  # the one host sync of the forward (reference: csrc/Intersect.cpp:259)
        isect_ids = torch.empty(n_isects, device=dev, dtype=torch.int64)
        flatten_ids = torch.empty(n_isects, device=dev, dtype=torch.int32)
        if n_isects == 0:
            return tiles_per_gauss, isect_ids, flatten_ids
        check(
            L.gsb200_isect_emit(
                I, N, ptr(means2d), ptr(radii), ptr(depths), ptr(conics) if accu else None,
                ptr(opacities) if accu else None, ptr(cum), ptr(img_ids), tile_size, tile_width, tile_height,
                ptr(isect_ids), ptr(flatten_ids), st,
            ),
            "intersect_tile (emit)",
        )
    return tiles_per_gauss, isect_ids, flatten_ids


class _IsectPredictor:
    """Capacities for gsb200_isect_sorted from the totals of the last calls on the same (device, image count, tile grid,
    row layout), and the asynchronous host read of the current totals (a kernel stores them into pinned memory, the host
    polls)."""

    def __init__(self, dev: torch.device):
        self.hist = []  # (n_isects, n_vis, max_tiles) of the last 8 calls
        self.hits = self.misses = 0
        self.pinned = torch.zeros(4, dtype=torch.int64).pin_memory()  # totals[3] + sequence word, written by the GPU
        self.words = self.pinned.numpy()  # same memory: what the host polls
        self.seq = 0
        self.zero_copy, self.copied, self.copy_done = True, None, None
        self.dev = dev

    def capacities(self, total_rows: int):
        if not self.hist:
            return None
        n_isects = max(h[0] for h in self.hist)
        n_vis = max(h[1] for h in self.hist)
        if n_isects == 0 or n_vis == 0:
            return None
        cap_vis = min(total_rows, n_vis + n_vis // 32 + 512)
        cap_isects = min(0x7FFFFFFF, n_isects + n_isects // 32 + 2048)
        return cap_vis, cap_isects, max(h[2] for h in self.hist)

    def observe(self, n_isects: int, n_vis: int, max_tiles: int):
        self.hist.append((n_isects, n_vis, max_tiles))
        del self.hist[:-8]

    def stage(self, totals: Tensor, st: int):
        """Queues, right behind the kernel that produced them, a one-warp kernel that stores the totals and then a
        sequence number into pinned host memory (no copy engine, no event)."""
        self.seq += 1
        self.copied = None
        if self.zero_copy:
            rc = lib().gsb200_publish_totals(ptr(totals), self.pinned.data_ptr(), self.seq, st)
            if rc == 0:
                return
            self.zero_copy = False  # pinned memory not device-mapped on this system: plain asynchronous copy from now on
        self.copied = torch.empty(3, dtype=torch.int64).pin_memory()
        self.copied.copy_(totals, non_blocking=True)
        self.copy_done = torch.cuda.Event()
        self.copy_done.record(torch.cuda.current_stream(self.dev))

    def read(self):
        """Polls the sequence word; the stores before it are ordered by the kernel's system-scope fence."""
        if self.copied is not None:
            self.copy_done.synchronize()
            return tuple(int(v) for v in self.copied.tolist())
        words, seq = self.words, self.seq
        spins = 0
        while int(words[3]) != seq:
            spins += 1
            if spins % 4_000_000 == 0:  # seconds without progress: surface a device-side failure instead of hanging
                torch.cuda.synchronize(self.dev)
                if int(words[3]) != seq:
                    raise RuntimeError("intersect_tile: the totals never arrived from the device")
        return int(words[0]), int(words[1]), int(words[2])


_predictors = {}


def _isect_predictor(dev: torch.device, I: int, tile_width: int, tile_height: int, packed: bool = False) -> _IsectPredictor:
    key = (dev.index, I, tile_width, tile_height, packed, stream(dev.index))
    p = _predictors.get(key)
    if p is None:
        p = _predictors[key] = _IsectPredictor(dev)
    return p


class SortedIntersections:
    """What the compositing needs from the tile intersection, from the narrow-key pipeline: ``tiles_per_gauss``,
    ``flatten_ids`` (sorted by (image, tile, depth)), ``isect_offsets`` [I, th, tw].  The reference's sorted int64
    ``isect_ids`` are rebuilt from the sorted tile ids and the depths only when asked for (``isect_ids()``)."""

    __slots__ = ("tiles_per_gauss", "flatten_ids", "isect_offsets", "_keys", "_key_bytes", "_depths", "_geom", "_ids")

    def __init__(self, tiles_per_gauss, flatten_ids, isect_offsets, keys, key_bytes, depths, geom):
        self.tiles_per_gauss, self.flatten_ids, self.isect_offsets = tiles_per_gauss, flatten_ids, isect_offsets
        self._keys, self._key_bytes, self._depths, self._geom, self._ids = keys, key_bytes, depths, geom, None

    def isect_ids(self) -> Tensor:
        if self._ids is None:
            I, tw, th = self._geom
            n = self.flatten_ids.shape[0]
            ids = torch.empty(n, device=self.flatten_ids.device, dtype=torch.int64)
            if n > 0:
                with _Ctx(ids.device) as st:
                    check(
                        lib().gsb200_isect_ids_from_tilekeys(
                            n, self._key_bytes, ptr(self._keys), ptr(self.flatten_ids), ptr(self._depths), I, tw, th, ptr(ids), st,
                        ),
                        "intersect_tile (ids)",
                    )
            self._ids = ids
        return self._ids


@torch.no_grad()
def isect_tiles_sorted(
    means2d: Tensor, radii: Tensor, depths: Tensor, tile_size: int, tile_width: int, tile_height: int,
    conics: Optional[Tensor] = None, opacities: Optional[Tensor] = None, precounted: Optional[RowSideOutputs] = None,
    n_images: Optional[int] = None, image_ids: Optional[Tensor] = None, _exact: bool = False,
    _tile_mask: Optional[Tensor] = None,
) -> SortedIntersections:
    """Sorted tile intersection + offsets, the reference's sorted ``isect_tiles`` + ``isect_offset_encode``
    (csrc/Intersect.cpp:203-326, 330-382), with the S-sized sort done on 2- or 4-byte dense tile ids instead of the
    8-byte (image | tile | depth) ids.  Rows are dense ([..., N, 2] means2d), or packed ([nnz, 2] means2d with
    ``n_images`` and the image of each row in ``image_ids``).  The stage is launched on capacities predicted from the
    earlier calls of the same shape.  ``_exact`` (isect_tiles) reads the totals first and sizes the stage exactly, and
    leaves that history alone: the call's own largest row then picks the emit kernel.  ``_tile_mask`` (isect_tiles_sparse,
    with ``_exact``): uint8 [I, th, tw]; only the tiles it sets are counted and listed."""
    dev = require_cuda(means2d, radii, depths)
    means2d, radii, depths, conics, opacities, image_ids, (image_dims, I, N, _, total, packed) = _isect_rows(
        means2d, radii, depths, conics, opacities, tile_width, tile_height, n_images, image_ids
    )
    L = lib()
    key_bits = _cabi.bits_for_count(I * tile_width * tile_height)
    key_bytes = 2 if key_bits <= 16 else 4
    key_dtype = torch.int16 if key_bytes == 2 else torch.int32  # raw storage; the kernels read them unsigned
    have_counts = (
        _tile_mask is None and not packed and precounted is not None and precounted.totals is not None and total > 0
        and (precounted.tile_size, precounted.tile_width, precounted.tile_height) == (tile_size, tile_width, tile_height)
        and precounted.tiles_per_gauss.numel() == total and conics is not None and opacities is not None
    )
    if have_counts:  # counted by the fused projection (same device function, same inputs)
        tiles_per_gauss = precounted.tiles_per_gauss.view(image_dims + (N,))
    else:
        tiles_per_gauss = torch.empty(image_dims + (N,), device=dev, dtype=torch.int32)
    offsets = torch.empty((I, tile_height, tile_width), device=dev, dtype=torch.int32)
    geom = (I, tile_width, tile_height)
    accu = conics is not None and opacities is not None

    def empty():
        offsets.zero_()
        return SortedIntersections(
            tiles_per_gauss.zero_(), torch.empty(0, device=dev, dtype=torch.int32), offsets,
            torch.empty(0, device=dev, dtype=key_dtype), key_bytes, depths, geom,
        )

    if total == 0:
        return empty()
    totals = precounted.totals if have_counts else torch.empty(3, device=dev, dtype=torch.int64)
    pred = None if _exact else _isect_predictor(dev, I, tile_width, tile_height, packed)
    with _Ctx(dev) as st:
        if not have_counts:
            check(
                L.gsb200_isect_count_totals(
                    I, N, ptr(means2d), ptr(radii), ptr(conics) if accu else None, ptr(opacities) if accu else None, ptr(image_ids),
                    ptr(_tile_mask), tile_size, tile_width, tile_height, ptr(tiles_per_gauss), ptr(totals), st,
                ),
                "intersect_tile (count)",
            )

        def run(cap_vis: int, cap_isects: int, max_tiles: int):
            # compaction, depth order, scan, emission, tile sort, offsets: one call, every launch sized by the capacities
            keys_out = torch.empty(cap_isects, device=dev, dtype=key_dtype)
            vals_out = torch.empty(cap_isects, device=dev, dtype=torch.int32)
            ws = _scratch_buffer(dev, "isect", L.gsb200_isect_sorted_workspace_bytes(I, total, cap_vis, cap_isects, key_bytes, tile_width, tile_height))
            check(
                L.gsb200_isect_sorted(
                    I, N, ptr(means2d), ptr(radii), ptr(depths), ptr(conics) if accu else None, ptr(opacities) if accu else None,
                    ptr(image_ids), ptr(_tile_mask), tile_size, tile_width, tile_height, ptr(tiles_per_gauss), ptr(totals), cap_vis, cap_isects,
                    max_tiles, key_bytes, ptr(keys_out), ptr(vals_out), ptr(offsets), ptr(ws), ws.numel(), st,
                ),
                "intersect_tile (sorted)",
            )
            return keys_out, vals_out

        caps = pred.capacities(total) if pred is not None else None
        if caps is not None:
            # Launch on PREDICTED capacities, then read the totals: the host read (the reference's one sync of the forward,
            # csrc/Intersect.cpp:259) overlaps the queued stage instead of idling the GPU.  A miss (a count above its
            # capacity) costs one exact re-run; nothing is ever written past a capacity.
            pred.stage(totals, st)
            keys_out, vals_out = run(*caps)
            n_isects, n_vis, max_tiles = pred.read()
            pred.observe(n_isects, n_vis, max_tiles)
            if n_isects == 0:
                return empty()
            if n_vis > caps[0] or n_isects > caps[1]:
                pred.misses += 1
                keys_out, vals_out = run(n_vis, n_isects, max_tiles)
            else:
                pred.hits += 1
                keys_out, vals_out = keys_out[:n_isects], vals_out[:n_isects]
        else:
            n_isects, n_vis, max_tiles = (int(v) for v in totals.tolist())  # exact sizes (first call of a shape)
            if pred is not None:
                pred.observe(n_isects, n_vis, max_tiles)
            if n_isects == 0:
                return empty()
            keys_out, vals_out = run(n_vis, n_isects, max_tiles)
    return SortedIntersections(tiles_per_gauss, vals_out, offsets, keys_out, key_bytes, depths, geom)


@torch.no_grad()
def isect_offset_encode(isect_ids: Tensor, n_images: int, tile_width: int, tile_height: int) -> Tensor:
    """Sorted intersection ids -> per-(image, tile) start offsets, int32 [n_images, tile_height, tile_width]."""
    dev = require_cuda(isect_ids)
    if isect_ids.dtype != torch.int64:
        raise TypeError("isect_ids must be int64")
    isect_ids = isect_ids.contiguous()
    offsets = torch.empty((n_images, tile_height, tile_width), device=dev, dtype=torch.int32)
    with _Ctx(dev) as st:
        check(
            lib().gsb200_isect_offsets(isect_ids.shape[0], ptr(isect_ids), n_images, tile_width, tile_height, ptr(offsets), st),
            "intersect_offset",
        )
    return offsets


# --------------------------------------------------------------------------------------------
# rasterize_to_pixels

_SUPPORTED_CHANNELS = (1, 2, 3, 4, 5, 8, 16, 32)


def _grad_record_width(D: int, absgrad: bool) -> int:
    return ((6 + D + (2 if absgrad else 0)) + 3) // 4 * 4


def _grad_records(row_dims: tuple, D: int, absgrad: bool, device) -> Tensor:
    """Zeroed gradient records of the compositing backward, one per Gaussian row (layout: gsb200_raster_bwd in
    include/gsplat_b200.h)."""
    return torch.zeros(tuple(row_dims) + (_grad_record_width(D, absgrad),), device=device, dtype=torch.float32)


def _split_grad_records(rec: Tensor, D: int, absgrad: bool):
    """Views (v_means2d, v_conics, v_colors, v_opacities, v_means2d_abs or None) into the records of _grad_records."""
    return rec[..., 0:2], rec[..., 2:5], rec[..., 6 : 6 + D], rec[..., 5], (rec[..., 6 + D : 8 + D] if absgrad else None)


def _composite_backward(ctx, render_alphas, v_render_colors, v_render_alphas, D, row_dims, run):
    """Both compositing backwards around their C call run(v_render_colors, v_render_alphas, absgrad, rec, stream).
    Returns the contiguous v_render_colors and the (v_means2d, v_conics, v_colors, v_opacities) gradients."""
    dev = render_alphas.device
    # set_materialize_grads(False): an output the loss does not use arrives as None instead of a zero-filled tensor
    # (render_alphas in a plain photometric loss: 8 MB of zeros per 1080p step); the kernel takes a null pointer for it
    if v_render_colors is None:
        v_render_colors = torch.zeros(render_alphas.shape[:-1] + (D,), device=dev, dtype=torch.float32)
    v_render_colors = v_render_colors.contiguous()
    v_render_alphas = v_render_alphas.contiguous() if v_render_alphas is not None else None
    absgrad = ctx.absgrad_holder is not None
    rec = _grad_records(row_dims, D, absgrad, dev)
    with _Ctx(dev) as st:
        run(v_render_colors, v_render_alphas, absgrad, rec, st)
    v_means2d, v_conics, v_colors, v_opacities, v_abs = _split_grad_records(rec, D, absgrad)
    if absgrad:
        ctx.absgrad_holder.copy_(v_abs)
    return v_render_colors, (v_means2d, v_conics, v_colors, v_opacities)


def _rasterize_padded(means2d, colors, backgrounds, tile_size, packed, absgrad, composite):
    """Shared by the compositing entry points: checks the arguments, pads colors / backgrounds with zero channels up to
    the next count the kernels are built for, runs composite(colors, backgrounds, absgrad_holder, padded), sets
    ``means2d.absgrad`` and cuts the padding off the rendered colours."""
    if packed != (means2d.dim() == 2):
        raise ValueError(f"packed={packed} but means2d has shape {tuple(means2d.shape)}")
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")
    D = colors.shape[-1]
    if D > 32:
        raise ValueError(
            f"Unsupported number of color channels: {D}. gsplat_b200 rasterizes up to 32 channels per pass "
            "(rasterization() chunks wider features with channel_chunk=32)."
        )
    pad = 0
    if D not in _SUPPORTED_CHANNELS:
        target = next(c for c in _SUPPORTED_CHANNELS if c >= D)
        pad = target - D
        colors = torch.nn.functional.pad(colors, (0, pad))
        if backgrounds is not None:
            backgrounds = torch.nn.functional.pad(backgrounds, (0, pad))
    holder = torch.zeros_like(means2d) if absgrad else None
    render_colors, render_alphas = composite(colors, backgrounds, holder, pad > 0)
    if absgrad:
        means2d.absgrad = holder
    if pad:
        render_colors = render_colors[..., :D]
    return render_colors, render_alphas


class _RasterizeToPixels(torch.autograd.Function):
    @staticmethod
    def forward(
        ctx, means2d, conics, colors, opacities, backgrounds, masks, width, height, tile_size, isect_offsets,
        flatten_ids, absgrad_holder, row_records=None,
    ):
        dev = require_cuda(means2d, conics, colors, opacities)
        means2d, conics, colors, opacities = f32c(means2d, "means2d"), f32c(conics, "conics"), f32c(colors, "colors"), f32c(opacities, "opacities")
        backgrounds = f32c(backgrounds, "backgrounds")
        # image dims come from the offsets; the gaussian rows may be dense [..., N, *] or packed [nnz, *]
        image_dims = tuple(isect_offsets.shape[:-2])
        row_dims = tuple(means2d.shape[:-1])
        I, R, D = _prod(image_dims), _prod(row_dims), colors.shape[-1]
        # N only feeds the C ABI's 32-bit offset guard (I * N * stride < 2^32).  Dense rows: R == I * N.  Packed rows
        # [nnz, *] are addressed flat: ceil(R / I) keeps I * N within I - 1 rows of the real row count R.
        N = (R + I - 1) // I if I > 0 else R
        th, tw = isect_offsets.shape[-2:]
        m8 = _mask_u8(masks)
        offsets = isect_offsets.contiguous()
        fl = flatten_ids.contiguous()
        if offsets.dtype != torch.int32 or fl.dtype != torch.int32:
            raise TypeError("isect_offsets and flatten_ids must be int32")
        S = fl.shape[0]
        L = lib()
        records = torch.empty(max(L.gsb200_raster_records_bytes(S, D, I * th * tw), 16), device=dev, dtype=torch.uint8)
        o = dict(device=dev, dtype=torch.float32)
        render_colors = torch.empty(image_dims + (height, width, D), **o)
        render_alphas = torch.empty(image_dims + (height, width, 1), **o)
        last_ids = torch.empty(image_dims + (height, width), device=dev, dtype=torch.int32)
        with _Ctx(dev) as st:
            if row_records is not None and D <= 4 and row_records.numel() == R * 16:
                check(
                    L.gsb200_raster_fwd_rows(
                        I, N, D, ptr(row_records), ptr(backgrounds), ptr(m8), width, height, tile_size, tw, th, ptr(offsets),
                        ptr(fl), S, ptr(records), ptr(render_colors), ptr(render_alphas), ptr(last_ids), st,
                    ),
                    "rasterize_to_pixels_3dgs (row records)",
                )
            else:
                check(
                    L.gsb200_raster_fwd(
                        I, N, D, ptr(means2d), ptr(conics), ptr(colors), ptr(opacities), ptr(backgrounds), ptr(m8), width,
                        height, tile_size, tw, th, ptr(offsets), ptr(fl), S, ptr(records), ptr(render_colors),
                        ptr(render_alphas), ptr(last_ids), st,
                    ),
                    "rasterize_to_pixels_3dgs",
                )
        ctx.save_for_backward(backgrounds, m8, offsets, fl, records, render_alphas, last_ids)
        ctx.set_materialize_grads(False)
        ctx.absgrad_holder = absgrad_holder  # filled in place by backward; deliberately not a saved tensor
        ctx.meta = (row_dims, I, N, D, width, height, tile_size, tw, th, S)
        return render_colors, render_alphas

    @staticmethod
    def backward(ctx, v_render_colors, v_render_alphas):
        backgrounds, m8, offsets, fl, records, render_alphas, last_ids = ctx.saved_tensors
        row_dims, I, N, D, width, height, tile_size, tw, th, S = ctx.meta
        def run(v_render_colors, v_render_alphas, absgrad, rec, st):
            check(
                lib().gsb200_raster_bwd(
                    I, N, D, ptr(backgrounds), ptr(m8), width, height, tile_size, tw, th, ptr(offsets), ptr(fl), S,
                    ptr(records), ptr(render_alphas), ptr(last_ids), ptr(v_render_colors), ptr(v_render_alphas), absgrad,
                    ptr(rec), st,
                ),
                "rasterize_to_pixels_3dgs_bwd",
            )
        v_render_colors, grads = _composite_backward(ctx, render_alphas, v_render_colors, v_render_alphas, D, row_dims, run)
        v_backgrounds = None
        if backgrounds is not None and ctx.needs_input_grad[4]:
            v_backgrounds = (v_render_colors * (1.0 - render_alphas)).sum(dim=(-3, -2))
        return grads + (v_backgrounds,) + (None,) * 8


def rasterize_to_pixels(
    means2d: Tensor,  # [..., N, 2]
    conics: Tensor,  # [..., N, 3]
    colors: Tensor,  # [..., N, channels]
    opacities: Tensor,  # [..., N]
    image_width: int,
    image_height: int,
    tile_size: int,
    isect_offsets: Tensor,  # [..., tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    backgrounds: Optional[Tensor] = None,  # [..., channels]
    masks: Optional[Tensor] = None,  # [..., tile_height, tile_width]
    packed: bool = False,
    absgrad: bool = False,
) -> Tuple[Tensor, Tensor]:
    """Front-to-back alpha compositing of depth-sorted Gaussians per 16x16 tile.
    Returns (render_colors [..., H, W, channels], render_alphas [..., H, W, 1]).  With ``absgrad`` the
    backward fills ``means2d.absgrad``."""
    return rasterize_to_pixels_rows(
        means2d, conics, colors, opacities, image_width, image_height, tile_size, isect_offsets, flatten_ids, backgrounds,
        masks, packed, absgrad, None,
    )


def rasterize_to_pixels_rows(
    means2d, conics, colors, opacities, image_width, image_height, tile_size, isect_offsets, flatten_ids, backgrounds=None,
    masks=None, packed=False, absgrad=False, _row_records: Optional[Tensor] = None,
) -> Tuple[Tensor, Tensor]:
    """rasterize_to_pixels with the optional ``RowSideOutputs.rows`` of the fused projection that produced the inputs
    (rasterization() passes them; the forward's pack pass then only gathers)."""

    def composite(colors, backgrounds, holder, padded):
        return _RasterizeToPixels.apply(
            means2d, conics, colors, opacities, backgrounds, masks, int(image_width), int(image_height), int(tile_size),
            isect_offsets, flatten_ids, holder, None if padded else _row_records,
        )

    return _rasterize_padded(means2d, colors, backgrounds, tile_size, packed, absgrad, composite)


# --------------------------------------------------------------------------------------------
# 2DGS (surfel splatting), dense rows: fully_fused_projection_2dgs / rasterize_to_pixels_2dgs
# (reference wrappers gsplat/cuda/_wrapper.py:2633, :2918 and their autograd hooks :2730-2806, :3004-3150)


def _check_shape(t: Tensor, shape: tuple, name: str) -> None:
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} must have shape {tuple(shape)}, got {tuple(t.shape)}")


class _FullyFusedProjection2DGS(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means, quats, scales, viewmats, Ks, width, height, near_plane, far_plane, radius_clip):
        dev = require_cuda(means, quats, scales, viewmats, Ks)
        means, quats, scales = f32c(means, "means"), f32c(quats, "quats"), f32c(scales, "scales")
        viewmats, Ks = f32c(viewmats, "viewmats"), f32c(Ks, "Ks")
        batch = tuple(means.shape[:-2])
        B, N, C = _prod(batch), means.shape[-2], viewmats.shape[-3]
        o = dict(device=dev, dtype=torch.float32)
        radii = torch.empty(batch + (C, N, 2), device=dev, dtype=torch.int32)
        means2d = torch.empty(batch + (C, N, 2), **o)
        depths = torch.empty(batch + (C, N), **o)
        ray_transforms = torch.empty(batch + (C, N, 3, 3), **o)
        normals = torch.empty(batch + (C, N, 3), **o)
        with _Ctx(dev) as st:
            check(
                lib().gsb200_surfel_projection_fwd(
                    B, C, N, ptr(means), ptr(quats), ptr(scales), ptr(viewmats), ptr(Ks), width, height, near_plane, far_plane,
                    radius_clip, ptr(radii), ptr(means2d), ptr(depths), ptr(ray_transforms), ptr(normals), st,
                ),
                "projection_2dgs_fused",
            )
        ctx.save_for_backward(means, quats, scales, viewmats, Ks, radii, ray_transforms)
        ctx.mark_non_differentiable(radii)
        return radii, means2d, depths, ray_transforms, normals

    @staticmethod
    def backward(ctx, v_radii, v_means2d, v_depths, v_ray_transforms, v_normals):
        means, quats, scales, viewmats, Ks, radii, ray_transforms = ctx.saved_tensors
        batch = tuple(means.shape[:-2])
        B, N, C = _prod(batch), means.shape[-2], viewmats.shape[-3]
        dev = means.device

        def grad(g, shape):
            return torch.zeros(batch + (C, N) + shape, device=dev, dtype=torch.float32) if g is None else g.float().contiguous()

        v_means2d, v_depths = grad(v_means2d, (2,)), grad(v_depths, ())
        v_ray_transforms, v_normals = grad(v_ray_transforms, (3, 3)), grad(v_normals, (3,))
        v_means, v_quats, v_scales = torch.empty_like(means), torch.empty_like(quats), torch.empty_like(scales)
        v_viewmats = torch.empty_like(viewmats) if ctx.needs_input_grad[3] else None
        with _Ctx(dev) as st:
            check(
                lib().gsb200_surfel_projection_bwd(
                    B, C, N, ptr(means), ptr(quats), ptr(scales), ptr(viewmats), ptr(Ks), ptr(radii), ptr(ray_transforms),
                    ptr(v_means2d), ptr(v_depths), ptr(v_ray_transforms), ptr(v_normals), ptr(v_means), ptr(v_quats),
                    ptr(v_scales), ptr(v_viewmats), st,
                ),
                "projection_2dgs_fused_bwd",
            )
        return (v_means, v_quats, v_scales, v_viewmats) + (None,) * 6


def fully_fused_projection_2dgs(
    means: Tensor,  # [..., N, 3]
    quats: Tensor,  # [..., N, 4]
    scales: Tensor,  # [..., N, 3]
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    width: int,
    height: int,
    eps2d: float = 0.3,
    near_plane: float = 0.01,
    far_plane: float = 1e10,
    radius_clip: float = 0.0,
    packed: bool = False,
    sparse_grad: bool = False,
) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """Projects 2D Gaussians (surfels).  Returns (radii int32 [..., C, N, 2], means2d [..., C, N, 2], depths [..., C, N],
    ray_transforms [..., C, N, 3, 3], normals [..., C, N, 3]).  ``radii == 0`` marks culled entries; their float outputs
    are zero.  ``eps2d`` is accepted and unused, as in the reference.  Only the dense layout is built: ``packed=True`` and
    ``sparse_grad=True`` raise NotImplementedError."""
    if packed or sparse_grad:
        raise NotImplementedError("fully_fused_projection_2dgs: only the dense layout (packed=False) is built")
    if means.dim() < 2 or means.shape[-1] != 3:
        raise ValueError(f"means must be [..., N, 3], got {tuple(means.shape)}")
    batch, N = tuple(means.shape[:-2]), means.shape[-2]
    _check_shape(quats, batch + (N, 4), "quats")
    _check_shape(scales, batch + (N, 3), "scales")
    if viewmats.dim() != len(batch) + 3:
        raise ValueError(f"viewmats must be [..., C, 4, 4], got {tuple(viewmats.shape)}")
    C = viewmats.shape[-3]
    _check_shape(viewmats, batch + (C, 4, 4), "viewmats")
    _check_shape(Ks, batch + (C, 3, 3), "Ks")
    return _FullyFusedProjection2DGS.apply(
        means, quats, scales, viewmats, Ks, int(width), int(height), float(near_plane), float(far_plane), float(radius_clip),
    )


class _RasterizeToPixels2DGS(torch.autograd.Function):
    @staticmethod
    def forward(
        ctx, means2d, ray_transforms, colors, opacities, normals, densify, backgrounds, masks, width, height, isect_offsets,
        flatten_ids, absgrad_holder,
    ):
        dev = require_cuda(means2d, ray_transforms, colors, opacities, normals)
        means2d, ray_transforms = f32c(means2d, "means2d"), f32c(ray_transforms, "ray_transforms")
        colors, opacities, normals = f32c(colors, "colors"), f32c(opacities, "opacities"), f32c(normals, "normals")
        backgrounds = f32c(backgrounds, "backgrounds")
        image_dims = tuple(isect_offsets.shape[:-2])
        I, N, D = _prod(image_dims), means2d.shape[-2], colors.shape[-1]
        th, tw = isect_offsets.shape[-2:]
        m8 = _mask_u8(masks)
        offsets, fl = isect_offsets.contiguous(), flatten_ids.contiguous()
        S = fl.shape[0]
        o = dict(device=dev, dtype=torch.float32)
        pix = image_dims + (height, width)
        if S == 0:
            # nothing intersects a tile: the background alone, no kernel launch
            if backgrounds is not None:
                render_colors = torch.broadcast_to(backgrounds[..., None, None, :], pix + (D,)).contiguous()
            else:
                render_colors = torch.zeros(pix + (D,), **o)
            render_alphas, render_distort, render_median = (torch.zeros(pix + (1,), **o) for _ in range(3))
            render_normals = torch.zeros(pix + (3,), **o)
            last_ids = median_ids = torch.zeros(pix, device=dev, dtype=torch.int32)
        else:
            render_colors = torch.empty(pix + (D,), **o)
            render_alphas, render_distort, render_median = (torch.empty(pix + (1,), **o) for _ in range(3))
            render_normals = torch.empty(pix + (3,), **o)
            last_ids = torch.empty(pix, device=dev, dtype=torch.int32)
            median_ids = torch.empty(pix, device=dev, dtype=torch.int32)
            with _Ctx(dev) as st:
                check(
                    lib().gsb200_surfel_raster_fwd(
                        I, N, D, ptr(means2d), ptr(ray_transforms), ptr(colors), ptr(opacities), ptr(normals), ptr(backgrounds),
                        ptr(m8), width, height, 16, tw, th, ptr(offsets), ptr(fl), S, ptr(render_colors), ptr(render_alphas),
                        ptr(render_normals), ptr(render_distort), ptr(render_median), ptr(last_ids), ptr(median_ids), st,
                    ),
                    "rasterize_to_pixels_2dgs",
                )
        ctx.save_for_backward(
            means2d, ray_transforms, colors, opacities, normals, backgrounds, m8, offsets, fl, render_colors, render_alphas,
            last_ids, median_ids,
        )
        ctx.set_materialize_grads(False)
        ctx.absgrad_holder = absgrad_holder  # filled in place by backward; deliberately not a saved tensor
        ctx.meta = (I, N, D, width, height, tw, th, S, tuple(densify.shape))
        return render_colors, render_alphas, render_normals, render_distort, render_median

    @staticmethod
    def backward(ctx, v_render_colors, v_render_alphas, v_render_normals, v_render_distort, v_render_median):
        (means2d, ray_transforms, colors, opacities, normals, backgrounds, m8, offsets, fl, render_colors, render_alphas,
         last_ids, median_ids) = ctx.saved_tensors
        I, N, D, width, height, tw, th, S, densify_shape = ctx.meta
        dev = render_alphas.device
        if v_render_colors is None:
            v_render_colors = torch.zeros_like(render_colors)
        v_render_colors = v_render_colors.contiguous()
        c = lambda g: None if g is None else g.contiguous()  # noqa: E731
        v_render_alphas, v_render_normals = c(v_render_alphas), c(v_render_normals)
        v_render_distort, v_render_median = c(v_render_distort), c(v_render_median)
        v_means2d, v_ray_transforms = torch.zeros_like(means2d), torch.zeros_like(ray_transforms)
        v_colors, v_opacities, v_normals = torch.zeros_like(colors), torch.zeros_like(opacities), torch.zeros_like(normals)
        v_densify = torch.zeros(densify_shape, device=dev, dtype=torch.float32)
        holder = ctx.absgrad_holder
        v_abs = torch.zeros_like(means2d) if holder is not None else None
        if S > 0:
            with _Ctx(dev) as st:
                check(
                    lib().gsb200_surfel_raster_bwd(
                        I, N, D, ptr(means2d), ptr(ray_transforms), ptr(colors), ptr(opacities), ptr(normals), ptr(backgrounds),
                        ptr(m8), width, height, 16, tw, th, ptr(offsets), ptr(fl), S, ptr(render_colors), ptr(render_alphas),
                        ptr(last_ids), ptr(median_ids), ptr(v_render_colors), ptr(v_render_alphas), ptr(v_render_normals),
                        ptr(v_render_distort), ptr(v_render_median), ptr(v_means2d), ptr(v_ray_transforms), ptr(v_colors),
                        ptr(v_opacities), ptr(v_normals), ptr(v_densify), ptr(v_abs), st,
                    ),
                    "rasterize_to_pixels_2dgs_bwd",
                )
        if holder is not None:
            holder.copy_(v_abs)
        v_backgrounds = None
        if backgrounds is not None and ctx.needs_input_grad[6]:
            v_backgrounds = (v_render_colors * (1.0 - render_alphas)).sum(dim=(-3, -2))
        return (v_means2d, v_ray_transforms, v_colors, v_opacities, v_normals, v_densify, v_backgrounds) + (None,) * 6


def rasterize_to_pixels_2dgs(
    means2d: Tensor,  # [..., N, 2]
    ray_transforms: Tensor,  # [..., N, 3, 3]
    colors: Tensor,  # [..., N, channels]
    opacities: Tensor,  # [..., N]
    normals: Tensor,  # [..., N, 3]
    densify: Tensor,  # [..., N, 2]
    image_width: int,
    image_height: int,
    tile_size: int,
    isect_offsets: Tensor,  # [..., tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    backgrounds: Optional[Tensor] = None,  # [..., channels]
    masks: Optional[Tensor] = None,  # [..., tile_height, tile_width]
    packed: bool = False,
    absgrad: bool = False,
    distloss: bool = False,
) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """Front-to-back compositing of depth-sorted surfels per 16x16 tile.  Returns (render_colors [..., H, W, channels],
    render_alphas [..., H, W, 1], render_normals [..., H, W, 3], render_distort [..., H, W, 1], render_median
    [..., H, W, 1]).  The last colour channel is the depth that the distortion and the median depth are taken from; the
    distortion is always computed (``distloss`` only matters to the caller that appends the depth channel, as in the
    reference).  ``densify`` receives the densification gradient; with ``absgrad`` the backward fills ``means2d.absgrad``."""
    if packed:
        raise NotImplementedError("rasterize_to_pixels_2dgs: only the dense layout (packed=False) is built")
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")
    if isect_offsets.dim() < 2:
        raise ValueError(f"isect_offsets must be [..., tile_height, tile_width], got {tuple(isect_offsets.shape)}")
    image_dims, (th, tw) = tuple(isect_offsets.shape[:-2]), tuple(isect_offsets.shape[-2:])
    if th * 16 < image_height or tw * 16 < image_width:
        raise ValueError(f"isect_offsets tile grid {tw}x{th} does not cover a {image_width}x{image_height} image")
    if means2d.dim() < 2 or tuple(means2d.shape[:-2]) != image_dims or means2d.shape[-1] != 2:
        raise ValueError(f"means2d must be {image_dims + ('N', 2)}, got {tuple(means2d.shape)}")
    N = means2d.shape[-2]
    if colors.dim() != means2d.dim():
        raise ValueError(f"colors must be [..., N, channels], got {tuple(colors.shape)}")
    D = colors.shape[-1]
    _check_shape(ray_transforms, image_dims + (N, 3, 3), "ray_transforms")
    _check_shape(colors, image_dims + (N, D), "colors")
    _check_shape(opacities, image_dims + (N,), "opacities")
    _check_shape(normals, image_dims + (N, 3), "normals")
    _check_shape(densify, image_dims + (N, 2), "densify")
    if backgrounds is not None:
        _check_shape(backgrounds, image_dims + (D,), "backgrounds")
    if masks is not None:
        _check_shape(masks, image_dims + (th, tw), "masks")
    if isect_offsets.dtype != torch.int32 or flatten_ids.dtype != torch.int32 or flatten_ids.dim() != 1:
        raise ValueError("isect_offsets and flatten_ids must be int32, flatten_ids one-dimensional")
    if D not in _SUPPORTED_CHANNELS:
        raise NotImplementedError(
            f"rasterize_to_pixels_2dgs: {D} channels; the 2DGS kernels are built for {_SUPPORTED_CHANNELS} (the last channel "
            "is the depth, so the channels cannot be padded)"
        )
    holder = torch.zeros_like(means2d) if absgrad else None
    outs = _RasterizeToPixels2DGS.apply(
        means2d, ray_transforms, colors, opacities, normals, densify, backgrounds, masks, int(image_width), int(image_height),
        isect_offsets, flatten_ids, holder,
    )
    if absgrad:
        means2d.absgrad = holder
    return outs


# --------------------------------------------------------------------------------------------
# rasterize_to_indices_in_range / rasterize_to_indices_in_range_2dgs (reference wrappers gsplat/cuda/_wrapper.py:2486,
# :3154): the pairs the compositing forward of this library composites, for iterative rasterization and picking.

_RANGE_MAX = 1 << 62  # any range end past the last batch means "to the end"


def _batch_index(v, name: str) -> int:
    """A batch index: an integer, or an integral float such as the reference docs' 1e10; negative is a ValueError."""
    if isinstance(v, float):
        if not math.isfinite(v) or not v.is_integer():
            raise ValueError(f"{name} must be a whole number of batches, got {v!r}")
        v = int(v)
    else:
        try:
            v = operator.index(v)
        except TypeError:
            raise TypeError(f"{name} must be an integer, got {type(v).__name__}") from None
    if v < 0:
        raise ValueError(f"{name} must be >= 0, got {v}")
    return min(v, _RANGE_MAX)


def _indices_in_range(
    what, entry, range_start, range_end, transmittances, means2d, rows, rows_tail, rows_name, opacities, image_width,
    image_height, tile_size, isect_offsets, flatten_ids,
):
    rs, re_ = _batch_index(range_start, "range_start"), _batch_index(range_end, "range_end")
    W, H = int(image_width), int(image_height)
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")
    if means2d.dim() < 2 or means2d.shape[-1] != 2:
        raise ValueError(f"means2d must be [..., N, 2], got {tuple(means2d.shape)}")
    image_dims, N = tuple(means2d.shape[:-2]), means2d.shape[-2]
    _check_shape(rows, image_dims + (N,) + rows_tail, rows_name)
    _check_shape(opacities, image_dims + (N,), "opacities")
    _check_shape(transmittances, image_dims + (H, W), "transmittances")
    if isect_offsets.dim() != means2d.dim() or tuple(isect_offsets.shape[:-2]) != image_dims:
        raise ValueError(f"isect_offsets must be {image_dims + ('tile_height', 'tile_width')}, got {tuple(isect_offsets.shape)}")
    th, tw = isect_offsets.shape[-2:]
    if th * 16 < H or tw * 16 < W:
        raise ValueError(f"isect_offsets tile grid {tw}x{th} does not cover a {W}x{H} image")
    if flatten_ids.dim() != 1:
        raise ValueError(f"flatten_ids must be one-dimensional, got {tuple(flatten_ids.shape)}")
    if isect_offsets.dtype != torch.int32 or flatten_ids.dtype != torch.int32:
        raise TypeError("isect_offsets and flatten_ids must be int32")
    for t, name in ((transmittances, "transmittances"), (means2d, "means2d"), (rows, rows_name), (opacities, "opacities")):
        if t.dtype != torch.float32:
            raise TypeError(f"{name}: expected float32, got {t.dtype} (gsplat_b200 computes in fp32 only)")
    dev = require_cuda(transmittances, means2d, rows, opacities, isect_offsets, flatten_ids)
    I, S = _prod(image_dims), flatten_ids.shape[0]
    P = I * H * W
    if N == 0 or S == 0 or P == 0 or re_ <= rs:
        return tuple(torch.empty(0, device=dev, dtype=torch.int64) for _ in range(3))
    tr, m2, rw, op = (t.contiguous() for t in (transmittances, means2d, rows, opacities))
    off, fl = isect_offsets.contiguous(), flatten_ids.contiguous()
    args = (I, N, ptr(m2), ptr(rw), ptr(op), ptr(tr), W, H, 16, tw, th, ptr(off), ptr(fl), S, rs, re_)
    return _index_passes(what, entry, args, P, dev)


def _index_passes(what, entry, args, P, dev):
    """The count and emit passes of a pair-query entry over P pixels: ``args`` are its arguments before ``emit`` (the
    tensors they point into are kept alive by the caller)."""
    L = lib()
    ws = torch.empty(L.gsb200_indices_workspace_bytes(P), device=dev, dtype=torch.uint8)
    total = torch.empty(1, device=dev, dtype=torch.int64)
    fn = getattr(L, entry)
    with _Ctx(dev) as st:

        def run(emit, outs):
            check(fn(*args, emit, ptr(ws), ws.numel(), ptr(total), *(ptr(o) for o in outs), st), what)

        run(0, (None, None, None))
        M = int(total.item())  # the host sync between the two passes (reference: csrc/Rasterization.cpp:1050)
        outs = tuple(torch.empty(M, device=dev, dtype=torch.int64) for _ in range(3))
        if M > 0:
            run(1, outs)
    return outs


@torch.no_grad()
def rasterize_to_indices_in_range(
    range_start: int,
    range_end: int,
    transmittances: Tensor,  # [..., image_height, image_width]
    means2d: Tensor,  # [..., N, 2]
    conics: Tensor,  # [..., N, 3]
    opacities: Tensor,  # [..., N]
    image_width: int,
    image_height: int,
    tile_size: int,
    isect_offsets: Tensor,  # [..., tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
) -> Tuple[Tensor, Tensor, Tensor]:
    """The (gaussian, pixel) pairs ``rasterize_to_pixels`` composites when every pixel starts from its transmittance
    and walks only the batches ``[range_start, range_end)`` of ``tile_size**2`` gaussians of its tile's depth-sorted list
    (``range_end`` past the last batch, e.g. 1e10, means "to the end").  A gaussian that would bring the transmittance
    to 1e-4 or below stops the pixel and is not returned.  The decisions are the compositing kernel's own.

    Returns int64 ``(gaussian_ids, pixel_ids, image_ids)`` [M]: ``gaussian_ids`` in [0, N), ``pixel_ids`` row-major
    within the image, ``image_ids`` the flattened image index; ordered by (image, row, col), front to back per pixel."""
    return _indices_in_range(
        "rasterize_to_indices_3dgs", "gsb200_raster_indices", range_start, range_end, transmittances, means2d, conics, (3,),
        "conics", opacities, image_width, image_height, tile_size, isect_offsets, flatten_ids,
    )


@torch.no_grad()
def rasterize_to_indices_in_range_2dgs(
    range_start: int,
    range_end: int,
    transmittances: Tensor,  # [..., image_height, image_width]
    means2d: Tensor,  # [..., N, 2]
    ray_transforms: Tensor,  # [..., N, 3, 3]
    opacities: Tensor,  # [..., N]
    image_width: int,
    image_height: int,
    tile_size: int,
    isect_offsets: Tensor,  # [..., tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
) -> Tuple[Tensor, Tensor, Tensor]:
    """``rasterize_to_indices_in_range`` for surfels: the pairs ``rasterize_to_pixels_2dgs`` composites, with the same
    ranges, outputs and order."""
    return _indices_in_range(
        "rasterize_to_indices_2dgs", "gsb200_surfel_indices", range_start, range_end, transmittances, means2d,
        ray_transforms, (3, 3), "ray_transforms", opacities, image_width, image_height, tile_size, isect_offsets, flatten_ids,
    )


# --------------------------------------------------------------------------------------------
# sparse pixels: build_sparse_tile_layout / isect_tiles_sparse / rasterize_to_pixels_sparse
# (reference wrappers /root/reference/gsplat/cuda/_wrapper.py:1352, :1433, :1566).  At every requested pixel the result
# is the dense rendering's; only the active tiles are intersected and composited, and only the requested pixels written.

_TILE_WORDS = 4  # uint64 words of a 16 x 16 tile's pixel mask


@torch.no_grad()
def build_sparse_tile_layout(
    pixels: Tensor,  # [P, 2] int, (row, col)
    image_ids: Tensor,  # [P] int
    n_images: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """Tile / pixel bookkeeping of a set of requested pixels ``pixels[p] = (row, col)`` of image ``image_ids[p]``.
    Returns (active_tiles int32 [AT] ascending dense tile ids ``image * th * tw + (row // 16) * tw + col // 16``,
    active_tile_mask bool [n_images, th, tw], tile_pixel_mask uint64 [AT, 4] raster-order in-tile bits,
    tile_pixel_cumsum int64 [AT] inclusive (length 1, zero, when P == 0), pixel_map int64 [P]: the pixel indices in
    (tile, in-tile) order).  Pixels must not repeat.  Reads the number of active tiles back to the host once."""
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")
    if pixels.dim() != 2 or pixels.shape[1] != 2:
        raise ValueError(f"pixels must be [P, 2], got {tuple(pixels.shape)}")
    P = pixels.shape[0]
    if tuple(image_ids.shape) != (P,):
        raise ValueError(f"image_ids must be [{P}], got {tuple(image_ids.shape)}")
    if pixels.is_floating_point() or image_ids.is_floating_point():
        raise TypeError("pixels and image_ids must be integer tensors")
    n_images, tile_width, tile_height = int(n_images), int(tile_width), int(tile_height)
    if n_images < 0 or tile_width <= 0 or tile_height <= 0:
        raise ValueError(f"bad layout n_images={n_images} tile_width={tile_width} tile_height={tile_height}")
    if n_images * tile_width * tile_height >= 1 << 31:
        raise ValueError(f"build_sparse_tile_layout: n_images * n_tiles ({n_images * tile_width * tile_height}) must be < 2^31.")
    if P > 0:
        # range checks on whatever device the inputs live on, before anything is launched here
        rows, cols = pixels[:, 0], pixels[:, 1]
        bad_px = (rows < 0) | (rows >= tile_height * tile_size) | (cols < 0) | (cols >= tile_width * tile_size)
        bad_id = (image_ids < 0) | (image_ids >= n_images)
        n_bad_px, n_bad_id = (int(v) for v in torch.stack([bad_px.sum(), bad_id.sum()]).tolist())
        if n_bad_px:
            raise ValueError(
                f"build_sparse_tile_layout: {n_bad_px} pixel(s) outside the {tile_height * tile_size} x {tile_width * tile_size} "
                "tile grid (pixels are (row, col))"
            )
        if n_bad_id:
            raise ValueError(f"build_sparse_tile_layout: {n_bad_id} image id(s) outside [0, {n_images})")
    dev = require_cuda(pixels, image_ids)
    i32 = dict(device=dev, dtype=torch.int32)
    i64 = dict(device=dev, dtype=torch.int64)
    mask8 = torch.empty((n_images, tile_height, tile_width), device=dev, dtype=torch.uint8)
    L = lib()
    with _Ctx(dev) as st:
        if P == 0:
            check(L.gsb200_sparse_layout_finish(0, n_images, tile_width, tile_height, 0, None, 0, None, ptr(mask8), None, None, None, st), "build_sparse_tile_layout")
            return (
                torch.empty(0, **i32), mask8.view(torch.bool), torch.empty((0, _TILE_WORDS), **i64).view(torch.uint64),
                torch.zeros(1, **i64), torch.empty(0, **i64),
            )
        px = pixels.to(torch.int32).contiguous()
        ids = image_ids.to(torch.int32).contiguous()
        ws = _scratch_buffer(dev, "sparse_layout", L.gsb200_sparse_layout_workspace_bytes(P, n_images, tile_width, tile_height))
        n_active = torch.empty(1, **i64)
        check(
            L.gsb200_sparse_layout_sort(P, ptr(px), ptr(ids), n_images, tile_size, tile_width, tile_height, ptr(ws), ws.numel(), ptr(n_active), st),
            "build_sparse_tile_layout (sort)",
        )
        AT = int(n_active.item())  # the one host sync of the layout (the reference's builder synchronises too)
        active_tiles = torch.empty(AT, **i32)
        tile_pixel_mask = torch.empty((AT, _TILE_WORDS), **i64)
        cumsum, pixel_map = torch.empty(AT, **i64), torch.empty(P, **i64)
        check(
            L.gsb200_sparse_layout_finish(
                P, n_images, tile_width, tile_height, AT, ptr(ws), ws.numel(), ptr(active_tiles), ptr(mask8), ptr(tile_pixel_mask),
                ptr(cumsum), ptr(pixel_map), st,
            ),
            "build_sparse_tile_layout (finish)",
        )
    return active_tiles, mask8.view(torch.bool), tile_pixel_mask.view(torch.uint64), cumsum, pixel_map


@torch.no_grad()
def isect_tiles_sparse(
    means2d: Tensor,  # [I, N, 2] or [nnz, 2]
    radii: Tensor,  # [I, N, 2] or [nnz, 2]
    depths: Tensor,  # [I, N] or [nnz]
    tile_mask: Tensor,  # [n_images, tile_height, tile_width] bool
    active_tiles: Tensor,  # [AT] int32
    n_images: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
    image_ids: Optional[Tensor] = None,  # [nnz], packed only
) -> Tuple[Tensor, Tensor]:
    """The intersections of ``isect_tiles(..., conics=None)`` that fall in tiles flagged by ``tile_mask`` (the
    ``active_tile_mask`` of build_sparse_tile_layout), in the same (image, tile, depth) order, with per-active-tile
    offsets.  Returns (tile_offsets int32 [AT + 1], ``tile_offsets[AT] == n_isects``; flatten_ids int32 [n_isects])."""
    packed = means2d.dim() == 2
    n_images = int(n_images)
    if packed:
        nnz = means2d.shape[0]
        if tuple(means2d.shape) != (nnz, 2) or tuple(radii.shape) != (nnz, 2) or tuple(depths.shape) != (nnz,):
            raise ValueError(f"packed inputs must be means2d [nnz, 2], radii [nnz, 2], depths [nnz]; got "
                             f"{tuple(means2d.shape)}, {tuple(radii.shape)}, {tuple(depths.shape)}")
        if image_ids is None or tuple(image_ids.shape) != (nnz,):
            raise ValueError("image_ids [nnz] is required when means2d is packed ([nnz, 2]).")
        I, N = n_images, nnz
    else:
        if means2d.dim() != 3:
            raise ValueError(f"means2d must be [I, N, 2] or [nnz, 2], got {tuple(means2d.shape)}")
        I, N = means2d.shape[0], means2d.shape[1]
        if tuple(means2d.shape) != (I, N, 2) or tuple(radii.shape) != (I, N, 2) or tuple(depths.shape) != (I, N):
            raise ValueError(f"dense inputs must be means2d [I, N, 2], radii [I, N, 2], depths [I, N]; got "
                             f"{tuple(means2d.shape)}, {tuple(radii.shape)}, {tuple(depths.shape)}")
        if I != n_images:
            raise ValueError(f"means2d has {I} images, n_images is {n_images}")
    if tuple(tile_mask.shape) != (n_images, tile_height, tile_width) or tile_mask.dtype != torch.bool:
        raise ValueError(f"tile_mask must be bool [{n_images}, {tile_height}, {tile_width}], got {tile_mask.dtype} {tuple(tile_mask.shape)}")
    if active_tiles.dim() != 1 or active_tiles.dtype != torch.int32:
        raise ValueError(f"active_tiles must be int32 [AT], got {active_tiles.dtype} {tuple(active_tiles.shape)}")
    if radii.dtype != torch.int32:
        raise TypeError("radii must be int32")
    image_bits, tile_bits = _cabi.bits_for_count(n_images), _cabi.bits_for_count(tile_width * tile_height)
    if image_bits + tile_bits > 32:
        raise RuntimeError(
            f"intersect_tile: (image, tile) id packing needs {image_bits + tile_bits} bits but only 32 are "
            f"available (I={n_images}, n_tiles={tile_width * tile_height})."
        )
    dev = require_cuda(means2d, radii, depths, tile_mask, active_tiles, image_ids)
    active = active_tiles.contiguous()
    AT = active.shape[0]
    # without rows the sorted stage lists nothing, and every tile offset is 0
    hits = isect_tiles_sorted(
        means2d, radii, depths, tile_size, tile_width, tile_height, n_images=n_images if packed else None,
        image_ids=image_ids if packed else None, _exact=True, _tile_mask=tile_mask.contiguous().view(torch.uint8),
    )
    tile_offsets = torch.empty(AT + 1, device=dev, dtype=torch.int32)
    with _Ctx(dev) as st:
        check(
            lib().gsb200_isect_active_offsets(
                AT, ptr(active), n_images, tile_width, tile_height, ptr(hits.isect_offsets), hits.flatten_ids.shape[0],
                ptr(tile_offsets), st,
            ),
            "intersect_tile_sparse (offsets)",
        )
    return tile_offsets, hits.flatten_ids


def _check_sparse_layout(image_ids, active_tiles, tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map,
                         image_width, image_height, tile_width, tile_height) -> Tuple[int, int]:
    """The layout checks of the sparse compositing ops, before anything is launched.  Returns (AT, P)."""
    AT, P = active_tiles.shape[0] if active_tiles.dim() == 1 else -1, pixel_map.shape[0] if pixel_map.dim() == 1 else -1
    if AT < 0 or P < 0 or active_tiles.dtype != torch.int32:
        raise ValueError("active_tiles must be int32 [AT] and pixel_map [P]")
    if tuple(tile_offsets.shape) != (AT + 1,) or tile_offsets.dtype != torch.int32 or flatten_ids.dtype != torch.int32:
        raise ValueError(f"tile_offsets must be int32 [{AT + 1}] and flatten_ids int32 (isect_tiles_sparse)")
    if tuple(tile_pixel_mask.shape) != (AT, _TILE_WORDS) or tile_pixel_mask.element_size() != 8:
        raise ValueError(f"tile_pixel_mask must be 64-bit [{AT}, {_TILE_WORDS}], got {tile_pixel_mask.dtype} {tuple(tile_pixel_mask.shape)}")
    n_cum = tile_pixel_cumsum.shape[0] if tile_pixel_cumsum.dim() == 1 else -1
    if n_cum not in ((AT,) if AT > 0 else (0, 1)) or tile_pixel_cumsum.dtype != torch.int64 or pixel_map.dtype != torch.int64:
        raise ValueError("tile_pixel_cumsum must be int64 [AT] and pixel_map int64 [P] (build_sparse_tile_layout)")
    if tuple(image_ids.shape) != (P,):
        raise ValueError(f"image_ids must be [{P}], got {tuple(image_ids.shape)}")
    if tile_width * 16 < image_width or tile_height * 16 < image_height:
        raise ValueError(f"a {tile_width} x {tile_height} tile grid does not cover {image_width} x {image_height} pixels")
    return AT, P


class _RasterizeToPixelsSparse(torch.autograd.Function):
    @staticmethod
    def forward(
        ctx, means2d, conics, colors, opacities, backgrounds, masks, image_ids, active_tiles, tile_offsets, flatten_ids,
        tile_pixel_mask, tile_pixel_cumsum, pixel_map, width, height, tile_width, tile_height, absgrad_holder,
    ):
        dev = require_cuda(means2d, conics, colors, opacities, active_tiles, tile_offsets, flatten_ids, pixel_map)
        means2d, conics, colors, opacities = f32c(means2d, "means2d"), f32c(conics, "conics"), f32c(colors, "colors"), f32c(opacities, "opacities")
        backgrounds = f32c(backgrounds, "backgrounds")
        row_dims = tuple(means2d.shape[:-1])
        R, D, P = _prod(row_dims), colors.shape[-1], pixel_map.shape[0]
        m8 = _mask_u8(masks)
        active, offsets, fl = active_tiles.contiguous(), tile_offsets.contiguous(), flatten_ids.contiguous()
        words = tile_pixel_mask.contiguous()
        cumsum, pmap = tile_pixel_cumsum.contiguous(), pixel_map.contiguous()
        AT, S = active.shape[0], fl.shape[0]
        L = lib()
        records = torch.empty(max(L.gsb200_raster_records_bytes(S, D, AT), 16), device=dev, dtype=torch.uint8)
        o = dict(device=dev, dtype=torch.float32)
        render_colors, render_alphas = torch.empty((P, D), **o), torch.empty((P, 1), **o)
        last_ids = torch.empty(P, device=dev, dtype=torch.int32)
        with _Ctx(dev) as st:
            check(
                L.gsb200_raster_sparse_fwd(
                    D, ptr(means2d), ptr(conics), ptr(colors), ptr(opacities), ptr(backgrounds), ptr(m8), width, height, 16,
                    tile_width, tile_height, AT, ptr(active), ptr(offsets), ptr(fl), S, ptr(words), ptr(cumsum), ptr(pmap),
                    ptr(records), ptr(render_colors), ptr(render_alphas), ptr(last_ids), st,
                ),
                "rasterize_to_pixels_sparse",
            )
        ctx.save_for_backward(backgrounds, m8, image_ids, active, offsets, fl, words, cumsum, pmap, records, render_alphas, last_ids)
        ctx.set_materialize_grads(False)
        ctx.absgrad_holder = absgrad_holder  # filled in place by backward; deliberately not a saved tensor
        ctx.meta = (row_dims, R, D, width, height, tile_width, tile_height)
        return render_colors, render_alphas

    @staticmethod
    def backward(ctx, v_render_colors, v_render_alphas):
        backgrounds, m8, image_ids, active, offsets, fl, words, cumsum, pmap, records, render_alphas, last_ids = ctx.saved_tensors
        row_dims, R, D, width, height, tw, th = ctx.meta
        def run(v_render_colors, v_render_alphas, absgrad, rec, st):
            check(
                lib().gsb200_raster_sparse_bwd(
                    R, D, ptr(backgrounds), ptr(m8), width, height, 16, tw, th, active.shape[0], ptr(active), ptr(offsets), ptr(fl),
                    fl.shape[0], ptr(words), ptr(cumsum), ptr(pmap), ptr(records), ptr(render_alphas), ptr(last_ids),
                    ptr(v_render_colors), ptr(v_render_alphas), absgrad, ptr(rec), st,
                ),
                "rasterize_to_pixels_sparse_bwd",
            )
        v_render_colors, grads = _composite_backward(ctx, render_alphas, v_render_colors, v_render_alphas, D, row_dims, run)
        v_backgrounds = None
        if backgrounds is not None and ctx.needs_input_grad[4]:
            v_backgrounds = torch.zeros_like(backgrounds).index_add_(0, image_ids.long(), v_render_colors * (1.0 - render_alphas))
        return grads + (v_backgrounds,) + (None,) * 13


def rasterize_to_pixels_sparse(
    means2d: Tensor,  # [..., N, 2] or [nnz, 2]
    conics: Tensor,  # [..., N, 3] or [nnz, 3]
    colors: Tensor,  # [..., N, channels] or [nnz, channels]
    opacities: Tensor,  # [..., N] or [nnz]
    image_ids: Tensor,  # [P]
    active_tiles: Tensor,  # [AT]
    tile_offsets: Tensor,  # [AT + 1]
    flatten_ids: Tensor,  # [n_isects]
    tile_pixel_mask: Tensor,  # [AT, 4]
    tile_pixel_cumsum: Tensor,  # [AT]
    pixel_map: Tensor,  # [P]
    image_width: int,
    image_height: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
    backgrounds: Optional[Tensor] = None,  # [n_images, channels]
    masks: Optional[Tensor] = None,  # [n_images, tile_height, tile_width]
    packed: bool = False,
    absgrad: bool = False,
) -> Tuple[Tensor, Tensor]:
    """rasterize_to_pixels at the pixels of a build_sparse_tile_layout layout only, with the lists of
    isect_tiles_sparse.  Returns (render_colors [P, channels], render_alphas [P, 1]) in the original pixel order; each
    value is the dense rendering's at that pixel (requested pixels in the margin of a partial tile included).  With
    ``absgrad`` the backward fills ``means2d.absgrad``."""
    _check_sparse_layout(
        image_ids, active_tiles, tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map, image_width,
        image_height, tile_width, tile_height,
    )

    def composite(colors, backgrounds, holder, padded):
        return _RasterizeToPixelsSparse.apply(
            means2d, conics, colors, opacities, backgrounds, masks, image_ids, active_tiles, tile_offsets, flatten_ids,
            tile_pixel_mask, tile_pixel_cumsum, pixel_map, int(image_width), int(image_height), int(tile_width),
            int(tile_height), holder,
        )

    return _rasterize_padded(means2d, colors, backgrounds, tile_size, packed, absgrad, composite)


class _RasterizeToPixels2DGSSparse(torch.autograd.Function):
    @staticmethod
    def forward(
        ctx, means2d, ray_transforms, colors, opacities, normals, densify, backgrounds, masks, image_ids, active_tiles,
        tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map, width, height, tile_width, tile_height,
        absgrad_holder,
    ):
        dev = require_cuda(means2d, ray_transforms, colors, opacities, normals, active_tiles, tile_offsets, flatten_ids, pixel_map)
        means2d, ray_transforms = f32c(means2d, "means2d"), f32c(ray_transforms, "ray_transforms")
        colors, opacities, normals = f32c(colors, "colors"), f32c(opacities, "opacities"), f32c(normals, "normals")
        backgrounds = f32c(backgrounds, "backgrounds")
        R, D, P = _prod(means2d.shape[:-1]), colors.shape[-1], pixel_map.shape[0]
        m8 = _mask_u8(masks)
        active, offsets, fl = active_tiles.contiguous(), tile_offsets.contiguous(), flatten_ids.contiguous()
        words, cumsum, pmap = tile_pixel_mask.contiguous(), tile_pixel_cumsum.contiguous(), pixel_map.contiguous()
        AT, S = active.shape[0], fl.shape[0]
        o = dict(device=dev, dtype=torch.float32)
        if P == 0 or S == 0:
            # no requested pixel, or nothing listed in any active tile: the background alone, no kernel launch
            if backgrounds is not None and P > 0:
                render_colors = backgrounds[image_ids.long()]
            else:
                render_colors = torch.zeros((P, D), **o)
            render_alphas, render_distort, render_median = (torch.zeros((P, 1), **o) for _ in range(3))
            render_normals = torch.zeros((P, 3), **o)
            last_ids = median_ids = torch.zeros(P, device=dev, dtype=torch.int32)
        else:
            render_colors = torch.empty((P, D), **o)
            render_alphas, render_distort, render_median = (torch.empty((P, 1), **o) for _ in range(3))
            render_normals = torch.empty((P, 3), **o)
            last_ids = torch.empty(P, device=dev, dtype=torch.int32)
            median_ids = torch.empty(P, device=dev, dtype=torch.int32)
            with _Ctx(dev) as st:
                check(
                    lib().gsb200_surfel_raster_sparse_fwd(
                        R, D, ptr(means2d), ptr(ray_transforms), ptr(colors), ptr(opacities), ptr(normals), ptr(backgrounds),
                        ptr(m8), width, height, 16, tile_width, tile_height, AT, ptr(active), ptr(offsets), ptr(fl), S,
                        ptr(words), ptr(cumsum), ptr(pmap), ptr(render_colors), ptr(render_alphas), ptr(render_normals),
                        ptr(render_distort), ptr(render_median), ptr(last_ids), ptr(median_ids), st,
                    ),
                    "rasterize_to_pixels_2dgs_sparse",
                )
        ctx.save_for_backward(
            means2d, ray_transforms, colors, opacities, normals, backgrounds, m8, image_ids, active, offsets, fl, words, cumsum,
            pmap, render_colors, render_alphas, last_ids, median_ids,
        )
        ctx.set_materialize_grads(False)
        ctx.absgrad_holder = absgrad_holder  # filled in place by backward; deliberately not a saved tensor
        ctx.meta = (R, D, width, height, tile_width, tile_height, tuple(densify.shape))
        return render_colors, render_alphas, render_normals, render_distort, render_median

    @staticmethod
    def backward(ctx, v_render_colors, v_render_alphas, v_render_normals, v_render_distort, v_render_median):
        (means2d, ray_transforms, colors, opacities, normals, backgrounds, m8, image_ids, active, offsets, fl, words, cumsum,
         pmap, render_colors, render_alphas, last_ids, median_ids) = ctx.saved_tensors
        R, D, width, height, tw, th, densify_shape = ctx.meta
        dev = render_alphas.device
        if v_render_colors is None:
            v_render_colors = torch.zeros_like(render_colors)
        v_render_colors = v_render_colors.contiguous()
        c = lambda g: None if g is None else g.contiguous()  # noqa: E731
        v_render_alphas, v_render_normals = c(v_render_alphas), c(v_render_normals)
        v_render_distort, v_render_median = c(v_render_distort), c(v_render_median)
        v_means2d, v_ray_transforms = torch.zeros_like(means2d), torch.zeros_like(ray_transforms)
        v_colors, v_opacities, v_normals = torch.zeros_like(colors), torch.zeros_like(opacities), torch.zeros_like(normals)
        v_densify = torch.zeros(densify_shape, device=dev, dtype=torch.float32)
        holder = ctx.absgrad_holder
        v_abs = torch.zeros_like(means2d) if holder is not None else None
        if fl.shape[0] > 0 and pmap.shape[0] > 0:
            with _Ctx(dev) as st:
                check(
                    lib().gsb200_surfel_raster_sparse_bwd(
                        R, D, ptr(means2d), ptr(ray_transforms), ptr(colors), ptr(opacities), ptr(normals), ptr(backgrounds),
                        ptr(m8), width, height, 16, tw, th, active.shape[0], ptr(active), ptr(offsets), ptr(fl), fl.shape[0],
                        ptr(words), ptr(cumsum), ptr(pmap), ptr(render_colors), ptr(render_alphas), ptr(last_ids),
                        ptr(median_ids), ptr(v_render_colors), ptr(v_render_alphas), ptr(v_render_normals),
                        ptr(v_render_distort), ptr(v_render_median), ptr(v_means2d), ptr(v_ray_transforms), ptr(v_colors),
                        ptr(v_opacities), ptr(v_normals), ptr(v_densify), ptr(v_abs), st,
                    ),
                    "rasterize_to_pixels_2dgs_sparse_bwd",
                )
        if holder is not None:
            holder.copy_(v_abs)
        v_backgrounds = None
        if backgrounds is not None and ctx.needs_input_grad[6]:
            v_backgrounds = torch.zeros_like(backgrounds).index_add_(0, image_ids.long(), v_render_colors * (1.0 - render_alphas))
        return (v_means2d, v_ray_transforms, v_colors, v_opacities, v_normals, v_densify, v_backgrounds) + (None,) * 13


def rasterize_to_pixels_2dgs_sparse(
    means2d: Tensor,  # [..., N, 2]
    ray_transforms: Tensor,  # [..., N, 3, 3]
    colors: Tensor,  # [..., N, channels]
    opacities: Tensor,  # [..., N]
    normals: Tensor,  # [..., N, 3]
    densify: Tensor,  # [..., N, 2]
    image_ids: Tensor,  # [P]
    active_tiles: Tensor,  # [AT]
    tile_offsets: Tensor,  # [AT + 1]
    flatten_ids: Tensor,  # [n_isects]
    tile_pixel_mask: Tensor,  # [AT, 4]
    tile_pixel_cumsum: Tensor,  # [AT]
    pixel_map: Tensor,  # [P]
    image_width: int,
    image_height: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
    backgrounds: Optional[Tensor] = None,  # [n_images, channels]
    masks: Optional[Tensor] = None,  # [n_images, tile_height, tile_width]
    absgrad: bool = False,
    distloss: bool = False,
) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """rasterize_to_pixels_2dgs at the pixels of a build_sparse_tile_layout layout only, with the lists of
    isect_tiles_sparse (conics=None) on the surfel rows.  The images are the leading dimensions of the rows, flattened:
    image ``i`` of the layout is row block ``i`` of ``means2d.reshape(-1, N, 2)``.  Returns (render_colors [P, channels],
    render_alphas [P, 1], render_normals [P, 3], render_distort [P, 1], render_median [P, 1]) in the original pixel
    order; each value is the dense rendering's at that pixel (requested pixels in the margin of a partial tile
    included).  The last colour channel is the depth that the distortion and the median depth are taken from.
    ``densify`` receives the densification gradient; with ``absgrad`` the backward fills ``means2d.absgrad``.
    ``distloss`` is accepted for symmetry with rasterize_to_pixels_2dgs: the distortion is always computed."""
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")
    AT, P = _check_sparse_layout(
        image_ids, active_tiles, tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map, image_width,
        image_height, tile_width, tile_height,
    )
    if flatten_ids.dim() != 1:
        raise ValueError(f"flatten_ids must be one-dimensional, got {tuple(flatten_ids.shape)}")
    if means2d.dim() < 2 or means2d.shape[-1] != 2:
        raise ValueError(f"means2d must be [..., N, 2], got {tuple(means2d.shape)}")
    lead, N = tuple(means2d.shape[:-2]), means2d.shape[-2]
    n_images = _prod(lead)
    if colors.dim() != means2d.dim():
        raise ValueError(f"colors must be [..., N, channels], got {tuple(colors.shape)}")
    D = colors.shape[-1]
    _check_shape(ray_transforms, lead + (N, 3, 3), "ray_transforms")
    _check_shape(colors, lead + (N, D), "colors")
    _check_shape(opacities, lead + (N,), "opacities")
    _check_shape(normals, lead + (N, 3), "normals")
    _check_shape(densify, lead + (N, 2), "densify")
    if backgrounds is not None:
        _check_shape(backgrounds, (n_images, D), "backgrounds")
    if masks is not None:
        _check_shape(masks, (n_images, tile_height, tile_width), "masks")
    if D not in _SUPPORTED_CHANNELS:
        raise NotImplementedError(
            f"rasterize_to_pixels_2dgs_sparse: {D} channels; the 2DGS kernels are built for {_SUPPORTED_CHANNELS} (the last "
            "channel is the depth, so the channels cannot be padded)"
        )
    holder = torch.zeros_like(means2d) if absgrad else None
    outs = _RasterizeToPixels2DGSSparse.apply(
        means2d, ray_transforms, colors, opacities, normals, densify, backgrounds, masks, image_ids, active_tiles,
        tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map, int(image_width), int(image_height),
        int(tile_width), int(tile_height), holder,
    )
    if absgrad:
        means2d.absgrad = holder
    return outs

# --------------------------------------------------------------------------------------------
# per-pixel contributor queries (reference wrappers gsplat/cuda/_wrapper.py:1668-2008): the pairs
# rasterize_to_indices_in_range(0, inf) composites from T = 1, per pixel, as counts, padded id lists or the K heaviest.
# Every query is one walk of the pair-query kernel (csrc/raster.cu, raster_indices_kernel) with its own per-pair sink,
# dense over every tile or sparse over the active tiles of a build_sparse_tile_layout layout.  The _2dgs forms (the
# reference has none) are the same queries over the surfel walk (csrc/indices.cuh, pair_walk_kernel with
# csrc/surfel.cu's SurfelModel).

class _ContribWalk(NamedTuple):
    """One pair-query walk of the contributor queries: its rows (tail and name) and its C entries."""

    rows_tail: Optional[tuple]  # (3,) conics or (3, 3) ray_transforms; None for the 3-D rows of the eval3d walk
    rows_name: Optional[str]
    packed: bool  # whether the dense form also takes packed [nnz, *] rows
    count: str
    ids: str
    top: str
    max_samples: str


_CONTRIB_3DGS = _ContribWalk((3,), "conics", True, "gsb200_contrib_count", "gsb200_contrib_ids", "gsb200_contrib_top",
                             "gsb200_contrib_max_samples")
_CONTRIB_2DGS = _ContribWalk((3, 3), "ray_transforms", False, "gsb200_surfel_contrib_count", "gsb200_surfel_contrib_ids",
                             "gsb200_surfel_contrib_top", "gsb200_surfel_contrib_max_samples")
_CONTRIB_EVAL3D = _ContribWalk(None, None, False, "gsb200_eval3d_contrib_count", "gsb200_eval3d_contrib_ids",
                               "gsb200_eval3d_contrib_top", "gsb200_eval3d_contrib_max_samples")

_max_samples_cache = {}


def _max_depth_samples(dev: torch.device, entry: str = _CONTRIB_3DGS.max_samples) -> int:
    """The largest num_depth_samples the top-K kernel of a walk (its ``*_max_samples`` entry) holds on this device (its
    opt-in shared memory per block), cached per walk and device."""
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    if (entry, idx) not in _max_samples_cache:
        with torch.cuda.device(idx):
            rc = getattr(lib(), entry)()
        check(min(rc, 0), entry)
        _max_samples_cache[entry, idx] = rc
    return _max_samples_cache[entry, idx]


def _depth_samples(num_depth_samples) -> int:
    try:
        K = operator.index(num_depth_samples)
    except TypeError:
        raise TypeError(f"num_depth_samples must be an integer, got {type(num_depth_samples).__name__}") from None
    if K <= 0:
        raise ValueError(f"num_depth_samples must be greater than 0, got {K}")
    return K


def _contrib_rows(walk, means2d, rows, opacities, image_dims=None) -> int:
    """Checks dense [..., N, *] rows, or packed [nnz, *] rows where the walk takes them; returns N (nnz when packed: ids
    are then row indices)."""
    if means2d.dim() < 2 or means2d.shape[-1] != 2:
        shapes = "[..., N, 2] or [nnz, 2]" if walk.packed else "[..., N, 2]"
        raise ValueError(f"means2d must be {shapes}, got {tuple(means2d.shape)}")
    lead = tuple(means2d.shape[:-1])
    if (means2d.dim() > 2 or not walk.packed) and image_dims is not None and lead[:-1] != tuple(image_dims):
        raise ValueError(f"means2d must be {tuple(image_dims) + ('N', 2)} to match tile_offsets, got {tuple(means2d.shape)}")
    _check_shape(rows, lead + walk.rows_tail, walk.rows_name)
    _check_shape(opacities, lead, "opacities")
    return lead[-1]


class _PlanarRows(NamedTuple):
    """What the 3DGS and 2DGS walks composite: means2d, conics or ray_transforms, opacities."""

    walk: _ContribWalk
    means2d: Tensor
    rows: Tensor
    opacities: Tensor

    def check(self, image_dims=None) -> int:
        """The shapes, against the images of a dense layout if given; returns N."""
        return _contrib_rows(self.walk, self.means2d, self.rows, self.opacities, image_dims)

    def floats(self):
        return (self.means2d, "means2d"), (self.rows, self.walk.rows_name), (self.opacities, "opacities")

    def tensors(self):
        return self.means2d, self.rows, self.opacities

    def head(self, I, N):
        """The C arguments before the image size, and the tensors they point into."""
        keep = [t.contiguous() for t in self.tensors()]
        return (I, N) + tuple(ptr(t) for t in keep), keep


class _Eval3dRows:
    """What the eval3d walk composites: the 3-D Gaussians, the (batch, camera) opacities and the cameras of
    rasterize_to_pixels_eval3d, checked as it checks them."""

    walk = _CONTRIB_EVAL3D

    def __init__(self, what, means, quats, scales, opacities, viewmats, Ks, width, height, camera_model, radial_coeffs,
                 tangential_coeffs, thin_prism_coeffs, ftheta_coeffs, rolling_shutter, viewmats_rs):
        self.what, self.means, self.quats, self.scales, self.opacities = what, means, quats, scales, opacities
        self.viewmats, self.Ks, self.width, self.height = viewmats, Ks, int(width), int(height)
        self.camera = (camera_model, radial_coeffs, tangential_coeffs, thin_prism_coeffs, ftheta_coeffs, rolling_shutter,
                       viewmats_rs)
        self.cam = None

    def check(self, image_dims=None) -> int:
        batch, C, N = _ut_geometry(self.what, self.means, self.quats, self.scales, self.viewmats, self.Ks)
        if image_dims is not None and tuple(image_dims) != batch + (C,):
            raise ValueError(f"{self.what}: tile_offsets must be {batch + (C, 'tile_height', 'tile_width')} to match the "
                             f"cameras, got images {tuple(image_dims)}")
        _check_shape(self.opacities, batch + (C, N), "opacities")
        model, radial, tangential, thin, ftheta, shutter, viewmats_rs = self.camera
        self.cam = _ut_camera(self.what, self.viewmats, self.width, self.height, model, radial, tangential, thin, ftheta,
                              None, None, shutter, viewmats_rs)
        self.B, self.C = _prod(batch), C
        return N

    def floats(self):
        return ((self.opacities, "opacities"),)  # the geometry's dtypes are _ut_geometry's

    def tensors(self):
        c = self.cam
        return (self.means, self.quats, self.scales, self.opacities, self.viewmats, self.Ks, c.radial, c.tangential, c.thin,
                c.viewmats_rs)

    def head(self, I, N):
        c = self.cam
        keep = [t.contiguous() for t in self.tensors()[:6]] + [c]  # c.ftheta is read through its host address
        return (self.B, self.C, N, *(ptr(t) for t in keep[:6]), c.model, ptr(c.radial), ptr(c.tangential), ptr(c.thin),
                _ftheta_ptr(c.ftheta), ptr(c.viewmats_rs), c.shutter), keep


def _contrib_dtypes(floats, ints) -> None:
    for t, name in floats:
        if t.dtype != torch.float32:
            raise TypeError(f"{name}: expected float32, got {t.dtype} (gsplat_b200 computes in fp32 only)")
    for t, name, dt in ints:
        if t.dtype != dt:
            raise TypeError(f"{name} must be {dt}, got {t.dtype}")


def _check_counts(num_contributing_gaussians, dims) -> None:
    nc = num_contributing_gaussians
    if nc is None:
        return
    if tuple(nc.shape) != tuple(dims):
        raise ValueError(f"num_contributing_gaussians must have shape {tuple(dims)}, got {tuple(nc.shape)}")
    if nc.dtype != torch.int32:
        raise TypeError(f"num_contributing_gaussians must have dtype int32, got {nc.dtype}")


def _contrib_dense(rows, tile_offsets, flatten_ids, image_width, image_height, tile_size, counts=None):
    """Checks the dense-layout arguments (and the per-pixel counts, if given) over the walk's rows (_PlanarRows or
    _Eval3dRows); returns (the walk, the output dims [..., H, W], (the C arguments before the outputs, the tensors they
    point into), the device)."""
    W, H = int(image_width), int(image_height)
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")
    if tile_offsets.dim() < 2:
        raise ValueError(f"tile_offsets must be [..., tile_height, tile_width], got {tuple(tile_offsets.shape)}")
    image_dims = tuple(tile_offsets.shape[:-2])
    th, tw = tile_offsets.shape[-2:]
    N = rows.check(image_dims)
    if th * 16 < H or tw * 16 < W:
        raise ValueError(f"tile_offsets tile grid {tw}x{th} does not cover a {W}x{H} image")
    if flatten_ids.dim() != 1:
        raise ValueError(f"flatten_ids must be one-dimensional, got {tuple(flatten_ids.shape)}")
    _contrib_dtypes(rows.floats(), ((tile_offsets, "tile_offsets", torch.int32), (flatten_ids, "flatten_ids", torch.int32)))
    _check_counts(counts, image_dims + (H, W))
    dev = require_cuda(*rows.tensors(), tile_offsets, flatten_ids, counts)
    head, keep = rows.head(_prod(image_dims), N)
    off, fl = tile_offsets.contiguous(), flatten_ids.contiguous()
    args = head + (W, H, 16, tw, th, ptr(off), ptr(fl), fl.shape[0], 0, None, None, None, None)
    return rows.walk, image_dims + (H, W), (args, keep + [off, fl]), dev


def _contrib_sparse(rows, active_tiles, tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map,
                    image_width, image_height, tile_size, tile_width, tile_height, counts=None):
    """_contrib_dense for a sparse layout: the output dims are [P]."""
    W, H, tw, th = int(image_width), int(image_height), int(tile_width), int(tile_height)
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")
    N = rows.check()
    if active_tiles.dim() != 1 or pixel_map.dim() != 1 or flatten_ids.dim() != 1:
        raise ValueError("active_tiles [AT], pixel_map [P] and flatten_ids [n_isects] must be one-dimensional")
    AT, P = active_tiles.shape[0], pixel_map.shape[0]
    if AT == 0 and P > 0:
        raise ValueError(f"pixel_map lists {P} pixels but the layout has no active tile (build_sparse_tile_layout)")
    _check_shape(tile_offsets, (AT + 1,), "tile_offsets")
    _check_shape(tile_pixel_mask, (AT, _TILE_WORDS), "tile_pixel_mask")
    if tuple(tile_pixel_cumsum.shape) not in (((AT,),) if AT > 0 else ((0,), (1,))):
        raise ValueError(f"tile_pixel_cumsum must be [{AT}], got {tuple(tile_pixel_cumsum.shape)}")
    if tw * 16 < W or th * 16 < H:
        raise ValueError(f"a {tw} x {th} tile grid does not cover {W} x {H} pixels")
    if tile_pixel_mask.element_size() != 8 or tile_pixel_mask.is_floating_point():
        raise TypeError(f"tile_pixel_mask must be a 64-bit integer tensor, got {tile_pixel_mask.dtype}")
    _contrib_dtypes(rows.floats(),
                    ((active_tiles, "active_tiles", torch.int32), (tile_offsets, "tile_offsets", torch.int32),
                     (flatten_ids, "flatten_ids", torch.int32), (tile_pixel_cumsum, "tile_pixel_cumsum", torch.int64),
                     (pixel_map, "pixel_map", torch.int64)))
    _check_counts(counts, (P,))
    dev = require_cuda(*rows.tensors(), active_tiles, tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum,
                       pixel_map, counts)
    head, keep = rows.head(1, N)
    layout = [t.contiguous() for t in (tile_offsets, flatten_ids, active_tiles, tile_pixel_mask, tile_pixel_cumsum,
                                       pixel_map)]
    off, fl, act, words, cum, pmap = layout
    args = head + (W, H, 16, tw, th, ptr(off), ptr(fl), fl.shape[0], AT, ptr(act), ptr(words), ptr(cum), ptr(pmap))
    return rows.walk, (P,), (args, keep + layout), dev


def _contrib_count(what, checked):
    walk, dims, (args, _keep), dev = checked
    counts = torch.empty(dims, device=dev, dtype=torch.int32)
    alphas = torch.empty(dims, device=dev, dtype=torch.float32)
    if counts.numel() > 0:  # a sparse layout without pixels has no active tile either: nothing to launch
        with _Ctx(dev) as st:
            check(getattr(lib(), walk.count)(*args, ptr(counts), ptr(alphas), st), what)
    return counts, alphas


def _contrib_ids(what, checked, nc):
    walk, dims, (args, _keep), dev = checked
    K = 0
    if nc.numel() > 0:
        lo, K = (int(v) for v in torch.stack(torch.aminmax(nc)).tolist())  # the one host read
        if lo < 0:
            raise ValueError("num_contributing_gaussians must be non-negative")
    ids = torch.empty(dims + (K,), device=dev, dtype=torch.int32)
    weights = torch.empty(dims + (K,), device=dev, dtype=torch.float32)
    if ids.numel() > 0:
        with _Ctx(dev) as st:
            check(getattr(lib(), walk.ids)(*args, K, ptr(ids), ptr(weights), st), what)
    return ids, weights


def _contrib_top(what, checked, K):
    walk, dims, (args, _keep), dev = checked
    # the 3DGS walk's bound is _max_depth_samples' default
    bound = _max_depth_samples(dev) if walk is _CONTRIB_3DGS else _max_depth_samples(dev, walk.max_samples)
    if K > bound:
        raise ValueError(f"num_depth_samples {K} exceeds {bound}, the most the top-K kernel holds in shared memory on {dev}")
    ids = torch.empty(dims + (K,), device=dev, dtype=torch.int32)
    weights = torch.empty(dims + (K,), device=dev, dtype=torch.float32)
    if ids.numel() > 0:
        with _Ctx(dev) as st:
            check(getattr(lib(), walk.top)(*args, K, ptr(ids), ptr(weights), st), what)
    return ids, weights


@torch.no_grad()
def rasterize_num_contributing_gaussians(
    means2d: Tensor,  # [..., N, 2] or [nnz, 2]
    conics: Tensor,  # [..., N, 3] or [nnz, 3]
    opacities: Tensor,  # [..., N] or [nnz]
    tile_offsets: Tensor,  # [..., tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    image_width: int,
    image_height: int,
    tile_size: int,
) -> Tuple[Tensor, Tensor]:
    """Per pixel, the number of Gaussians ``rasterize_to_pixels`` composites and its accumulated alpha.  The decisions
    are the compositing kernel's own, so the alphas equal ``render_alphas``.  Returns (counts int32 [..., H, W],
    alphas float32 [..., H, W])."""
    checked = _contrib_dense(_PlanarRows(_CONTRIB_3DGS, means2d, conics, opacities), tile_offsets, flatten_ids,
                             image_width, image_height, tile_size)
    return _contrib_count("rasterize_num_contributing_gaussians", checked)


@torch.no_grad()
def rasterize_num_contributing_gaussians_sparse(
    means2d: Tensor,  # [..., N, 2] or [nnz, 2]
    conics: Tensor,  # [..., N, 3] or [nnz, 3]
    opacities: Tensor,  # [..., N] or [nnz]
    active_tiles: Tensor,  # [AT]
    tile_offsets: Tensor,  # [AT + 1]
    flatten_ids: Tensor,  # [n_isects]
    tile_pixel_mask: Tensor,  # [AT, 4]
    tile_pixel_cumsum: Tensor,  # [AT]
    pixel_map: Tensor,  # [P]
    image_width: int,
    image_height: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
) -> Tuple[Tensor, Tensor]:
    """``rasterize_num_contributing_gaussians`` at the pixels of a build_sparse_tile_layout layout, with the lists of
    isect_tiles_sparse.  Returns (counts int32 [P], alphas float32 [P]) in the original pixel order."""
    checked = _contrib_sparse(_PlanarRows(_CONTRIB_3DGS, means2d, conics, opacities), active_tiles, tile_offsets,
                              flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map, image_width, image_height,
                              tile_size, tile_width, tile_height)
    return _contrib_count("rasterize_num_contributing_gaussians_sparse", checked)


@torch.no_grad()
def rasterize_contributing_gaussian_ids(
    means2d: Tensor,  # [..., N, 2] or [nnz, 2]
    conics: Tensor,  # [..., N, 3] or [nnz, 3]
    opacities: Tensor,  # [..., N] or [nnz]
    tile_offsets: Tensor,  # [..., tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    image_width: int,
    image_height: int,
    tile_size: int,
    num_contributing_gaussians: Tensor,  # [..., image_height, image_width]
) -> Tuple[Tensor, Tensor]:
    """Every Gaussian each pixel composites, front to back, with its weight ``alpha * T`` (T before it).  Returns
    (ids int32, weights float32) [..., H, W, K] with K = ``num_contributing_gaussians.max()`` (read back to the host
    once): a pixel's first K pairs (later ones are dropped), then -1 / 0.  Ids index N (dense rows) or nnz (packed)."""
    checked = _contrib_dense(_PlanarRows(_CONTRIB_3DGS, means2d, conics, opacities), tile_offsets, flatten_ids,
                             image_width, image_height, tile_size, num_contributing_gaussians)
    return _contrib_ids("rasterize_contributing_gaussian_ids", checked, num_contributing_gaussians)


@torch.no_grad()
def rasterize_contributing_gaussian_ids_sparse(
    means2d: Tensor,  # [..., N, 2] or [nnz, 2]
    conics: Tensor,  # [..., N, 3] or [nnz, 3]
    opacities: Tensor,  # [..., N] or [nnz]
    active_tiles: Tensor,  # [AT]
    tile_offsets: Tensor,  # [AT + 1]
    flatten_ids: Tensor,  # [n_isects]
    tile_pixel_mask: Tensor,  # [AT, 4]
    tile_pixel_cumsum: Tensor,  # [AT]
    pixel_map: Tensor,  # [P]
    num_contributing_gaussians: Tensor,  # [P] int32
    image_width: int,
    image_height: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
) -> Tuple[Tensor, Tensor]:
    """``rasterize_contributing_gaussian_ids`` at the pixels of a sparse layout: (ids, weights) [P, K] in the original
    pixel order."""
    checked = _contrib_sparse(_PlanarRows(_CONTRIB_3DGS, means2d, conics, opacities), active_tiles, tile_offsets,
                              flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map, image_width, image_height,
                              tile_size, tile_width, tile_height, num_contributing_gaussians)
    return _contrib_ids("rasterize_contributing_gaussian_ids_sparse", checked, num_contributing_gaussians)


@torch.no_grad()
def rasterize_top_contributing_gaussian_ids(
    means2d: Tensor,  # [..., N, 2] or [nnz, 2]
    conics: Tensor,  # [..., N, 3] or [nnz, 3]
    opacities: Tensor,  # [..., N] or [nnz]
    tile_offsets: Tensor,  # [..., tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    image_width: int,
    image_height: int,
    tile_size: int,
    num_depth_samples: int,
) -> Tuple[Tensor, Tensor]:
    """The ``num_depth_samples`` heaviest pairs of each pixel by ``alpha * T``, front to back: (ids int32, weights
    float32) [..., H, W, K], -1 / 0 in unused slots.  A pair replaces the lightest kept one (the first on ties) only when
    strictly heavier, as in the reference.  K must lie in [1, the device's bound] (about 71 on an H100: K slots per pixel
    live in shared memory); outside it a ValueError is raised before anything runs."""
    K = _depth_samples(num_depth_samples)
    checked = _contrib_dense(_PlanarRows(_CONTRIB_3DGS, means2d, conics, opacities), tile_offsets, flatten_ids,
                             image_width, image_height, tile_size)
    return _contrib_top("rasterize_top_contributing_gaussian_ids", checked, K)


@torch.no_grad()
def rasterize_top_contributing_gaussian_ids_sparse(
    means2d: Tensor,  # [..., N, 2] or [nnz, 2]
    conics: Tensor,  # [..., N, 3] or [nnz, 3]
    opacities: Tensor,  # [..., N] or [nnz]
    active_tiles: Tensor,  # [AT]
    tile_offsets: Tensor,  # [AT + 1]
    flatten_ids: Tensor,  # [n_isects]
    tile_pixel_mask: Tensor,  # [AT, 4]
    tile_pixel_cumsum: Tensor,  # [AT]
    pixel_map: Tensor,  # [P]
    image_width: int,
    image_height: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
    num_depth_samples: int,
) -> Tuple[Tensor, Tensor]:
    """``rasterize_top_contributing_gaussian_ids`` at the pixels of a sparse layout: (ids, weights) [P, K] in the
    original pixel order."""
    K = _depth_samples(num_depth_samples)
    checked = _contrib_sparse(_PlanarRows(_CONTRIB_3DGS, means2d, conics, opacities), active_tiles, tile_offsets,
                              flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map, image_width, image_height,
                              tile_size, tile_width, tile_height)
    return _contrib_top("rasterize_top_contributing_gaussian_ids_sparse", checked, K)


@torch.no_grad()
def rasterize_num_contributing_gaussians_2dgs(
    means2d: Tensor,  # [..., N, 2]
    ray_transforms: Tensor,  # [..., N, 3, 3]
    opacities: Tensor,  # [..., N]
    tile_offsets: Tensor,  # [..., tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    image_width: int,
    image_height: int,
    tile_size: int,
) -> Tuple[Tensor, Tensor]:
    """``rasterize_num_contributing_gaussians`` for surfels: per pixel, the number of surfels
    ``rasterize_to_pixels_2dgs`` composites and its accumulated alpha.  The decisions are the 2DGS compositing kernel's
    own, so the alphas equal its ``render_alphas`` bit for bit.  Returns (counts int32 [..., H, W], alphas float32
    [..., H, W])."""
    checked = _contrib_dense(_PlanarRows(_CONTRIB_2DGS, means2d, ray_transforms, opacities), tile_offsets, flatten_ids,
                             image_width, image_height, tile_size)
    return _contrib_count("rasterize_num_contributing_gaussians_2dgs", checked)


@torch.no_grad()
def rasterize_num_contributing_gaussians_2dgs_sparse(
    means2d: Tensor,  # [..., N, 2]
    ray_transforms: Tensor,  # [..., N, 3, 3]
    opacities: Tensor,  # [..., N]
    active_tiles: Tensor,  # [AT]
    tile_offsets: Tensor,  # [AT + 1]
    flatten_ids: Tensor,  # [n_isects]
    tile_pixel_mask: Tensor,  # [AT, 4]
    tile_pixel_cumsum: Tensor,  # [AT]
    pixel_map: Tensor,  # [P]
    image_width: int,
    image_height: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
) -> Tuple[Tensor, Tensor]:
    """``rasterize_num_contributing_gaussians_2dgs`` at the pixels of a build_sparse_tile_layout layout, with the lists
    of isect_tiles_sparse (conics=None) on the surfel rows.  Returns (counts int32 [P], alphas float32 [P]) in the
    original pixel order."""
    checked = _contrib_sparse(_PlanarRows(_CONTRIB_2DGS, means2d, ray_transforms, opacities), active_tiles,
                              tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map, image_width,
                              image_height, tile_size, tile_width, tile_height)
    return _contrib_count("rasterize_num_contributing_gaussians_2dgs_sparse", checked)


@torch.no_grad()
def rasterize_contributing_gaussian_ids_2dgs(
    means2d: Tensor,  # [..., N, 2]
    ray_transforms: Tensor,  # [..., N, 3, 3]
    opacities: Tensor,  # [..., N]
    tile_offsets: Tensor,  # [..., tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    image_width: int,
    image_height: int,
    tile_size: int,
    num_contributing_gaussians: Tensor,  # [..., image_height, image_width]
) -> Tuple[Tensor, Tensor]:
    """Every surfel each pixel composites, front to back, with its weight ``alpha * T`` (T before it).  Returns
    (ids int32, weights float32) [..., H, W, K] with K = ``num_contributing_gaussians.max()`` (read back to the host
    once): a pixel's first K pairs (later ones are dropped), then -1 / 0.  Ids index N."""
    checked = _contrib_dense(_PlanarRows(_CONTRIB_2DGS, means2d, ray_transforms, opacities), tile_offsets, flatten_ids,
                             image_width, image_height, tile_size, num_contributing_gaussians)
    return _contrib_ids("rasterize_contributing_gaussian_ids_2dgs", checked, num_contributing_gaussians)


@torch.no_grad()
def rasterize_contributing_gaussian_ids_2dgs_sparse(
    means2d: Tensor,  # [..., N, 2]
    ray_transforms: Tensor,  # [..., N, 3, 3]
    opacities: Tensor,  # [..., N]
    active_tiles: Tensor,  # [AT]
    tile_offsets: Tensor,  # [AT + 1]
    flatten_ids: Tensor,  # [n_isects]
    tile_pixel_mask: Tensor,  # [AT, 4]
    tile_pixel_cumsum: Tensor,  # [AT]
    pixel_map: Tensor,  # [P]
    num_contributing_gaussians: Tensor,  # [P] int32
    image_width: int,
    image_height: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
) -> Tuple[Tensor, Tensor]:
    """``rasterize_contributing_gaussian_ids_2dgs`` at the pixels of a sparse layout: (ids, weights) [P, K] in the
    original pixel order."""
    checked = _contrib_sparse(_PlanarRows(_CONTRIB_2DGS, means2d, ray_transforms, opacities), active_tiles,
                              tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map, image_width,
                              image_height, tile_size, tile_width, tile_height, num_contributing_gaussians)
    return _contrib_ids("rasterize_contributing_gaussian_ids_2dgs_sparse", checked, num_contributing_gaussians)


@torch.no_grad()
def rasterize_top_contributing_gaussian_ids_2dgs(
    means2d: Tensor,  # [..., N, 2]
    ray_transforms: Tensor,  # [..., N, 3, 3]
    opacities: Tensor,  # [..., N]
    tile_offsets: Tensor,  # [..., tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    image_width: int,
    image_height: int,
    tile_size: int,
    num_depth_samples: int,
) -> Tuple[Tensor, Tensor]:
    """The ``num_depth_samples`` heaviest surfels of each pixel by ``alpha * T``, front to back: (ids int32, weights
    float32) [..., H, W, K], -1 / 0 in unused slots, by the rule of ``rasterize_top_contributing_gaussian_ids``.  K must
    lie in [1, the surfel walk's bound on the device] (71 on an H100); outside it a ValueError is raised before anything
    runs."""
    K = _depth_samples(num_depth_samples)
    checked = _contrib_dense(_PlanarRows(_CONTRIB_2DGS, means2d, ray_transforms, opacities), tile_offsets, flatten_ids,
                             image_width, image_height, tile_size)
    return _contrib_top("rasterize_top_contributing_gaussian_ids_2dgs", checked, K)


@torch.no_grad()
def rasterize_top_contributing_gaussian_ids_2dgs_sparse(
    means2d: Tensor,  # [..., N, 2]
    ray_transforms: Tensor,  # [..., N, 3, 3]
    opacities: Tensor,  # [..., N]
    active_tiles: Tensor,  # [AT]
    tile_offsets: Tensor,  # [AT + 1]
    flatten_ids: Tensor,  # [n_isects]
    tile_pixel_mask: Tensor,  # [AT, 4]
    tile_pixel_cumsum: Tensor,  # [AT]
    pixel_map: Tensor,  # [P]
    image_width: int,
    image_height: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
    num_depth_samples: int,
) -> Tuple[Tensor, Tensor]:
    """``rasterize_top_contributing_gaussian_ids_2dgs`` at the pixels of a sparse layout: (ids, weights) [P, K] in the
    original pixel order."""
    K = _depth_samples(num_depth_samples)
    checked = _contrib_sparse(_PlanarRows(_CONTRIB_2DGS, means2d, ray_transforms, opacities), active_tiles,
                              tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map, image_width,
                              image_height, tile_size, tile_width, tile_height)
    return _contrib_top("rasterize_top_contributing_gaussian_ids_2dgs_sparse", checked, K)


# --------------------------------------------------------------------------------------------
# MCMC strategy ops ("next" row, SURVEY.md section 8f.3)


@torch.no_grad()
def compute_relocation(
    opacities: Tensor, scales: Tensor, ratios: Tensor, binoms: Tensor, min_opacity: float = 0.005
) -> Tuple[Tensor, Tensor]:
    """Eq. 9 of "3D Gaussian Splatting as Markov Chain Monte Carlo": opacities / scales of Gaussians that are
    split into ``ratios`` copies.  Mirrors gsplat.relocation.compute_relocation
    (/root/reference/gsplat/relocation.py:25-80): ``ratios`` is clamped to [1, n_max] in place."""
    dev = require_cuda(opacities, scales, ratios, binoms)
    N = opacities.shape[0]
    n_max = binoms.shape[0]
    assert scales.shape == (N, 3), scales.shape
    assert ratios.shape == (N,), ratios.shape
    opacities, scales, binoms = f32c(opacities, "opacities"), f32c(scales, "scales"), f32c(binoms, "binoms")
    ratios.clamp_(min=1, max=n_max)
    r32 = ratios.int().contiguous()
    new_opacities, new_scales = torch.empty_like(opacities), torch.empty_like(scales)
    with _Ctx(dev) as st:
        check(
            lib().gsb200_relocation(
                N, ptr(opacities), ptr(scales), ptr(r32), ptr(binoms), n_max, float(min_opacity), ptr(new_opacities),
                ptr(new_scales), st,
            ),
            "relocation",
        )
    return new_opacities, new_scales


@torch.no_grad()
def mcmc_perturb_positions(
    positions: Tensor, quats: Tensor, scales_log: Tensor, opacities_logit: Tensor, noise: Tensor, noise_scale: float,
    t: float = 0.005, k: float = 100.0,
) -> None:
    """In place: positions += Sigma(quats, exp(scales_log)) @ (noise * sigmoid(-k (sigmoid(opacities_logit) - t))
    * noise_scale)   (/root/reference/gsplat/cuda/csrc/MCMCPerturbCUDA.cu:28-60)."""
    dev = require_cuda(positions, quats, scales_log, opacities_logit, noise)
    if not positions.is_contiguous() or positions.dtype != torch.float32:
        raise ValueError("positions must be a contiguous float32 tensor (updated in place)")
    N = positions.shape[0]
    quats, scales_log = f32c(quats, "quats"), f32c(scales_log, "scales")
    opacities_logit, noise = f32c(opacities_logit, "opacities"), f32c(noise, "noise")
    with _Ctx(dev) as st:
        check(
            lib().gsb200_mcmc_perturb_positions(
                N, ptr(positions), ptr(quats), ptr(scales_log), ptr(opacities_logit), ptr(noise), float(noise_scale),
                float(t), float(k), st,
            ),
            "mcmc_perturb_positions",
        )


@torch.no_grad()
def adam(
    param: Tensor, param_grad: Tensor, exp_avg: Tensor, exp_avg_sq: Tensor, valid: Optional[Tensor], lr: float, b1: float,
    b2: float, eps: float,
) -> None:
    """Selective Adam step, in place on ``param`` / ``exp_avg`` / ``exp_avg_sq`` ([N, ...]); rows with
    ``valid[n] == False`` keep their value and their moments (/root/reference/gsplat/cuda/_wrapper.py:419-432,
    csrc/AdamCUDA.cu:34-70; no bias correction, like the reference)."""
    dev = require_cuda(param, param_grad, exp_avg, exp_avg_sq)
    for name, t in (("param", param), ("exp_avg", exp_avg), ("exp_avg_sq", exp_avg_sq)):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous float32 tensor (updated in place)")
        if t.shape != param.shape:
            raise ValueError(f"{name} must have the shape of param")
    if param_grad.shape != param.shape:
        raise ValueError("param_grad must have the shape of param")
    param_grad = f32c(param_grad, "param_grad")
    N = param.shape[0] if param.dim() > 0 else 1
    D = param.numel() // max(N, 1)
    vmask = None
    if valid is not None:
        if valid.numel() != N:
            raise ValueError(f"valid must have {N} entries, got {valid.numel()}")
        vmask = valid.to(device=dev, dtype=torch.bool).contiguous()
    with _Ctx(dev) as st:
        check(
            lib().gsb200_adam(
                N, D, ptr(param), ptr(param_grad), ptr(exp_avg), ptr(exp_avg_sq), ptr(vmask), float(lr), float(b1), float(b2),
                float(eps), st,
            ),
            "adam",
        )


# --------------------------------------------------------------------------------------------
# 3DGUT (reference wrappers gsplat/cuda/_wrapper.py: fully_fused_projection_with_ut, rasterize_to_pixels_eval3d): the
# unscented-transform projection through a distorted pinhole or fisheye camera and the compositing that evaluates
# each gaussian in 3-D along the pixel's ray.  Pinhole, fisheye or FTheta cameras, global or rolling shutter, dense rows,
# RendererConfig_MixedBatch.

_UT_DEFAULTS = {"alpha": 0.1, "beta": 2.0, "kappa": 0.0, "in_image_margin_factor": 0.1, "require_all_sigma_points_valid": False}
_UT_CAMERAS = {"pinhole": 0, "fisheye": 2, "ftheta": 3}


def _ut_params(ut_params) -> tuple:
    """(alpha, beta, kappa, in_image_margin_factor, require_all_sigma_points_valid) of any object with the reference's
    UnscentedTransformParameters fields (a missing field takes its default), or the defaults for None."""
    v = {k: (d if ut_params is None else getattr(ut_params, k, d)) for k, d in _UT_DEFAULTS.items()}
    alpha, kappa = float(v["alpha"]), float(v["kappa"])
    if not alpha * alpha * (3.0 + kappa) > 0.0:
        raise ValueError(f"ut_params: alpha^2 * (3 + kappa) must be > 0 (alpha={alpha}, kappa={kappa})")
    return alpha, float(v["beta"]), kappa, float(v["in_image_margin_factor"]), bool(v["require_all_sigma_points_valid"])


class RollingShutterType(enum.IntEnum):
    """How a camera's sensor is exposed (the reference's RollingShutterType): row by row or column by column in the
    given direction, each row or column at its own pose between ``viewmats`` and ``viewmats_rs``, or all at once."""

    ROLLING_TOP_TO_BOTTOM = 0
    ROLLING_LEFT_TO_RIGHT = 1
    ROLLING_BOTTOM_TO_TOP = 2
    ROLLING_RIGHT_TO_LEFT = 3
    GLOBAL = 4


def _shutter_type(rolling_shutter) -> RollingShutterType:
    """The RollingShutterType of None (GLOBAL), of an int value, of any enum or object whose ``.name`` is a member's
    name (this package's, the reference's), or of such a name as a string ("GLOBAL", "RollingShutterType.GLOBAL")."""
    if rolling_shutter is None:
        return RollingShutterType.GLOBAL
    name = getattr(rolling_shutter, "name", None)
    if name is None and isinstance(rolling_shutter, str):
        name = rolling_shutter.rsplit(".", 1)[-1]
    if name is not None:
        if name in RollingShutterType.__members__:
            return RollingShutterType[name]
    elif isinstance(rolling_shutter, int) and rolling_shutter in set(RollingShutterType):
        return RollingShutterType(rolling_shutter)
    raise ValueError(f"unknown rolling_shutter {rolling_shutter!r}")


class FThetaPolynomialType(enum.IntEnum):
    """Which of an FTheta calibration's two polynomials is the reference (the reference's FThetaPolynomialType): the
    other direction inverts it by Newton steps."""

    PIXELDIST_TO_ANGLE = 0
    ANGLE_TO_PIXELDIST = 1


class FThetaCameraDistortionParameters:
    """The parameters of an FTheta camera, shared by every camera of a call (the reference's
    FThetaCameraDistortionParameters, same keywords and defaults).  ``pixeldist_to_angle_poly`` (backward) and
    ``angle_to_pixeldist_poly`` (forward) are the coefficients c0 .. c5 of two degree-5 polynomials between the angle
    of a ray from the optical axis and its distance in pixels from the principal point; ``reference_poly`` names the one
    evaluated directly; ``max_angle`` bounds the field of view (radians, beyond pi / 2 for lenses that see behind the
    camera plane); ``linear_cde`` = (c, d, e) maps the radial offset to the image by [[c, d], [e, 1]].  The principal
    point is each camera's ``Ks`` (cx, cy) + 0.5, FTheta's image origin being the centre of the first pixel; fx and fy
    are unused.  The operators accept any object with these five attributes."""

    def __init__(self, reference_poly=0, pixeldist_to_angle_poly=(0.0,) * 6, angle_to_pixeldist_poly=(0.0,) * 6,
                 max_angle=0.0, linear_cde=(0.0,) * 3):
        self.reference_poly = reference_poly
        self.pixeldist_to_angle_poly = list(pixeldist_to_angle_poly)
        self.angle_to_pixeldist_poly = list(angle_to_pixeldist_poly)
        self.max_angle = max_angle
        self.linear_cde = list(linear_cde)

    def __repr__(self):
        return (f"FThetaCameraDistortionParameters(reference_poly={int(self.reference_poly)}, "
                f"pixeldist_to_angle_poly={self.pixeldist_to_angle_poly}, angle_to_pixeldist_poly={self.angle_to_pixeldist_poly}, "
                f"max_angle={self.max_angle}, linear_cde={self.linear_cde})")


def _ftheta_params(what, ftheta_coeffs) -> "_cabi.FThetaParams":
    """The gsb200_ftheta_params of any object with the five attributes of FThetaCameraDistortionParameters (this
    package's, the reference's torch class).  ValueError for a missing attribute, a wrong length, a reference_poly other
    than 0 / 1 or a non-finite value."""
    fields = {}
    for name, n in (("reference_poly", None), ("pixeldist_to_angle_poly", 6), ("angle_to_pixeldist_poly", 6),
                    ("max_angle", None), ("linear_cde", 3)):
        if not hasattr(ftheta_coeffs, name):
            raise ValueError(f"{what}: ftheta_coeffs has no {name} (expected FThetaCameraDistortionParameters)")
        v = getattr(ftheta_coeffs, name)
        try:
            v = [float(x) for x in v] if n is not None else float(v)
        except (TypeError, ValueError) as e:
            raise ValueError(f"{what}: ftheta_coeffs.{name} is not {'a sequence of ' if n else 'a '}number{'s' if n else ''}: {v!r}") from e
        if n is not None and len(v) != n:
            raise ValueError(f"{what}: ftheta_coeffs.{name} must have {n} values, got {len(v)}")
        if not all(math.isfinite(x) for x in (v if n is not None else [v])):
            raise ValueError(f"{what}: ftheta_coeffs.{name} must be finite, got {v}")
        fields[name] = v
    if fields["reference_poly"] not in (0.0, 1.0):
        raise ValueError(f"{what}: ftheta_coeffs.reference_poly must be 0 (PIXELDIST_TO_ANGLE) or 1 (ANGLE_TO_PIXELDIST), "
                         f"got {ftheta_coeffs.reference_poly!r}")
    p = _cabi.FThetaParams()
    p.reference_poly = int(fields["reference_poly"])
    p.pixeldist_to_angle_poly[:] = fields["pixeldist_to_angle_poly"]
    p.angle_to_pixeldist_poly[:] = fields["angle_to_pixeldist_poly"]
    p.max_angle = fields["max_angle"]
    p.linear_cde[:] = fields["linear_cde"]
    return p


def _ftheta_ptr(params) -> int:
    """Host address of a gsb200_ftheta_params (0 for None); the caller keeps ``params`` alive across the call."""
    import ctypes

    return 0 if params is None else ctypes.addressof(params)


class _UtCamera(NamedTuple):
    """A checked 3DGUT camera, shared by the projection and the compositing: the camera model id, the coefficient
    tensors [..., C, k] float32 (None where absent), the FTheta parameters (a gsb200_ftheta_params, or None for the other
    models), the shutter type id, the end-of-frame poses (detached and contiguous, None under the global shutter) and
    the depth order."""

    model: int
    radial: Optional[Tensor]
    tangential: Optional[Tensor]
    thin: Optional[Tensor]
    ftheta: Optional["_cabi.FThetaParams"]
    shutter: int
    viewmats_rs: Optional[Tensor]
    global_z_order: bool


def _ut_camera(what, viewmats: Tensor, width: int, height: int, camera_model, radial_coeffs, tangential_coeffs,
               thin_prism_coeffs, ftheta_coeffs, lidar_coeffs, external_distortion_coeffs, rolling_shutter, viewmats_rs,
               global_z_order: bool = True) -> _UtCamera:
    """Checks the camera and shutter arguments of the 3DGUT path.  What the kernels are not built for raises
    NotImplementedError, naming the argument: lidar and external distortion, the camera arguments of another model, a
    rolling shutter without ``viewmats_rs`` or ``viewmats_rs`` under the global shutter.  Malformed values raise
    ValueError (or TypeError for a dtype), among them a rolling shutter over a single row or column, which has no frame
    time."""
    for name, v in (("lidar_coeffs", lidar_coeffs), ("external_distortion_coeffs", external_distortion_coeffs)):
        if v is not None:
            raise NotImplementedError(f"{what}: {name} is not supported (pinhole / fisheye / ftheta only)")
    if ftheta_coeffs is not None and camera_model != "ftheta":
        raise NotImplementedError(f"{what}: ftheta_coeffs is not supported with camera_model={camera_model!r} "
                                  "(the FTheta parameters belong to camera_model='ftheta')")
    if camera_model not in _UT_CAMERAS:
        if camera_model in ("ortho", "lidar"):
            raise NotImplementedError(f"{what}: camera_model={camera_model!r} is not supported (pinhole / fisheye / ftheta only)")
        raise ValueError(f"{what}: unknown camera_model {camera_model!r}")
    if camera_model == "ftheta" and ftheta_coeffs is None:
        raise NotImplementedError(f"{what}: camera_model='ftheta' requires ftheta_coeffs (FThetaCameraDistortionParameters)")
    if not global_z_order and camera_model != "ftheta":
        raise NotImplementedError(f"{what}: global_z_order=False is not supported with camera_model={camera_model!r} "
                                  "(the Euclidean depth order is built for ftheta cameras)")
    coeffs, ftheta = [None, None, None], None
    if camera_model == "ftheta":
        for name, v in (("radial_coeffs", radial_coeffs), ("tangential_coeffs", tangential_coeffs),
                        ("thin_prism_coeffs", thin_prism_coeffs)):
            if v is not None:
                raise ValueError(f"{what}: {name} does not apply to the ftheta camera (its distortion is ftheta_coeffs)")
        ftheta = _ftheta_params(what, ftheta_coeffs)
    else:
        if camera_model == "fisheye":
            for name, v in (("tangential_coeffs", tangential_coeffs), ("thin_prism_coeffs", thin_prism_coeffs)):
                if v is not None:
                    raise ValueError(f"{what}: {name} applies to the pinhole camera only")
        widths = (("radial_coeffs", radial_coeffs, 6 if camera_model == "pinhole" else 4),
                  ("tangential_coeffs", tangential_coeffs, 2), ("thin_prism_coeffs", thin_prism_coeffs, 4))
        for i, (name, v, k) in enumerate(widths):
            if v is not None:
                _check_shape(v, tuple(viewmats.shape[:-2]) + (k,), name)
                coeffs[i] = f32c(v, name)

    shutter = _shutter_type(rolling_shutter)
    if shutter == RollingShutterType.GLOBAL:
        if viewmats_rs is not None:
            raise NotImplementedError(f"{what}: viewmats_rs is not supported with the global shutter (rolling_shutter=GLOBAL)")
    else:
        if viewmats_rs is None:
            raise NotImplementedError(f"{what}: rolling_shutter={rolling_shutter!r} requires viewmats_rs, the end-of-frame poses")
        _check_shape(viewmats_rs, tuple(viewmats.shape), "viewmats_rs")
        if viewmats_rs.dtype != torch.float32:
            raise TypeError(f"{what}: viewmats_rs must be float32, got {viewmats_rs.dtype}")
        rows = shutter in (RollingShutterType.ROLLING_TOP_TO_BOTTOM, RollingShutterType.ROLLING_BOTTOM_TO_TOP)
        if (height if rows else width) < 2:
            raise ValueError(f"{what}: rolling_shutter={shutter.name} needs at least two image {'rows' if rows else 'columns'}, "
                             f"got {width}x{height}")
        viewmats_rs = viewmats_rs.detach().contiguous()
    return _UtCamera(_UT_CAMERAS[camera_model], *coeffs, ftheta, int(shutter), viewmats_rs, bool(global_z_order))


def _ut_geometry(what, means, quats, scales, viewmats, Ks) -> tuple:
    if means.dim() < 2 or means.shape[-1] != 3:
        raise ValueError(f"{what}: means must be [..., N, 3], got {tuple(means.shape)}")
    batch, N = tuple(means.shape[:-2]), means.shape[-2]
    _check_shape(quats, batch + (N, 4), "quats")
    _check_shape(scales, batch + (N, 3), "scales")
    if viewmats.dim() != len(batch) + 3:
        raise ValueError(f"{what}: viewmats must be [..., C, 4, 4], got {tuple(viewmats.shape)}")
    C = viewmats.shape[-3]
    _check_shape(viewmats, batch + (C, 4, 4), "viewmats")
    _check_shape(Ks, batch + (C, 3, 3), "Ks")
    for name, t in (("means", means), ("quats", quats), ("scales", scales), ("viewmats", viewmats), ("Ks", Ks)):
        if t.dtype != torch.float32:
            raise TypeError(f"{what}: {name} must be float32, got {t.dtype}")
    return batch, C, N


def fully_fused_projection_with_ut(
    means: Tensor,  # [..., N, 3]
    quats: Tensor,  # [..., N, 4]
    scales: Tensor,  # [..., N, 3]
    opacities: Optional[Tensor],  # [..., N]
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    width: int,
    height: int,
    eps2d: float = 0.3,
    near_plane: float = 0.01,
    far_plane: float = 1e10,
    radius_clip: float = 0.0,
    calc_compensations: bool = False,
    camera_model: str = "pinhole",
    ut_params=None,
    radial_coeffs: Optional[Tensor] = None,  # [..., C, 6] pinhole or [..., C, 4] fisheye
    tangential_coeffs: Optional[Tensor] = None,  # [..., C, 2]
    thin_prism_coeffs: Optional[Tensor] = None,  # [..., C, 4]
    ftheta_coeffs=None,
    lidar_coeffs=None,
    external_distortion_coeffs=None,
    rolling_shutter: int = 4,
    viewmats_rs: Optional[Tensor] = None,
    global_z_order: bool = True,
) -> Tuple[Tensor, Tensor, Tensor, Tensor, Optional[Tensor]]:
    """Projects 3D Gaussians through a distorted pinhole, fisheye or FTheta camera with the unscented transform: 7 sigma points
    per Gaussian are projected through the camera model and reduced to a 2-D mean and covariance, then blurred by
    ``eps2d`` and culled as in ``fully_fused_projection``.  Returns (radii int32 [..., C, N, 2], means2d [..., C, N, 2],
    depths [..., C, N], conics [..., C, N, 3], compensations [..., C, N] or None); culled rows have radii 0 and zero
    floats.  Not differentiable, as in the reference.  ``ut_params``: any object with the fields of the reference's
    UnscentedTransformParameters, or None for their defaults.

    FTheta (``camera_model="ftheta"`` with ``ftheta_coeffs``, an FThetaCameraDistortionParameters shared by every
    camera; the principal point is each camera's Ks (cx, cy) + 0.5): no z > 0 requirement, a sigma point is valid below
    ``max_angle`` inside the image grown by the margin.  ``global_z_order=False`` (FTheta only) culls on and returns the
    distance |mean_c| from the camera centre as the depth, so that tile lists sort by distance, as a lens beyond 180
    degrees needs; True culls and orders on the camera-frame z.

    Rolling shutter: ``rolling_shutter`` (a RollingShutterType or its value) other than GLOBAL with ``viewmats_rs``
    [..., C, 4, 4], the end-of-frame poses.  Each sigma point is projected at the pose of the image row or column it
    lands in (translation lerp and rotation slerp between the two poses at that row's or column's frame time, iterated
    up to 10 times from the start pose's projection); the depths and the near / far cull take the mid-frame pose."""
    what = "fully_fused_projection_with_ut"
    batch, C, N = _ut_geometry(what, means, quats, scales, viewmats, Ks)
    cam = _ut_camera(what, viewmats, width, height, camera_model, radial_coeffs, tangential_coeffs, thin_prism_coeffs,
                     ftheta_coeffs, lidar_coeffs, external_distortion_coeffs, rolling_shutter, viewmats_rs, global_z_order)
    if opacities is not None:
        _check_shape(opacities, batch + (N,), "opacities")
    return _project_ut(means, quats, scales, opacities, viewmats, Ks, width, height, eps2d, near_plane, far_plane,
                       radius_clip, calc_compensations, _ut_params(ut_params), cam)


@torch.no_grad()
def _project_ut(means, quats, scales, opacities, viewmats, Ks, width, height, eps2d, near_plane, far_plane, radius_clip,
                calc_compensations, ut: tuple, cam: _UtCamera):
    """fully_fused_projection_with_ut on checked arguments: ``ut`` from _ut_params, ``cam`` from _ut_camera."""
    batch, C, N = tuple(means.shape[:-2]), viewmats.shape[-3], means.shape[-2]
    alpha, beta, kappa, margin, require_all = ut
    opacities = None if opacities is None else f32c(opacities, "opacities")
    dev = require_cuda(means, quats, scales, viewmats, Ks, opacities, cam.radial, cam.tangential, cam.thin, cam.viewmats_rs)
    means, quats, scales, viewmats, Ks = (t.contiguous() for t in (means, quats, scales, viewmats, Ks))
    o = dict(device=dev, dtype=torch.float32)
    radii = torch.empty(batch + (C, N, 2), device=dev, dtype=torch.int32)
    means2d = torch.empty(batch + (C, N, 2), **o)
    depths = torch.empty(batch + (C, N), **o)
    conics = torch.empty(batch + (C, N, 3), **o)
    comps = torch.empty(batch + (C, N), **o) if calc_compensations else None
    with _Ctx(dev) as st:
        check(
            lib().gsb200_ut_projection_fwd(
                _prod(batch), C, N, ptr(means), ptr(quats), ptr(scales), ptr(opacities), ptr(viewmats), ptr(Ks), cam.model,
                ptr(cam.radial), ptr(cam.tangential), ptr(cam.thin), _ftheta_ptr(cam.ftheta), ptr(cam.viewmats_rs),
                cam.shutter, int(cam.global_z_order), int(width), int(height), float(eps2d), float(near_plane),
                float(far_plane), float(radius_clip), alpha, beta, kappa, margin, int(require_all), ptr(radii),
                ptr(means2d), ptr(depths), ptr(conics), ptr(comps), st,
            ),
            "fully_fused_projection_with_ut",
        )
    return radii, means2d, depths, conics, comps


class _RasterizeToPixelsEval3D(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means, quats, scales, colors, opacities, backgrounds, masks, viewmats, Ks, cam: _UtCamera, width, height,
                isect_offsets, flatten_ids):
        dev = require_cuda(means, quats, scales, colors, opacities, viewmats, Ks)
        means, quats, scales = means.contiguous(), quats.contiguous(), scales.contiguous()
        colors, opacities = f32c(colors, "colors"), f32c(opacities, "opacities")
        backgrounds, viewmats, Ks = f32c(backgrounds, "backgrounds"), viewmats.contiguous(), Ks.contiguous()
        batch, N = tuple(means.shape[:-2]), means.shape[-2]
        B, C, D = _prod(batch), viewmats.shape[-3], colors.shape[-1]
        image_dims = batch + (C,)
        th, tw = isect_offsets.shape[-2:]
        m8 = _mask_u8(masks)
        offsets, fl = isect_offsets.contiguous(), flatten_ids.contiguous()
        S = fl.shape[0]
        o = dict(device=dev, dtype=torch.float32)
        pix = image_dims + (height, width)
        if S == 0:
            # nothing intersects a tile: the background alone, no kernel launch
            if backgrounds is not None:
                render_colors = torch.broadcast_to(backgrounds[..., None, None, :], pix + (D,)).contiguous()
            else:
                render_colors = torch.zeros(pix + (D,), **o)
            render_alphas = torch.zeros(pix + (1,), **o)
            last_ids = torch.full(pix, -1, device=dev, dtype=torch.int32)
        else:
            render_colors = torch.empty(pix + (D,), **o)
            render_alphas = torch.empty(pix + (1,), **o)
            last_ids = torch.empty(pix, device=dev, dtype=torch.int32)
            with _Ctx(dev) as st:
                check(
                    lib().gsb200_eval3d_fwd(
                        B, C, N, D, ptr(means), ptr(quats), ptr(scales), ptr(colors), ptr(opacities), ptr(backgrounds),
                        ptr(m8), ptr(viewmats), ptr(Ks), cam.model, ptr(cam.radial), ptr(cam.tangential), ptr(cam.thin),
                        _ftheta_ptr(cam.ftheta), ptr(cam.viewmats_rs), cam.shutter, width, height, 16, tw, th, ptr(offsets),
                        ptr(fl), S, ptr(render_colors),
                        ptr(render_alphas), ptr(last_ids), st,
                    ),
                    "rasterize_to_pixels_eval3d",
                )
        ctx.save_for_backward(means, quats, scales, colors, opacities, backgrounds, m8, viewmats, Ks, offsets, fl,
                              render_alphas, last_ids)
        ctx.set_materialize_grads(False)
        ctx.meta = (B, C, N, D, cam, width, height, tw, th, S)
        ctx.mark_non_differentiable(last_ids)
        return render_colors, render_alphas

    @staticmethod
    def backward(ctx, v_render_colors, v_render_alphas):
        means, quats, scales, colors, opacities, backgrounds, m8, viewmats, Ks, offsets, fl, render_alphas, last_ids = ctx.saved_tensors
        B, C, N, D, cam, width, height, tw, th, S = ctx.meta
        dev = render_alphas.device
        if v_render_colors is None:
            v_render_colors = torch.zeros(render_alphas.shape[:-1] + (D,), device=dev, dtype=torch.float32)
        v_render_colors = v_render_colors.float().contiguous()
        v_render_alphas = None if v_render_alphas is None else v_render_alphas.float().contiguous()
        v_colors, v_opacities = torch.zeros_like(colors), torch.zeros_like(opacities)
        v_means, v_quats, v_scales = torch.empty_like(means), torch.empty_like(quats), torch.empty_like(scales)
        records = torch.zeros((B * N, 12), device=dev, dtype=torch.float32)
        with _Ctx(dev) as st:
            check(
                lib().gsb200_eval3d_bwd(
                    B, C, N, D, ptr(means), ptr(quats), ptr(scales), ptr(colors), ptr(opacities), ptr(backgrounds), ptr(m8),
                    ptr(viewmats), ptr(Ks), cam.model, ptr(cam.radial), ptr(cam.tangential), ptr(cam.thin),
                    _ftheta_ptr(cam.ftheta), ptr(cam.viewmats_rs), cam.shutter, width, height, 16, tw, th, ptr(offsets),
                    ptr(fl), S, ptr(render_alphas), ptr(last_ids), ptr(v_render_colors), ptr(v_render_alphas),
                    ptr(records), ptr(v_colors), ptr(v_opacities), ptr(v_means), ptr(v_quats), ptr(v_scales), st,
                ),
                "rasterize_to_pixels_eval3d_bwd",
            )
        v_backgrounds = None
        if backgrounds is not None and ctx.needs_input_grad[5]:
            v_backgrounds = (v_render_colors * (1.0 - render_alphas)).sum(dim=(-3, -2))
        # viewmats, Ks and the camera (its coefficients, viewmats_rs) get no gradient, as in the reference's backward
        return (v_means, v_quats, v_scales, v_colors, v_opacities, v_backgrounds) + (None,) * 8


def rasterize_to_pixels_eval3d(
    means: Tensor,  # [..., N, 3]
    quats: Tensor,  # [..., N, 4]
    scales: Tensor,  # [..., N, 3]
    colors: Tensor,  # [..., C, N, channels]
    opacities: Tensor,  # [..., C, N]
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    image_width: int,
    image_height: int,
    tile_size: int,
    isect_offsets: Tensor,  # [..., C, tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    backgrounds: Optional[Tensor] = None,  # [..., C, channels]
    masks: Optional[Tensor] = None,  # [..., C, tile_height, tile_width]
    camera_model: str = "pinhole",
    ut_params=None,
    rays: Optional[Tensor] = None,
    radial_coeffs: Optional[Tensor] = None,  # [..., C, 6] pinhole or [..., C, 4] fisheye
    tangential_coeffs: Optional[Tensor] = None,  # [..., C, 2]
    thin_prism_coeffs: Optional[Tensor] = None,  # [..., C, 4]
    ftheta_coeffs=None,
    lidar_coeffs=None,
    external_distortion_coeffs=None,
    rolling_shutter: int = 4,
    viewmats_rs: Optional[Tensor] = None,
    use_hit_distance: bool = False,
    return_normals: bool = False,
    renderer_config=None,
) -> Tuple[Tensor, Tensor]:
    """Composites depth-sorted Gaussians front to back per 16x16 tile, evaluating each in 3-D along the pixel's
    world-space ray (from the camera model, the distortion inverted by Newton iteration) instead of as a 2-D conic: the
    maximum response along the ray times the opacity is the alpha (min 0.99, skipped below 1/255, stop at T <= 1e-4).
    Returns (render_colors [..., C, H, W, channels], render_alphas [..., C, H, W, 1]).  Differentiable in means, quats,
    scales, colors, opacities and backgrounds; viewmats get no gradient, as in the reference.  ``ut_params`` is accepted
    for the reference's signature and does not enter the compositing.  Dense rows, the MixedBatch renderer only.

    Rolling shutter (``rolling_shutter`` other than GLOBAL with the end-of-frame poses ``viewmats_rs``): the ray of each
    pixel leaves the camera at the pose of the pixel's row or column (translation lerp and rotation slerp between
    ``viewmats`` and ``viewmats_rs`` at its frame time).  viewmats_rs gets no gradient either.

    FTheta (``camera_model="ftheta"`` with ``ftheta_coeffs``): each pixel centre is unprojected through the shared FTheta
    parameters; with the forward polynomial as the reference, a pixel whose Newton inversion does not converge
    composites nothing."""
    what = "rasterize_to_pixels_eval3d"
    for name, v in (("rays", rays),):
        if v is not None:
            raise NotImplementedError(f"{what}: {name} is not supported")
    if use_hit_distance:
        raise NotImplementedError(f"{what}: use_hit_distance=True is not supported")
    if return_normals:
        raise NotImplementedError(f"{what}: return_normals=True is not supported")
    if renderer_config is not None and type(renderer_config).__name__ != "RendererConfig_MixedBatch":
        raise NotImplementedError(f"{what}: renderer_config={renderer_config!r} is not supported (RendererConfig_MixedBatch only)")
    if colors.dim() == 2 or opacities.dim() == 1:
        raise NotImplementedError(f"{what}: packed [nnz, channels] rows are not supported")
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")
    batch, C, N = _ut_geometry(what, means, quats, scales, viewmats, Ks)
    image_dims = batch + (C,)
    cam = _ut_camera(what, viewmats, image_width, image_height, camera_model, radial_coeffs, tangential_coeffs,
                     thin_prism_coeffs, ftheta_coeffs, lidar_coeffs, external_distortion_coeffs, rolling_shutter, viewmats_rs)
    _ut_params(ut_params)
    if colors.dim() != len(image_dims) + 2:
        raise ValueError(f"{what}: colors must be [..., C, N, channels], got {tuple(colors.shape)}")
    D = colors.shape[-1]
    _check_shape(colors, image_dims + (N, D), "colors")
    _check_shape(opacities, image_dims + (N,), "opacities")
    if isect_offsets.dim() != len(image_dims) + 2 or tuple(isect_offsets.shape[:-2]) != image_dims:
        raise ValueError(f"isect_offsets must be {image_dims + ('tile_height', 'tile_width')}, got {tuple(isect_offsets.shape)}")
    th, tw = isect_offsets.shape[-2:]
    if th * 16 < image_height or tw * 16 < image_width:
        raise ValueError(f"isect_offsets tile grid {tw}x{th} does not cover a {image_width}x{image_height} image")
    if backgrounds is not None:
        _check_shape(backgrounds, image_dims + (D,), "backgrounds")
    if masks is not None:
        _check_shape(masks, image_dims + (th, tw), "masks")
    if isect_offsets.dtype != torch.int32 or flatten_ids.dtype != torch.int32 or flatten_ids.dim() != 1:
        raise ValueError("isect_offsets and flatten_ids must be int32, flatten_ids one-dimensional")
    for name, t in (("colors", colors), ("opacities", opacities), ("backgrounds", backgrounds)):
        if t is not None and t.dtype != torch.float32:
            raise TypeError(f"{what}: {name} must be float32, got {t.dtype}")
    if D not in _SUPPORTED_CHANNELS:
        raise NotImplementedError(f"{what}: {D} channels; the eval3d kernels are built for {_SUPPORTED_CHANNELS}")
    return _rasterize_eval3d(means, quats, scales, colors, opacities, viewmats, Ks, image_width, image_height,
                             isect_offsets, flatten_ids, backgrounds, masks, cam)


def _rasterize_eval3d(means, quats, scales, colors, opacities, viewmats, Ks, width, height, isect_offsets, flatten_ids,
                      backgrounds, masks, cam: _UtCamera):
    """rasterize_to_pixels_eval3d on checked arguments: ``cam`` from _ut_camera."""
    require_cuda(means, quats, scales, colors, opacities, viewmats, Ks, backgrounds, masks, isect_offsets, flatten_ids,
                 cam.radial, cam.tangential, cam.thin, cam.viewmats_rs)
    return _RasterizeToPixelsEval3D.apply(means, quats, scales, colors, opacities, backgrounds, masks, viewmats, Ks, cam,
                                          int(width), int(height), isect_offsets, flatten_ids)


class _RasterizeToPixelsEval3DSparse(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means, quats, scales, colors, opacities, backgrounds, masks, viewmats, Ks, cam: _UtCamera, width, height,
                tile_width, tile_height, image_ids, active_tiles, tile_offsets, flatten_ids, tile_pixel_mask,
                tile_pixel_cumsum, pixel_map):
        dev = require_cuda(means, quats, scales, colors, opacities, viewmats, Ks, active_tiles, tile_offsets, flatten_ids,
                           pixel_map)
        means, quats, scales = means.contiguous(), quats.contiguous(), scales.contiguous()
        colors, opacities = f32c(colors, "colors"), f32c(opacities, "opacities")
        backgrounds, viewmats, Ks = f32c(backgrounds, "backgrounds"), viewmats.contiguous(), Ks.contiguous()
        B, C, N, D = _prod(means.shape[:-2]), viewmats.shape[-3], means.shape[-2], colors.shape[-1]
        m8 = _mask_u8(masks)
        active, offsets, fl = active_tiles.contiguous(), tile_offsets.contiguous(), flatten_ids.contiguous()
        words, cumsum, pmap = tile_pixel_mask.contiguous(), tile_pixel_cumsum.contiguous(), pixel_map.contiguous()
        AT, S, P = active.shape[0], fl.shape[0], pmap.shape[0]
        o = dict(device=dev, dtype=torch.float32)
        if P == 0 or S == 0 or AT == 0:
            # no requested pixel, or nothing listed in any active tile: the background alone, no kernel launch
            if backgrounds is not None and P > 0:
                render_colors = backgrounds[image_ids.long()]
            else:
                render_colors = torch.zeros((P, D), **o)
            render_alphas = torch.zeros((P, 1), **o)
            last_ids = torch.full((P,), -1, device=dev, dtype=torch.int32)
        else:
            render_colors, render_alphas = torch.empty((P, D), **o), torch.empty((P, 1), **o)
            last_ids = torch.empty(P, device=dev, dtype=torch.int32)
            with _Ctx(dev) as st:
                check(
                    lib().gsb200_eval3d_sparse_fwd(
                        B, C, N, D, ptr(means), ptr(quats), ptr(scales), ptr(colors), ptr(opacities), ptr(backgrounds),
                        ptr(m8), ptr(viewmats), ptr(Ks), cam.model, ptr(cam.radial), ptr(cam.tangential), ptr(cam.thin),
                        _ftheta_ptr(cam.ftheta), ptr(cam.viewmats_rs), cam.shutter, width, height, 16, tile_width,
                        tile_height, AT, ptr(active), ptr(offsets), ptr(fl), S, ptr(words), ptr(cumsum), ptr(pmap),
                        ptr(render_colors), ptr(render_alphas), ptr(last_ids), st,
                    ),
                    "rasterize_to_pixels_eval3d_sparse",
                )
        ctx.save_for_backward(means, quats, scales, colors, opacities, backgrounds, m8, viewmats, Ks, image_ids, active,
                              offsets, fl, words, cumsum, pmap, render_alphas, last_ids)
        ctx.set_materialize_grads(False)
        ctx.meta = (B, C, N, D, cam, width, height, tile_width, tile_height)
        return render_colors, render_alphas

    @staticmethod
    def backward(ctx, v_render_colors, v_render_alphas):
        (means, quats, scales, colors, opacities, backgrounds, m8, viewmats, Ks, image_ids, active, offsets, fl, words,
         cumsum, pmap, render_alphas, last_ids) = ctx.saved_tensors
        B, C, N, D, cam, width, height, tw, th = ctx.meta
        dev = render_alphas.device
        if v_render_colors is None:
            v_render_colors = torch.zeros((pmap.shape[0], D), device=dev, dtype=torch.float32)
        v_render_colors = v_render_colors.float().contiguous()
        v_render_alphas = None if v_render_alphas is None else v_render_alphas.float().contiguous()
        v_colors, v_opacities = torch.zeros_like(colors), torch.zeros_like(opacities)
        if fl.shape[0] == 0 or pmap.shape[0] == 0 or active.shape[0] == 0:
            # nothing was composited: zero gradients, no kernel launch
            v_means, v_quats, v_scales = torch.zeros_like(means), torch.zeros_like(quats), torch.zeros_like(scales)
        else:
            v_means, v_quats, v_scales = torch.empty_like(means), torch.empty_like(quats), torch.empty_like(scales)
            records = torch.zeros((B * N, 12), device=dev, dtype=torch.float32)
            with _Ctx(dev) as st:
                check(
                    lib().gsb200_eval3d_sparse_bwd(
                        B, C, N, D, ptr(means), ptr(quats), ptr(scales), ptr(colors), ptr(opacities), ptr(backgrounds),
                        ptr(m8), ptr(viewmats), ptr(Ks), cam.model, ptr(cam.radial), ptr(cam.tangential), ptr(cam.thin),
                        _ftheta_ptr(cam.ftheta), ptr(cam.viewmats_rs), cam.shutter, width, height, 16, tw, th,
                        active.shape[0], ptr(active), ptr(offsets), ptr(fl), fl.shape[0], ptr(words), ptr(cumsum),
                        ptr(pmap), ptr(render_alphas), ptr(last_ids), ptr(v_render_colors), ptr(v_render_alphas),
                        ptr(records), ptr(v_colors), ptr(v_opacities), ptr(v_means), ptr(v_quats), ptr(v_scales), st,
                    ),
                    "rasterize_to_pixels_eval3d_sparse_bwd",
                )
        v_backgrounds = None
        if backgrounds is not None and ctx.needs_input_grad[5]:
            v_backgrounds = torch.zeros_like(backgrounds).index_add_(0, image_ids.long(), v_render_colors * (1.0 - render_alphas))
        # viewmats, Ks and the camera (its coefficients, viewmats_rs) get no gradient, as in rasterize_to_pixels_eval3d
        return (v_means, v_quats, v_scales, v_colors, v_opacities, v_backgrounds) + (None,) * 15


def rasterize_to_pixels_eval3d_sparse(
    means: Tensor,  # [..., N, 3]
    quats: Tensor,  # [..., N, 4]
    scales: Tensor,  # [..., N, 3]
    colors: Tensor,  # [..., C, N, channels]
    opacities: Tensor,  # [..., C, N]
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    image_ids: Tensor,  # [P]
    active_tiles: Tensor,  # [AT]
    tile_offsets: Tensor,  # [AT + 1]
    flatten_ids: Tensor,  # [n_isects]
    tile_pixel_mask: Tensor,  # [AT, 4]
    tile_pixel_cumsum: Tensor,  # [AT]
    pixel_map: Tensor,  # [P]
    image_width: int,
    image_height: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
    backgrounds: Optional[Tensor] = None,  # [n_images, channels]
    masks: Optional[Tensor] = None,  # [n_images, tile_height, tile_width]
    camera_model: str = "pinhole",
    ut_params=None,
    radial_coeffs: Optional[Tensor] = None,  # [..., C, 6] pinhole or [..., C, 4] fisheye
    tangential_coeffs: Optional[Tensor] = None,  # [..., C, 2]
    thin_prism_coeffs: Optional[Tensor] = None,  # [..., C, 4]
    ftheta_coeffs=None,
    rolling_shutter: int = RollingShutterType.GLOBAL,
    viewmats_rs: Optional[Tensor] = None,  # [..., C, 4, 4]
) -> Tuple[Tensor, Tensor]:
    """rasterize_to_pixels_eval3d at the pixels of a build_sparse_tile_layout layout only, with the lists of
    isect_tiles_sparse (conics=None) on the UT rows of fully_fused_projection_with_ut.  The geometry, colours,
    opacities, cameras and camera arguments are those of rasterize_to_pixels_eval3d; the images are its (batch, camera)
    images flattened: image ``i`` of the layout is camera ``i % C`` of batch ``i // C``.  ``backgrounds`` is
    [n_images, channels] and ``masks`` [n_images, tile_height, tile_width], as in the other sparse ops.  Returns
    (render_colors [P, channels], render_alphas [P, 1]) in the original pixel order.  Differentiable in means, quats,
    scales, colors, opacities and backgrounds; viewmats, ``viewmats_rs`` and the camera coefficients get no gradient.

    - A requested pixel inside the W x H image gets the value rasterize_to_pixels_eval3d gives it, bit for bit, for the
      same rows, lists, camera and shutter.
    - A requested pixel in the margin of a partial tile (inside the tile grid, outside the image) gets the background
      (or 0) and alpha 0, and passes no gradient to the Gaussians; its colour cotangent goes to its background.
      rasterize_to_pixels_sparse and rasterize_to_pixels_2dgs_sparse render such pixels, but an eval3d pixel's ray comes
      from the camera model and its rolling-shutter frame time is defined on the W x H image, and the dense op has no
      such pixel to agree with.
    - An FTheta pixel whose unprojection does not converge composites nothing, as in the dense op.

    ``ut_params`` is checked and does not enter the compositing.  With no requested pixel, or no Gaussian listed in any
    active tile, nothing is launched: the background (or 0) with alpha 0, and zero gradients."""
    what = "rasterize_to_pixels_eval3d_sparse"
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")
    _check_sparse_layout(
        image_ids, active_tiles, tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map, image_width,
        image_height, tile_width, tile_height,
    )
    if flatten_ids.dim() != 1:
        raise ValueError(f"flatten_ids must be one-dimensional, got {tuple(flatten_ids.shape)}")
    batch, C, N = _ut_geometry(what, means, quats, scales, viewmats, Ks)
    image_dims = batch + (C,)
    n_images = _prod(image_dims)
    cam = _ut_camera(what, viewmats, image_width, image_height, camera_model, radial_coeffs, tangential_coeffs,
                     thin_prism_coeffs, ftheta_coeffs, None, None, rolling_shutter, viewmats_rs)
    _ut_params(ut_params)
    if colors.dim() != len(image_dims) + 2:
        raise ValueError(f"{what}: colors must be [..., C, N, channels], got {tuple(colors.shape)}")
    D = colors.shape[-1]
    _check_shape(colors, image_dims + (N, D), "colors")
    _check_shape(opacities, image_dims + (N,), "opacities")
    if backgrounds is not None:
        _check_shape(backgrounds, (n_images, D), "backgrounds")
    if masks is not None:
        _check_shape(masks, (n_images, tile_height, tile_width), "masks")
    for name, t in (("colors", colors), ("opacities", opacities), ("backgrounds", backgrounds)):
        if t is not None and t.dtype != torch.float32:
            raise TypeError(f"{what}: {name} must be float32, got {t.dtype}")
    if D not in _SUPPORTED_CHANNELS:
        raise NotImplementedError(f"{what}: {D} channels; the eval3d kernels are built for {_SUPPORTED_CHANNELS}")
    require_cuda(means, quats, scales, colors, opacities, viewmats, Ks, backgrounds, masks, image_ids, active_tiles,
                 tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum, pixel_map, cam.radial, cam.tangential,
                 cam.thin, cam.viewmats_rs)
    return _RasterizeToPixelsEval3DSparse.apply(
        means, quats, scales, colors, opacities, backgrounds, masks, viewmats, Ks, cam, int(image_width),
        int(image_height), int(tile_width), int(tile_height), image_ids, active_tiles, tile_offsets, flatten_ids,
        tile_pixel_mask, tile_pixel_cumsum, pixel_map,
    )


# --------------------------------------------------------------------------------------------
# 3DGUT pair query and per-pixel contributor queries (the reference has none): the pairs rasterize_to_pixels_eval3d
# composites, from the walk of csrc/indices.cuh (pair_walk_kernel with csrc/ut.cu's Eval3dModel) with the forward's
# rays, responses and stop rule.  The contributor forms are those of the 3DGS / 2DGS queries over that walk, with the
# geometry and cameras of rasterize_to_pixels_eval3d in place of 2-D rows.

@torch.no_grad()
def rasterize_to_indices_in_range_eval3d(
    range_start: int,
    range_end: int,
    transmittances: Tensor,  # [..., C, image_height, image_width]
    means: Tensor,  # [..., N, 3]
    quats: Tensor,  # [..., N, 4]
    scales: Tensor,  # [..., N, 3]
    opacities: Tensor,  # [..., C, N]
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    image_width: int,
    image_height: int,
    tile_size: int,
    isect_offsets: Tensor,  # [..., C, tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    camera_model: str = "pinhole",
    radial_coeffs: Optional[Tensor] = None,  # [..., C, 6] pinhole or [..., C, 4] fisheye
    tangential_coeffs: Optional[Tensor] = None,  # [..., C, 2]
    thin_prism_coeffs: Optional[Tensor] = None,  # [..., C, 4]
    ftheta_coeffs=None,
    rolling_shutter: int = RollingShutterType.GLOBAL,
    viewmats_rs: Optional[Tensor] = None,  # [..., C, 4, 4]
) -> Tuple[Tensor, Tensor, Tensor]:
    """``rasterize_to_indices_in_range`` for 3DGUT: the (gaussian, pixel) pairs ``rasterize_to_pixels_eval3d``
    composites when every pixel starts from its transmittance and walks only the batches ``[range_start, range_end)``
    of 256 Gaussians of its tile's list, with the forward's own decisions (the pixel's ray through the camera model and
    shutter, the largest response along it, the stop at T <= 1e-4).  A pixel whose ray cannot be unprojected (an FTheta
    pixel whose inversion does not converge) has no pairs.  Dense rows only.  Returns int64 ``(gaussian_ids, pixel_ids,
    image_ids)`` [M], ordered as ``rasterize_to_indices_in_range``'s; ``image_ids`` index the flattened (batch,
    camera) images."""
    what = "rasterize_to_indices_in_range_eval3d"
    rs, re_ = _batch_index(range_start, "range_start"), _batch_index(range_end, "range_end")
    W, H = int(image_width), int(image_height)
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")
    rows = _Eval3dRows(what, means, quats, scales, opacities, viewmats, Ks, W, H, camera_model, radial_coeffs,
                       tangential_coeffs, thin_prism_coeffs, ftheta_coeffs, rolling_shutter, viewmats_rs)
    if isect_offsets.dim() < 2:
        raise ValueError(f"isect_offsets must be [..., C, tile_height, tile_width], got {tuple(isect_offsets.shape)}")
    image_dims = tuple(isect_offsets.shape[:-2])
    N = rows.check(image_dims)
    _check_shape(transmittances, image_dims + (H, W), "transmittances")
    th, tw = isect_offsets.shape[-2:]
    if th * 16 < H or tw * 16 < W:
        raise ValueError(f"isect_offsets tile grid {tw}x{th} does not cover a {W}x{H} image")
    if flatten_ids.dim() != 1:
        raise ValueError(f"flatten_ids must be one-dimensional, got {tuple(flatten_ids.shape)}")
    if isect_offsets.dtype != torch.int32 or flatten_ids.dtype != torch.int32:
        raise TypeError("isect_offsets and flatten_ids must be int32")
    _contrib_dtypes(rows.floats() + ((transmittances, "transmittances"),), ())
    dev = require_cuda(*rows.tensors(), transmittances, isect_offsets, flatten_ids)
    S, P = flatten_ids.shape[0], _prod(image_dims) * H * W
    if N == 0 or S == 0 or P == 0 or re_ <= rs:
        return tuple(torch.empty(0, device=dev, dtype=torch.int64) for _ in range(3))
    head, keep = rows.head(_prod(image_dims), N)
    tr, off, fl = transmittances.contiguous(), isect_offsets.contiguous(), flatten_ids.contiguous()
    args = head + (ptr(tr), W, H, 16, tw, th, ptr(off), ptr(fl), S, rs, re_)
    return _index_passes(what, "gsb200_eval3d_indices", args, P, dev)


@torch.no_grad()
def rasterize_num_contributing_gaussians_eval3d(
    means: Tensor,  # [..., N, 3]
    quats: Tensor,  # [..., N, 4]
    scales: Tensor,  # [..., N, 3]
    opacities: Tensor,  # [..., C, N]
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    tile_offsets: Tensor,  # [..., C, tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    image_width: int,
    image_height: int,
    tile_size: int,
    camera_model: str = "pinhole",
    radial_coeffs: Optional[Tensor] = None,  # [..., C, 6] pinhole or [..., C, 4] fisheye
    tangential_coeffs: Optional[Tensor] = None,  # [..., C, 2]
    thin_prism_coeffs: Optional[Tensor] = None,  # [..., C, 4]
    ftheta_coeffs=None,
    rolling_shutter: int = RollingShutterType.GLOBAL,
    viewmats_rs: Optional[Tensor] = None,  # [..., C, 4, 4]
) -> Tuple[Tensor, Tensor]:
    """``rasterize_num_contributing_gaussians`` for 3DGUT: per pixel, the number of Gaussians
    ``rasterize_to_pixels_eval3d`` composites and its accumulated alpha, equal to its ``render_alphas`` bit for bit for
    the same Gaussians, cameras and lists (after ``rasterization(..., with_ut=True, with_eval3d=True)``: its
    ``meta["opacities"]``, ``meta["isect_offsets"]`` and ``meta["flatten_ids"]``).  A pixel that composites nothing
    (an FTheta pixel whose unprojection does not converge) has count 0 and alpha 0.  Returns (counts int32 [..., C, H,
    W], alphas float32 [..., C, H, W])."""
    what = "rasterize_num_contributing_gaussians_eval3d"
    rows = _Eval3dRows(what, means, quats, scales, opacities, viewmats, Ks, image_width, image_height, camera_model,
                       radial_coeffs, tangential_coeffs, thin_prism_coeffs, ftheta_coeffs, rolling_shutter, viewmats_rs)
    checked = _contrib_dense(rows, tile_offsets, flatten_ids, image_width, image_height, tile_size)
    return _contrib_count(what, checked)


@torch.no_grad()
def rasterize_num_contributing_gaussians_eval3d_sparse(
    means: Tensor,  # [..., N, 3]
    quats: Tensor,  # [..., N, 4]
    scales: Tensor,  # [..., N, 3]
    opacities: Tensor,  # [..., C, N]
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    active_tiles: Tensor,  # [AT]
    tile_offsets: Tensor,  # [AT + 1]
    flatten_ids: Tensor,  # [n_isects]
    tile_pixel_mask: Tensor,  # [AT, 4]
    tile_pixel_cumsum: Tensor,  # [AT]
    pixel_map: Tensor,  # [P]
    image_width: int,
    image_height: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
    camera_model: str = "pinhole",
    radial_coeffs: Optional[Tensor] = None,  # [..., C, 6] pinhole or [..., C, 4] fisheye
    tangential_coeffs: Optional[Tensor] = None,  # [..., C, 2]
    thin_prism_coeffs: Optional[Tensor] = None,  # [..., C, 4]
    ftheta_coeffs=None,
    rolling_shutter: int = RollingShutterType.GLOBAL,
    viewmats_rs: Optional[Tensor] = None,  # [..., C, 4, 4]
) -> Tuple[Tensor, Tensor]:
    """``rasterize_num_contributing_gaussians_eval3d`` at the pixels of a build_sparse_tile_layout layout, with the lists
    of isect_tiles_sparse (conics=None) on the UT rows, as rasterize_to_pixels_eval3d_sparse takes them.  A requested
    pixel in the margin of a partial tile composites nothing (count 0, alpha 0), as in that op.  Returns (counts int32
    [P], alphas float32 [P]) in the original pixel order."""
    what = "rasterize_num_contributing_gaussians_eval3d_sparse"
    rows = _Eval3dRows(what, means, quats, scales, opacities, viewmats, Ks, image_width, image_height, camera_model,
                       radial_coeffs, tangential_coeffs, thin_prism_coeffs, ftheta_coeffs, rolling_shutter, viewmats_rs)
    checked = _contrib_sparse(rows, active_tiles, tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum,
                              pixel_map, image_width, image_height, tile_size, tile_width, tile_height)
    return _contrib_count(what, checked)


@torch.no_grad()
def rasterize_contributing_gaussian_ids_eval3d(
    means: Tensor,  # [..., N, 3]
    quats: Tensor,  # [..., N, 4]
    scales: Tensor,  # [..., N, 3]
    opacities: Tensor,  # [..., C, N]
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    tile_offsets: Tensor,  # [..., C, tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    image_width: int,
    image_height: int,
    tile_size: int,
    num_contributing_gaussians: Tensor,  # [..., C, image_height, image_width] int32
    camera_model: str = "pinhole",
    radial_coeffs: Optional[Tensor] = None,  # [..., C, 6] pinhole or [..., C, 4] fisheye
    tangential_coeffs: Optional[Tensor] = None,  # [..., C, 2]
    thin_prism_coeffs: Optional[Tensor] = None,  # [..., C, 4]
    ftheta_coeffs=None,
    rolling_shutter: int = RollingShutterType.GLOBAL,
    viewmats_rs: Optional[Tensor] = None,  # [..., C, 4, 4]
) -> Tuple[Tensor, Tensor]:
    """Every Gaussian each pixel composites in ``rasterize_to_pixels_eval3d``, front to back, with its weight
    ``alpha * T`` (T before it).  Returns (ids int32, weights float32) [..., C, H, W, K] with K =
    ``num_contributing_gaussians.max()`` (read back to the host once): a pixel's first K pairs (later ones are
    dropped), then -1 / 0.  Ids index N."""
    what = "rasterize_contributing_gaussian_ids_eval3d"
    rows = _Eval3dRows(what, means, quats, scales, opacities, viewmats, Ks, image_width, image_height, camera_model,
                       radial_coeffs, tangential_coeffs, thin_prism_coeffs, ftheta_coeffs, rolling_shutter, viewmats_rs)
    checked = _contrib_dense(rows, tile_offsets, flatten_ids, image_width, image_height, tile_size,
                             num_contributing_gaussians)
    return _contrib_ids(what, checked, num_contributing_gaussians)


@torch.no_grad()
def rasterize_contributing_gaussian_ids_eval3d_sparse(
    means: Tensor,  # [..., N, 3]
    quats: Tensor,  # [..., N, 4]
    scales: Tensor,  # [..., N, 3]
    opacities: Tensor,  # [..., C, N]
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    active_tiles: Tensor,  # [AT]
    tile_offsets: Tensor,  # [AT + 1]
    flatten_ids: Tensor,  # [n_isects]
    tile_pixel_mask: Tensor,  # [AT, 4]
    tile_pixel_cumsum: Tensor,  # [AT]
    pixel_map: Tensor,  # [P]
    num_contributing_gaussians: Tensor,  # [P] int32
    image_width: int,
    image_height: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
    camera_model: str = "pinhole",
    radial_coeffs: Optional[Tensor] = None,  # [..., C, 6] pinhole or [..., C, 4] fisheye
    tangential_coeffs: Optional[Tensor] = None,  # [..., C, 2]
    thin_prism_coeffs: Optional[Tensor] = None,  # [..., C, 4]
    ftheta_coeffs=None,
    rolling_shutter: int = RollingShutterType.GLOBAL,
    viewmats_rs: Optional[Tensor] = None,  # [..., C, 4, 4]
) -> Tuple[Tensor, Tensor]:
    """``rasterize_contributing_gaussian_ids_eval3d`` at the pixels of a sparse layout: (ids, weights) [P, K] in the
    original pixel order."""
    what = "rasterize_contributing_gaussian_ids_eval3d_sparse"
    rows = _Eval3dRows(what, means, quats, scales, opacities, viewmats, Ks, image_width, image_height, camera_model,
                       radial_coeffs, tangential_coeffs, thin_prism_coeffs, ftheta_coeffs, rolling_shutter, viewmats_rs)
    checked = _contrib_sparse(rows, active_tiles, tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum,
                              pixel_map, image_width, image_height, tile_size, tile_width, tile_height,
                              num_contributing_gaussians)
    return _contrib_ids(what, checked, num_contributing_gaussians)


@torch.no_grad()
def rasterize_top_contributing_gaussian_ids_eval3d(
    means: Tensor,  # [..., N, 3]
    quats: Tensor,  # [..., N, 4]
    scales: Tensor,  # [..., N, 3]
    opacities: Tensor,  # [..., C, N]
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    tile_offsets: Tensor,  # [..., C, tile_height, tile_width]
    flatten_ids: Tensor,  # [n_isects]
    image_width: int,
    image_height: int,
    tile_size: int,
    num_depth_samples: int,
    camera_model: str = "pinhole",
    radial_coeffs: Optional[Tensor] = None,  # [..., C, 6] pinhole or [..., C, 4] fisheye
    tangential_coeffs: Optional[Tensor] = None,  # [..., C, 2]
    thin_prism_coeffs: Optional[Tensor] = None,  # [..., C, 4]
    ftheta_coeffs=None,
    rolling_shutter: int = RollingShutterType.GLOBAL,
    viewmats_rs: Optional[Tensor] = None,  # [..., C, 4, 4]
) -> Tuple[Tensor, Tensor]:
    """The ``num_depth_samples`` heaviest Gaussians of each pixel of ``rasterize_to_pixels_eval3d`` by ``alpha * T``,
    front to back: (ids int32, weights float32) [..., C, H, W, K], -1 / 0 in unused slots, by the rule of
    ``rasterize_top_contributing_gaussian_ids``.  K must lie in [1, the eval3d walk's bound on the device], one bound
    for every camera and shutter; outside it a ValueError is raised before anything runs."""
    what = "rasterize_top_contributing_gaussian_ids_eval3d"
    K = _depth_samples(num_depth_samples)
    rows = _Eval3dRows(what, means, quats, scales, opacities, viewmats, Ks, image_width, image_height, camera_model,
                       radial_coeffs, tangential_coeffs, thin_prism_coeffs, ftheta_coeffs, rolling_shutter, viewmats_rs)
    checked = _contrib_dense(rows, tile_offsets, flatten_ids, image_width, image_height, tile_size)
    return _contrib_top(what, checked, K)


@torch.no_grad()
def rasterize_top_contributing_gaussian_ids_eval3d_sparse(
    means: Tensor,  # [..., N, 3]
    quats: Tensor,  # [..., N, 4]
    scales: Tensor,  # [..., N, 3]
    opacities: Tensor,  # [..., C, N]
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    active_tiles: Tensor,  # [AT]
    tile_offsets: Tensor,  # [AT + 1]
    flatten_ids: Tensor,  # [n_isects]
    tile_pixel_mask: Tensor,  # [AT, 4]
    tile_pixel_cumsum: Tensor,  # [AT]
    pixel_map: Tensor,  # [P]
    image_width: int,
    image_height: int,
    tile_size: int,
    tile_width: int,
    tile_height: int,
    num_depth_samples: int,
    camera_model: str = "pinhole",
    radial_coeffs: Optional[Tensor] = None,  # [..., C, 6] pinhole or [..., C, 4] fisheye
    tangential_coeffs: Optional[Tensor] = None,  # [..., C, 2]
    thin_prism_coeffs: Optional[Tensor] = None,  # [..., C, 4]
    ftheta_coeffs=None,
    rolling_shutter: int = RollingShutterType.GLOBAL,
    viewmats_rs: Optional[Tensor] = None,  # [..., C, 4, 4]
) -> Tuple[Tensor, Tensor]:
    """``rasterize_top_contributing_gaussian_ids_eval3d`` at the pixels of a sparse layout: (ids, weights) [P, K] in
    the original pixel order."""
    what = "rasterize_top_contributing_gaussian_ids_eval3d_sparse"
    K = _depth_samples(num_depth_samples)
    rows = _Eval3dRows(what, means, quats, scales, opacities, viewmats, Ks, image_width, image_height, camera_model,
                       radial_coeffs, tangential_coeffs, thin_prism_coeffs, ftheta_coeffs, rolling_shutter, viewmats_rs)
    checked = _contrib_sparse(rows, active_tiles, tile_offsets, flatten_ids, tile_pixel_mask, tile_pixel_cumsum,
                              pixel_map, image_width, image_height, tile_size, tile_width, tile_height)
    return _contrib_top(what, checked, K)
