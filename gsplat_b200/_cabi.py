"""ctypes binding of libgsplat_b200.so (the C ABI declared in include/gsplat_b200.h).

The library is the only compute path: if it cannot be loaded this module raises -- there is no
PyTorch / CPU fallback (tests would otherwise pass on a silent eager path).
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgsplat_b200.so")

_lib = None

c_i64, c_u32, c_int, c_f32, c_vp, c_sz = (
    ctypes.c_int64,
    ctypes.c_uint32,
    ctypes.c_int,
    ctypes.c_float,
    ctypes.c_void_p,
    ctypes.c_size_t,
)

class FThetaParams(ctypes.Structure):
    """gsb200_ftheta_params of include/gsplat_b200.h: the FTheta camera parameters of the 3DGUT entry points."""

    _fields_ = [
        ("reference_poly", ctypes.c_int),
        ("pixeldist_to_angle_poly", ctypes.c_float * 6),
        ("angle_to_pixeldist_poly", ctypes.c_float * 6),
        ("max_angle", ctypes.c_float),
        ("linear_cde", ctypes.c_float * 3),
    ]


# name -> (restype, argtypes) ; mirrors include/gsplat_b200.h one to one
_SIGNATURES = {
    "gsb200_version": (ctypes.c_char_p, []),
    "gsb200_source_hash": (ctypes.c_char_p, []),
    "gsb200_error_string": (ctypes.c_char_p, [c_int]),
    "gsb200_last_cuda_error": (ctypes.c_char_p, []),
    "gsb200_bits_for_count": (c_u32, [c_i64]),
    "gsb200_raster_supports_channels": (c_int, [c_int]),
    "gsb200_quat_scale_to_covar_preci_fwd": (c_int, [c_i64, c_vp, c_vp, c_int, c_vp, c_vp, c_vp]),
    "gsb200_quat_scale_to_covar_preci_bwd": (c_int, [c_i64, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "gsb200_projection_fwd": (
        c_int,
        [c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_f32, c_f32, c_f32, c_f32, c_int,
         c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_projection_bwd": (
        c_int,
        [c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_f32, c_int, c_vp, c_vp, c_vp,
         c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_sh_fwd": (c_int, [c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "gsb200_sh_bwd": (c_int, [c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "gsb200_project_sh_fwd": (
        c_int,
        [c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_f32, c_f32, c_f32, c_f32,
         c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_project_sh_bwd": (
        c_int,
        [c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_f32, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_sh_rows_fwd": (c_int, [c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "gsb200_sh_rows_bwd": (
        c_int, [c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_projection_packed_workspace_bytes": (c_sz, [c_i64, c_i64, c_i64]),
    "gsb200_projection_packed_count": (
        c_int,
        [c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_f32, c_f32, c_f32, c_f32, c_int, c_int,
         c_vp, c_sz, c_vp, c_vp],
    ),
    "gsb200_projection_packed_emit": (
        c_int,
        [c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_f32, c_f32, c_f32, c_f32, c_int,
         c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_projection_packed_bwd": (
        c_int,
        [c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_f32, c_int, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_isect_scan_workspace_bytes": (c_sz, [c_i64]),
    "gsb200_isect_count": (c_int, [c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "gsb200_isect_emit": (c_int, [c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_vp, c_vp, c_vp]),
    "gsb200_l1_loss_workspace_bytes": (c_sz, []),
    "gsb200_l1_loss_fwd": (c_int, [c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "gsb200_l1_loss_bwd": (c_int, [c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "gsb200_ssim_workspace_bytes": (c_sz, [c_i64, c_i64, c_i64, c_i64]),
    "gsb200_ssim_fwd": (c_int, [c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "gsb200_ssim_bwd": (c_int, [c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "gsb200_adam": (c_int, [c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_f32, c_f32, c_f32, c_f32, c_vp]),
    "gsb200_nvls_allreduce_f32": (c_int, [c_vp, c_i64, c_int, c_int, c_vp, c_i64, c_int, c_vp]),
    "gsb200_p2p_allreduce_f32": (c_int, [c_vp, c_i64, c_int, c_int, c_vp, c_i64, c_int, c_vp]),
    "gsb200_rows_allreduce_f32": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_i64, c_i64, c_int, c_int, c_vp, c_i64, c_int, c_vp, c_vp]),
    "gsb200_isect_count_totals": (c_int, [c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_vp, c_vp, c_vp]),
    "gsb200_project_sh_fwd_rows": (
        c_int,
        [c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_f32, c_f32, c_f32, c_f32, c_u32,
         c_u32, c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_raster_fwd_rows": (
        c_int,
        [c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_publish_totals": (c_int, [c_vp, c_vp, c_i64, c_vp]),
    "gsb200_isect_sorted_workspace_bytes": (c_sz, [c_i64, c_i64, c_i64, c_i64, c_int, c_u32, c_u32]),
    "gsb200_isect_sorted": (
        c_int,
        [c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_vp,
         c_vp, c_vp, c_vp, c_sz, c_vp],
    ),
    "gsb200_isect_ids_from_tilekeys": (c_int, [c_i64, c_int, c_vp, c_vp, c_vp, c_i64, c_u32, c_u32, c_vp, c_vp]),
    "gsb200_isect_offsets": (c_int, [c_i64, c_vp, c_i64, c_u32, c_u32, c_vp, c_vp]),
    "gsb200_relocation": (c_int, [c_i64, c_vp, c_vp, c_vp, c_vp, c_int, c_f32, c_vp, c_vp, c_vp]),
    "gsb200_mcmc_perturb_positions": (c_int, [c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_f32, c_f32, c_f32, c_vp]),
    "gsb200_raster_records_bytes": (c_sz, [c_i64, c_int, c_i64]),
    "gsb200_raster_pack": (c_int, [c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "gsb200_raster_fwd": (
        c_int,
        [c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64,
         c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_raster_bwd": (
        c_int,
        [c_i64, c_i64, c_int, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_int, c_vp, c_vp],
    ),
    "gsb200_sparse_layout_workspace_bytes": (c_sz, [c_i64, c_i64, c_u32, c_u32]),
    "gsb200_sparse_layout_sort": (c_int, [c_i64, c_vp, c_vp, c_i64, c_u32, c_u32, c_u32, c_vp, c_sz, c_vp, c_vp]),
    "gsb200_sparse_layout_finish": (c_int, [c_i64, c_i64, c_u32, c_u32, c_i64, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "gsb200_isect_active_offsets": (c_int, [c_i64, c_vp, c_i64, c_u32, c_u32, c_vp, c_i64, c_vp, c_vp]),
    "gsb200_raster_sparse_fwd": (
        c_int,
        [c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp,
         c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_raster_sparse_bwd": (
        c_int,
        [c_i64, c_int, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp],
    ),
    "gsb200_surfel_projection_fwd": (
        c_int,
        [c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_f32, c_f32, c_f32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_surfel_projection_bwd": (
        c_int,
        [c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_surfel_raster_fwd": (
        c_int,
        [c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64,
         c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_surfel_raster_bwd": (
        c_int,
        [c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64,
         c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_surfel_raster_sparse_fwd": (
        c_int,
        [c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_i64, c_vp, c_vp, c_vp,
         c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_surfel_raster_sparse_bwd": (
        c_int,
        [c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_i64, c_vp, c_vp, c_vp,
         c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_vp],
    ),
    "gsb200_indices_workspace_bytes": (c_sz, [c_i64]),
    "gsb200_raster_indices": (
        c_int,
        [c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_vp,
         c_sz, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_surfel_indices": (
        c_int,
        [c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_vp,
         c_sz, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_contrib_max_samples": (c_int, []),
    "gsb200_contrib_count": (
        c_int,
        [c_i64, c_i64, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_vp, c_vp],
    ),
    "gsb200_contrib_ids": (
        c_int,
        [c_i64, c_i64, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp,
         c_int, c_vp, c_vp, c_vp],
    ),
    "gsb200_contrib_top": (
        c_int,
        [c_i64, c_i64, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp,
         c_int, c_vp, c_vp, c_vp],
    ),
    "gsb200_surfel_contrib_max_samples": (c_int, []),
    "gsb200_surfel_contrib_count": (
        c_int,
        [c_i64, c_i64, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_vp, c_vp],
    ),
    "gsb200_surfel_contrib_ids": (
        c_int,
        [c_i64, c_i64, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp,
         c_int, c_vp, c_vp, c_vp],
    ),
    "gsb200_surfel_contrib_top": (
        c_int,
        [c_i64, c_i64, c_vp, c_vp, c_vp, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp,
         c_int, c_vp, c_vp, c_vp],
    ),
    "gsb200_ut_projection_fwd": (
        c_int,
        [c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_u32,
         c_u32, c_f32, c_f32, c_f32, c_f32, c_f32, c_f32, c_f32, c_f32, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_eval3d_fwd": (
        c_int,
        [c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_int, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_eval3d_bwd": (
        c_int,
        [c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_int, c_u32, c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_vp],
    ),
    "gsb200_eval3d_sparse_fwd": (
        c_int,
        [c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_int, c_u32, c_u32, c_u32, c_u32, c_u32, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
         c_vp],
    ),
    "gsb200_eval3d_sparse_bwd": (
        c_int,
        [c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_int, c_u32, c_u32, c_u32, c_u32, c_u32, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
         c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_eval3d_indices": (
        c_int,
        [c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_u32,
         c_u32, c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_vp, c_sz, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_eval3d_contrib_max_samples": (c_int, []),
    "gsb200_eval3d_contrib_count": (
        c_int,
        [c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_u32, c_u32,
         c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    ),
    "gsb200_eval3d_contrib_ids": (
        c_int,
        [c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_u32, c_u32,
         c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp],
    ),
    "gsb200_eval3d_contrib_top": (
        c_int,
        [c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_u32, c_u32,
         c_u32, c_u32, c_u32, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp],
    ),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


class GsplatB200Error(RuntimeError):
    pass


def lib():
    """The loaded library; raises if it has not been built (python -m gsplat_b200.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise GsplatB200Error(
                f"{LIB_PATH} is missing: build it with `python -m gsplat_b200.build` "
                "(nvcc, sm_90a). gsplat_b200 has no CPU / PyTorch fallback."
            )
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the .so does not export what the header declares
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(rc: int, what: str) -> None:
    if rc == 0:
        return
    L = lib()
    msg = L.gsb200_error_string(rc).decode()
    if rc == -3:
        msg += ": " + L.gsb200_last_cuda_error().decode()
    text = f"{what}: {msg}"
    if rc in (-1, -2):
        raise ValueError(text)  # reference: TORCH_CHECK_VALUE -> ValueError
    raise GsplatB200Error(text)


def ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def stream(device_index: Optional[int] = None) -> int:
    """Raw handle of torch's current stream on a device (default: the current device).  The private getter is the one
    torch's own code generators use; it skips the Stream object torch.cuda.current_stream() builds (3 us a call, a dozen
    calls per step)."""
    if device_index is None:
        device_index = torch._C._cuda_getDevice()
    return torch._C._cuda_getCurrentRawStream(device_index)


def require_cuda(*tensors: Optional[torch.Tensor]) -> torch.device:
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise GsplatB200Error(
                "gsplat_b200 operators run only on CUDA tensors (sm_90a kernels; there is no CPU fallback)"
            )
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise ValueError("all tensors must be on the same CUDA device")
    if dev is None:
        raise ValueError("no tensor arguments")
    return dev


def f32c(t: Optional[torch.Tensor], name: str) -> Optional[torch.Tensor]:
    """contiguous float32 view/copy of t (the reference wrappers call .contiguous() too)."""
    if t is None:
        return None
    if t.dtype != torch.float32:
        raise TypeError(f"{name}: expected float32, got {t.dtype} (gsplat_b200 computes in fp32 only)")
    return t.contiguous()


def bits_for_count(count: int) -> int:
    return int(lib().gsb200_bits_for_count(int(count)))
