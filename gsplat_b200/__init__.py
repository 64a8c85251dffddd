"""gsplat_b200 -- H100-native (sm_90a) kernels behind gsplat's rasterization() operator surface.

Public names mirror /root/reference/gsplat/__init__.py:19-104 for the hot path:
rasterization, fully_fused_projection, spherical_harmonics, isect_tiles, isect_offset_encode,
rasterize_to_pixels, quat_scale_to_covar_preci, the sparse-pixel ops build_sparse_tile_layout,
isect_tiles_sparse, rasterize_to_pixels_sparse, and 2DGS: rasterization_2dgs, fully_fused_projection_2dgs,
rasterize_to_pixels_2dgs (dense layout) and its sparse-pixel form rasterize_to_pixels_2dgs_sparse (this library's own:
the reference has no such op), the sparse-pixel form of the 3DGUT compositing rasterize_to_pixels_eval3d_sparse (also
this library's own), the pair queries rasterize_to_indices_in_range /
rasterize_to_indices_in_range_2dgs, and the per-pixel contributor queries rasterize_num_contributing_gaussians,
rasterize_contributing_gaussian_ids, rasterize_top_contributing_gaussian_ids and their _sparse forms (the pair query's
walk with the compositing kernel's decisions: against the reference's ops they can differ only at pairs on the 1/255
and 1e-4 thresholds), and their 2DGS forms rasterize_num_contributing_gaussians_2dgs,
rasterize_contributing_gaussian_ids_2dgs, rasterize_top_contributing_gaussian_ids_2dgs and their _2dgs_sparse forms
(this library's own: the reference has no such ops; the surfel walk takes rasterize_to_pixels_2dgs's decisions, so
their alphas equal its render_alphas bit for bit), and for 3DGUT the pair query rasterize_to_indices_in_range_eval3d and
the contributor queries rasterize_num_contributing_gaussians_eval3d, rasterize_contributing_gaussian_ids_eval3d,
rasterize_top_contributing_gaussian_ids_eval3d and their _eval3d_sparse forms (this library's own as well; the eval3d
walk takes rasterize_to_pixels_eval3d's decisions, so their alphas equal its render_alphas bit for bit).  Importing the
package does not need a GPU; calling an operator does (and needs gsplat_b200/libgsplat_b200.so, built by ``python -m gsplat_b200.build``).
"""
from .ops import (  # noqa: F401
    FThetaCameraDistortionParameters,
    FThetaPolynomialType,
    RollingShutterType,
    adam,
    build_sparse_tile_layout,
    compute_relocation,
    mcmc_perturb_positions,
    fully_fused_projection,
    fully_fused_projection_2dgs,
    fully_fused_projection_with_ut,
    fused_project_sh,
    isect_offset_encode,
    isect_tiles,
    isect_tiles_sparse,
    quat_scale_to_covar_preci,
    rasterize_contributing_gaussian_ids,
    rasterize_contributing_gaussian_ids_2dgs,
    rasterize_contributing_gaussian_ids_2dgs_sparse,
    rasterize_contributing_gaussian_ids_eval3d,
    rasterize_contributing_gaussian_ids_eval3d_sparse,
    rasterize_contributing_gaussian_ids_sparse,
    rasterize_num_contributing_gaussians,
    rasterize_num_contributing_gaussians_2dgs,
    rasterize_num_contributing_gaussians_2dgs_sparse,
    rasterize_num_contributing_gaussians_eval3d,
    rasterize_num_contributing_gaussians_eval3d_sparse,
    rasterize_num_contributing_gaussians_sparse,
    rasterize_to_indices_in_range,
    rasterize_to_indices_in_range_2dgs,
    rasterize_to_indices_in_range_eval3d,
    rasterize_to_pixels,
    rasterize_to_pixels_2dgs,
    rasterize_to_pixels_2dgs_sparse,
    rasterize_to_pixels_eval3d,
    rasterize_to_pixels_eval3d_sparse,
    rasterize_to_pixels_sparse,
    rasterize_top_contributing_gaussian_ids,
    rasterize_top_contributing_gaussian_ids_2dgs,
    rasterize_top_contributing_gaussian_ids_2dgs_sparse,
    rasterize_top_contributing_gaussian_ids_eval3d,
    rasterize_top_contributing_gaussian_ids_eval3d_sparse,
    rasterize_top_contributing_gaussian_ids_sparse,
    spherical_harmonics,
)
from .losses import l1_loss, ssim_loss  # noqa: F401
from .optimizers import SelectiveAdam  # noqa: F401
from .rendering import rasterization, rasterization_2dgs  # noqa: F401

__version__ = "0.1.0"


def has_3dgs() -> bool:
    """Reference: gsplat._wrapper.has_3dgs (build_config flag, ext.cpp:83-97).  The 3DGS path is the
    one thing this library is built for."""
    return True


def has_adam() -> bool:
    """Reference: _wrapper.py:286 -- the selective ``adam`` op is built."""
    return True


def has_reloc() -> bool:
    """Reference: _wrapper.py:290 -- ``relocation`` (and the MCMC position perturbation) are built."""
    return True


def has_2dgs() -> bool:
    """Reference: _wrapper.py:274 -- 2DGS (surfel) projection and compositing are built (dense layout)."""
    return True


def has_3dgut() -> bool:
    """Reference: _wrapper.py has_3dgut -- False.  In the reference this flag gates 3DGUT tests that need lidar cameras,
    hit-distance modes and tile_size 8, none of which is built here.  What is built:
    ``rasterization(with_ut=True, with_eval3d=True)`` with dense rows, and the two 3DGUT operators it runs on,
    ``fully_fused_projection_with_ut`` and ``rasterize_to_pixels_eval3d`` (distorted pinhole, fisheye and FTheta cameras,
    the FTheta ones also in the Euclidean depth order ``global_z_order=False``; global or rolling shutter:
    ``rolling_shutter`` with the end-of-frame poses ``viewmats_rs``), which also chain with
    ``isect_tiles`` / ``isect_offset_encode`` as in the reference's ``_rasterization``."""
    return False


def has_losses() -> bool:
    """The reference's fused Gaussian regularisation losses (losses_fused.py) are out of scope."""
    return False


def has_camera_wrappers() -> bool:
    return False


__all__ = [
    "rasterization",
    "fully_fused_projection",
    "fully_fused_projection_with_ut",
    "rasterize_to_pixels_eval3d",
    "rasterize_to_pixels_eval3d_sparse",
    "fused_project_sh",
    "spherical_harmonics",
    "RollingShutterType",
    "FThetaPolynomialType",
    "FThetaCameraDistortionParameters",
    "isect_tiles",
    "isect_offset_encode",
    "rasterize_to_pixels",
    "build_sparse_tile_layout",
    "isect_tiles_sparse",
    "rasterize_to_pixels_sparse",
    "rasterization_2dgs",
    "fully_fused_projection_2dgs",
    "rasterize_to_pixels_2dgs",
    "rasterize_to_pixels_2dgs_sparse",
    "rasterize_to_indices_in_range",
    "rasterize_to_indices_in_range_2dgs",
    "rasterize_num_contributing_gaussians",
    "rasterize_num_contributing_gaussians_sparse",
    "rasterize_contributing_gaussian_ids",
    "rasterize_contributing_gaussian_ids_sparse",
    "rasterize_top_contributing_gaussian_ids",
    "rasterize_top_contributing_gaussian_ids_sparse",
    "rasterize_num_contributing_gaussians_2dgs",
    "rasterize_num_contributing_gaussians_2dgs_sparse",
    "rasterize_contributing_gaussian_ids_2dgs",
    "rasterize_contributing_gaussian_ids_2dgs_sparse",
    "rasterize_top_contributing_gaussian_ids_2dgs",
    "rasterize_top_contributing_gaussian_ids_2dgs_sparse",
    "rasterize_to_indices_in_range_eval3d",
    "rasterize_num_contributing_gaussians_eval3d",
    "rasterize_num_contributing_gaussians_eval3d_sparse",
    "rasterize_contributing_gaussian_ids_eval3d",
    "rasterize_contributing_gaussian_ids_eval3d_sparse",
    "rasterize_top_contributing_gaussian_ids_eval3d",
    "rasterize_top_contributing_gaussian_ids_eval3d_sparse",
    "quat_scale_to_covar_preci",
    "compute_relocation",
    "mcmc_perturb_positions",
    "adam",
    "SelectiveAdam",
    "l1_loss",
    "ssim_loss",
    "has_3dgs",
    "has_adam",
    "has_reloc",
    "has_2dgs",
    "has_3dgut",
    "has_losses",
    "has_camera_wrappers",
]
