"""gsplat_b200 -- H100-native (sm_90a) kernels behind gsplat's rasterization() operator surface.

Public names mirror /root/reference/gsplat/__init__.py:19-104 for the hot path:
rasterization, fully_fused_projection, spherical_harmonics, isect_tiles, isect_offset_encode,
rasterize_to_pixels, quat_scale_to_covar_preci.  Importing the package does not need a GPU; calling an
operator does (and needs gsplat_b200/libgsplat_b200.so, built by ``python -m gsplat_b200.build``).
"""
from .ops import (  # noqa: F401
    adam,
    compute_relocation,
    mcmc_perturb_positions,
    fully_fused_projection,
    fused_project_sh,
    isect_offset_encode,
    isect_tiles,
    quat_scale_to_covar_preci,
    rasterize_to_pixels,
    spherical_harmonics,
)
from .losses import l1_loss, ssim_loss  # noqa: F401
from .optimizers import SelectiveAdam  # noqa: F401
from .rendering import rasterization  # noqa: F401

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
    return False


def has_3dgut() -> bool:
    return False


def has_losses() -> bool:
    """The reference's fused Gaussian regularisation losses (losses_fused.py) are out of scope."""
    return False


def has_camera_wrappers() -> bool:
    return False


__all__ = [
    "rasterization",
    "fully_fused_projection",
    "fused_project_sh",
    "spherical_harmonics",
    "isect_tiles",
    "isect_offset_encode",
    "rasterize_to_pixels",
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
