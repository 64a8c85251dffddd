"""Drop-in: route an installed ``gsplat`` package's hot path through gsplat_b200 (INTEGRATION.md section A,
executable form).  ``apply()`` rebinds, in place, the names the reference's callers resolve:

  gsplat.rasterization / gsplat.rendering.rasterization                      (rendering.py:234)
  gsplat.cuda._wrapper.{quat_scale_to_covar_preci, fully_fused_projection, spherical_harmonics, isect_tiles,
                        isect_offset_encode, rasterize_to_pixels, adam}        (_wrapper.py:419,436,657,819,1196,1328,1497)
  gsplat.<the same re-exports>                                               (__init__.py:23-62)
  gsplat.relocation.compute_relocation (+ its import in gsplat.strategy.ops) (relocation.py:25, strategy/ops.py:26)
  gsplat.strategy.ops._cuda_fused_mcmc_perturb                               (strategy/ops.py:405)
  gsplat.optimizers.SelectiveAdam                                            (optimizers/selective_adam.py)
  gsplat.losses.ssim_loss when ``losses=True``                               (losses.py:154)

Calls the b200 path does not implement (3DGUT / eval3d, lidar, extra signals, float64 inputs, tile_size != 16, ...)
and calls with invalid arguments are handed to the package's own implementation -- gsplat_b200 raises
NotImplementedError / ValueError / TypeError before launching anything -- so upstream behaviour and error messages are
preserved; ``stats`` counts per name how many calls ran on the b200 kernels and how many were handed over (and why).

Nothing else of the package is touched: strategies, exporters, the Python reference implementations
(``_rasterization``, ``_torch_impl``) keep running the package's own code -- which is what lets the reference's
own tests compare the b200 kernels with the reference's Python twins and lets
``examples/simple_trainer.py`` run unchanged (it imports ``from gsplat.rendering import rasterization`` after
this has been applied, e.g. from a ``sitecustomize`` / ``GSPLAT_BACKEND=b200`` hook).

``undo()`` restores the originals.  The module imports ``gsplat`` lazily: gsplat_b200 itself has no dependency
on it.
"""
from __future__ import annotations

import importlib
from typing import Dict, List, Tuple

_OPS = (
    "quat_scale_to_covar_preci",
    "fully_fused_projection",
    "spherical_harmonics",
    "isect_tiles",
    "isect_offset_encode",
    "rasterize_to_pixels",
)

_saved: List[Tuple[object, str, object]] = []

# per rebound name: how many calls ran on the b200 kernels, how many were handed to the package's own implementation
# (and why).  The policy of the drop-in: anything the b200 path does not implement -- 3DGUT / eval3d, lidar, extra
# signals, float64 inputs, tile_size != 16, ... -- and every argument error is the STOCK implementation's business
# (same results, same messages as upstream); gsplat_b200 declines BEFORE launching anything, so the hand-over is clean.
stats: Dict[str, Dict[str, object]] = {}


def _delegating(name: str, ours, stock):
    import functools

    st = stats.setdefault(name, {"b200": 0, "stock": 0, "reasons": {}})

    @functools.wraps(stock)
    def wrapper(*args, **kwargs):
        try:
            out = ours(*args, **kwargs)
        except (NotImplementedError, TypeError, ValueError) as e:
            st["stock"] += 1
            key = f"{type(e).__name__}: {str(e)[:90]}"
            st["reasons"][key] = st["reasons"].get(key, 0) + 1
            return stock(*args, **kwargs)
        st["b200"] += 1
        return out

    wrapper.__gsb200_ours__ = ours
    return wrapper


def _set(mod, name: str, value) -> None:
    _saved.append((mod, name, getattr(mod, name, None)))
    setattr(mod, name, value)


def applied() -> bool:
    return bool(_saved)


def apply(losses: bool = True, ops: bool = True) -> Dict[str, object]:
    """Rebind the hot-path names of the importable ``gsplat`` package to gsplat_b200.  Idempotent.
    ``ops=False`` leaves the rasterization path alone and only installs the fused SSIM (used by the trainer bench to
    separate the two effects)."""
    if _saved:
        return {"already": True}
    import gsplat_b200 as B

    G = importlib.import_module("gsplat")
    if ops:
        _apply_ops(B, G)
    if losses:
        _apply_losses(G)
    return {"package": G.__file__, "ops": (list(_OPS) + ["adam", "rasterization", "compute_relocation"]) if ops else [], "losses": losses}


def _apply_ops(B, G) -> None:
    W = importlib.import_module("gsplat.cuda._wrapper")
    R = importlib.import_module("gsplat.rendering")
    for name in _OPS:
        fn = _delegating(name, getattr(B, name), getattr(W, name))
        _set(W, name, fn)
        if hasattr(G, name):
            _set(G, name, fn)
    _set(W, "adam", _delegating("adam", B.adam, W.adam))
    rast = _delegating("rasterization", B.rasterization, R.rasterization)
    _set(R, "rasterization", rast)
    _set(G, "rasterization", rast)

    rel = importlib.import_module("gsplat.relocation")
    reloc = _delegating("compute_relocation", B.compute_relocation, rel.compute_relocation)
    _set(rel, "compute_relocation", reloc)
    sops = importlib.import_module("gsplat.strategy.ops")
    _set(sops, "compute_relocation", reloc)

    def _b200_fused_mcmc_perturb(positions, quats, scales, opacities, noise_scale=None, *, scaler=None, t=0.005, k=100.0):
        # same contract as strategy/ops.py:405-461: True when the fused kernel ran
        import torch

        if not positions.is_cuda or not positions.is_contiguous() or positions.dtype != torch.float32:
            return False
        ns = sops._resolve_noise_scale(noise_scale, scaler)
        noise = torch.randn_like(positions)
        B.mcmc_perturb_positions(positions, quats, scales, opacities.flatten(), noise, float(ns), float(t), float(k))
        return True

    _set(sops, "_cuda_fused_mcmc_perturb", _b200_fused_mcmc_perturb)
    opt = importlib.import_module("gsplat.optimizers")
    _set(opt, "SelectiveAdam", B.SelectiveAdam)
    if hasattr(G, "SelectiveAdam"):
        _set(G, "SelectiveAdam", B.SelectiveAdam)


def _apply_losses(G) -> None:
    if True:  # (block kept flat for the diff; always taken)
        # the reference's l1_loss is element-wise (the trainer reduces it), so only the SSIM term has a fused
        # replacement: same semantics as the torch fallback the reference runs when the third-party
        # ``fused_ssim`` package is absent (losses.py:190-201: zero padding, mean over B*C*H*W)
        Ls = importlib.import_module("gsplat.losses")
        from . import losses as BL

        stock_ssim = Ls.ssim_loss

        def ssim_loss(img1, img2, window_size: int = 11):
            # the fused kernel takes over exactly where the reference would take its own fused path
            # (losses.py:177-181: window 11, no gradient to the target, CUDA tensors); everything else
            # -- CPU tensors, other windows, ENFORCE_CONTRACTS input checks -- stays the package's code
            if window_size == 11 and img1.is_cuda and img1.dtype == img2.dtype and not img2.requires_grad and not Ls.ENFORCE_CONTRACTS:
                import torch

                if img1.dtype == torch.float32:
                    return BL.ssim_loss(img1, img2)
            return stock_ssim(img1, img2, window_size)

        ssim_loss.__doc__ = stock_ssim.__doc__
        _set(Ls, "ssim_loss", ssim_loss)
        if hasattr(G, "ssim_loss"):
            _set(G, "ssim_loss", ssim_loss)


def undo() -> None:
    while _saved:
        mod, name, old = _saved.pop()
        if old is None:
            try:
                delattr(mod, name)
            except AttributeError:
                pass
        else:
            setattr(mod, name, old)
