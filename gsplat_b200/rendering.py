"""rasterization(): the public entry point, signature-compatible with the reference
(/root/reference/gsplat/rendering.py:234-690).  Orchestration (projection -> SH -> tile intersection ->
offsets -> compositing, channel chunking, depth channels, meta dict) stays in Python and follows the
reference's own Python restatement ``_rasterization`` (rendering.py:722-1106) and the C++ orchestrator it
mirrors (csrc/Rendering.cpp:745-1481); every kernel is ours (gsplat_b200.ops).

Scope: the 3DGS EWA path named by BASELINE.json (pinhole / orthographic / fisheye cameras, dense or
``packed=True`` rows with optional ``sparse_grad``, classic / antialiased, RGB / D / ED / RGB+D / RGB+ED,
backgrounds, masks, absgrad, SH or post-activation colours, ``distributed=True`` Gaussian sharding).

3DGUT (``with_ut=True, with_eval3d=True`` together): the unscented-transform projection and the eval3d compositing
through a distorted pinhole (radial / tangential / thin-prism coefficients), fisheye (radial) or FTheta
(``ftheta_coeffs``) camera, dense rows, global or rolling shutter, classic mode, RGB / D / ED / RGB+D / RGB+ED,
following the reference's orchestrator (csrc/Rendering.cpp:890-934, 1307-1308, 1353-1410).  FTheta cameras also take
``global_z_order=False``: the depths, the tile order and the D / ED channels are then the distance from the camera
centre.  ``tile_size=None`` resolves to 16 here; the reference resolves it to 8 below 1080p.  with_ut or with_eval3d
alone, lidar cameras, external distortion, ``global_z_order=False`` for pinhole / fisheye, hit-distance modes, normals,
extra signals and packed 3DGUT rows raise NotImplementedError.

rasterization_2dgs(): surfel splatting (2DGS) on the dense layout, following the reference's orchestrator
(csrc/Rendering.cpp:1705-1958): ray-transform projection -> radius-box tile intersection -> compositing of colours,
normals, distortion and median depth.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch
from torch import Tensor

from .ops import (
    _SUPPORTED_CHANNELS,
    _project_ut,
    _rasterize_eval3d,
    _shutter_type,
    _ut_camera,
    _ut_geometry,
    _ut_params,
    RollingShutterType,
    RowSideOutputs,
    fully_fused_projection,
    fully_fused_projection_2dgs,
    fused_project_sh,
    isect_tiles_sorted,
    rasterize_to_pixels,
    rasterize_to_pixels_2dgs,
    rasterize_to_pixels_rows,
    spherical_harmonics,
    spherical_harmonics_rows,
)


_COLOR_MODES = {"RGB", "RGB-d", "RGB-Ed", "RGB+D", "RGB+ED"}
_HIT_DISTANCE_MODES = {"d", "Ed", "RGB-d", "RGB-Ed"}
_DEPTH_MODES = {"D", "ED", "RGB+D", "RGB+ED"}
_EXPECTED_MODES = {"Ed", "ED", "RGB-Ed", "RGB+ED"}
_ALL_MODES = _COLOR_MODES | _HIT_DISTANCE_MODES | _DEPTH_MODES


class _Lazy:
    """A meta value that is only computed when somebody reads it."""

    __slots__ = ("fn",)

    def __init__(self, fn):
        self.fn = fn


class _Meta(dict):
    """The meta dict of rasterization(); ``_Lazy`` values are computed on first access and then stored.  Every read path
    resolves them (the Python-level ``__iter__`` also keeps ``dict(meta)`` / ``{**meta}`` off CPython's raw-entry fast path)."""

    def _resolve(self, key):
        v = dict.__getitem__(self, key)
        if isinstance(v, _Lazy):
            v = v.fn()
            dict.__setitem__(self, key, v)
        return v

    def _resolve_all(self):
        for k in list(dict.keys(self)):
            self._resolve(k)

    def __getitem__(self, key):
        return self._resolve(key)

    def get(self, key, default=None):
        return self._resolve(key) if dict.__contains__(self, key) else default

    def __iter__(self):
        return dict.__iter__(self)

    def items(self):
        self._resolve_all()
        return dict.items(self)

    def values(self):
        self._resolve_all()
        return dict.values(self)

    def copy(self):
        self._resolve_all()
        return dict(dict.items(self))

    def pop(self, key, *default):
        if dict.__contains__(self, key):
            self._resolve(key)
        return dict.pop(self, key, *default)


def _unsupported(name: str, why: str = "out of scope for the gsplat_b200 hot path (SURVEY.md section 8)"):
    raise NotImplementedError(f"rasterization({name}): {why}")


def _check_colors(colors, sh_degree, batch_dims, C, N):
    """The colour shapes both rasterizers accept: post-activation [..., N, D] or [..., C, N, D], or SH [N, K, D]."""
    nb = len(batch_dims)
    if sh_degree is None:
        ok = (colors.dim() == nb + 2 and tuple(colors.shape[:-1]) == batch_dims + (N,)) or (
            colors.dim() == nb + 3 and tuple(colors.shape[:-1]) == batch_dims + (C, N)
        )
        if not ok:
            raise ValueError(f"colors must be [..., N, D] or [..., C, N, D], got {tuple(colors.shape)}")
    else:
        if colors.dim() != 3 or colors.shape[0] != N:
            raise ValueError(f"SH colors must be [N, K, D], got {tuple(colors.shape)}")
        if (sh_degree + 1) ** 2 > colors.shape[-2]:
            raise ValueError(f"sh_degree={sh_degree} needs K >= {(sh_degree + 1) ** 2}, got {colors.shape[-2]}")


def _color_features(colors, sh_degree, means, viewmats, radii, batch_dims, C, N, viewmats_rs=None):
    """[..., C, N, D] features of the dense rows: the post-activation colours broadcast over the cameras, or the SH
    colours evaluated for every visible row (seen from the mean of the two poses' positions with ``viewmats_rs``)."""
    if sh_degree is None:
        if colors.dim() == len(batch_dims) + 2:
            return torch.broadcast_to(colors[..., None, :, :], batch_dims + (C, N, colors.shape[-1]))
        return colors
    valid = (radii > 0).all(dim=-1)
    feat = spherical_harmonics(sh_degree, means, viewmats, colors, masks=valid, viewmats_rs=viewmats_rs)
    return torch.clamp_min(feat + 0.5, 0.0)


def _with_depth_channel(feat, depths, backgrounds, has_color, has_depth, batch_dims, C):
    """[colour | depth] features and backgrounds: D / ED / RGB+D / RGB+ED append the depths as the last channel and a
    zero channel to the backgrounds (a depth-only mode renders the depths alone)."""
    if has_color and has_depth:
        feat = torch.cat((feat, depths[..., None]), dim=-1)
        if backgrounds is not None:
            backgrounds = torch.cat([backgrounds, torch.zeros(batch_dims + (C, 1), device=backgrounds.device)], dim=-1)
    elif not has_color:
        feat = depths[..., None]
        if backgrounds is not None:
            backgrounds = torch.zeros(batch_dims + (C, 1), device=backgrounds.device)
    return feat, backgrounds


def _normalize_expected_depth(render_colors, render_alphas, render_mode):
    """ED / RGB+ED: the last channel is the accumulated depth; divide it by the alpha."""
    if render_mode not in _EXPECTED_MODES:
        return render_colors
    depth = render_colors[..., -1:] / render_alphas.clamp(min=1e-10)
    return torch.cat([render_colors[..., :-1], depth], dim=-1)


def _project_dense(
    means, covars, quats, scales, opacities, colors, viewmats, Ks, width, height, sh_degree, eps2d, near_plane, far_plane,
    radius_clip, antialiased, camera_model, has_color, nb, batch_dims, C, N, rows_out=None,
):
    """Dense [..., C, N] projection (+ SH): the fused single pass when it applies, else the per-op kernels."""
    fused = (
        has_color and sh_degree is not None and covars is None and nb == 0 and colors.shape[-1] == 3
        and not viewmats.requires_grad and camera_model == "pinhole"
    )
    if fused:
        radii, means2d, depths, conics, feat, compensations = fused_project_sh(
            means, quats, scales, opacities, colors, viewmats, Ks, width, height, sh_degree, eps2d, near_plane,
            far_plane, radius_clip, antialiased, rows_out=rows_out,
        )
    else:
        radii, means2d, depths, conics, compensations = fully_fused_projection(
            means, covars, quats, scales, viewmats, Ks, width, height, eps2d=eps2d, near_plane=near_plane,
            far_plane=far_plane, radius_clip=radius_clip, packed=False, calc_compensations=antialiased,
            camera_model=camera_model, opacities=opacities,
        )
        feat = _color_features(colors, sh_degree, means, viewmats, radii, batch_dims, C, N) if has_color else None

    opac = torch.broadcast_to(opacities[..., None, :], batch_dims + (C, N))
    if compensations is not None:
        opac = opac * compensations
    return radii, means2d, depths, conics, feat, compensations, opac


def rasterization(
    means: Tensor,  # [..., N, 3]
    quats: Optional[Tensor],  # [..., N, 4]
    scales: Optional[Tensor],  # [..., N, 3]
    opacities: Tensor,  # [..., N]
    colors: Optional[Tensor],  # [..., (C,) N, D] or [N, K, 3] SH coefficients
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    width: int,
    height: int,
    near_plane: float = 0.01,
    far_plane: float = 1e10,
    radius_clip: float = 0.0,
    eps2d: float = 0.3,
    sh_degree: Optional[int] = None,
    packed: bool = True,
    tile_size: Optional[int] = None,
    backgrounds: Optional[Tensor] = None,
    render_mode: str = "RGB",
    sparse_grad: bool = False,
    absgrad: bool = False,
    rasterize_mode: str = "classic",
    channel_chunk: int = 32,
    distributed: bool = False,
    camera_model: str = "pinhole",
    segmented: bool = False,
    covars: Optional[Tensor] = None,
    with_ut: bool = False,
    with_eval3d: bool = False,
    return_normals: bool = False,
    global_z_order: bool = True,
    rays: Optional[Tensor] = None,
    radial_coeffs: Optional[Tensor] = None,
    tangential_coeffs: Optional[Tensor] = None,
    thin_prism_coeffs: Optional[Tensor] = None,
    ftheta_coeffs=None,
    lidar_coeffs=None,
    external_distortion_coeffs=None,
    rolling_shutter=None,
    viewmats_rs: Optional[Tensor] = None,
    ut_params=None,
    extra_signals: Optional[Tensor] = None,
    extra_signals_sh_degree: Optional[int] = None,
    renderer_config=None,
) -> Tuple[Tensor, Tensor, Dict]:
    """Rasterize N 3D Gaussians to C image planes.  Returns (render_colors [..., C, H, W, X],
    render_alphas [..., C, H, W, 1], meta) with the reference's meta keys.

    ``with_ut=True, with_eval3d=True`` renders 3DGUT: the unscented-transform projection through a distorted pinhole
    (``radial_coeffs`` [..., C, 6], ``tangential_coeffs`` [..., C, 2], ``thin_prism_coeffs`` [..., C, 4]) or fisheye
    (``radial_coeffs`` [..., C, 4]) or FTheta (``camera_model="ftheta"`` with ``ftheta_coeffs``, one
    FThetaCameraDistortionParameters shared by every camera) camera, radius-box tile lists, and compositing that
    evaluates each Gaussian in 3-D along the pixel's ray.  With an FTheta camera, ``global_z_order=False`` orders the
    tile lists by the distance from the camera centre and renders that distance in D / ED.  Dense rows only: pass ``packed=False``.  Gradients reach means, quats, scales, colours or SH
    coefficients, opacities and backgrounds, and viewmats through the SH view directions only; ``meta["means2d"]``
    carries none and ``absgrad`` is accepted and does nothing, as in the reference.  ``tile_size=None`` means 16; the
    reference picks 8 below 1080p, which changes ``meta["tile_size"]`` and the tile grid, and can change pixels where a
    Gaussian's 3-D response reaches outside its radius box (a 16-pixel tile list keeps pairs an 8-pixel one drops)."""
    # ---- 3DGUT: the unscented-transform projection + eval3d compositing, only as the pair
    if with_ut and with_eval3d:
        return _rasterization_3dgut(
            means, quats, scales, opacities, colors, viewmats, Ks, width, height, near_plane, far_plane, radius_clip,
            eps2d, sh_degree, packed, tile_size, backgrounds, render_mode, sparse_grad, rasterize_mode, channel_chunk,
            distributed, camera_model, covars, return_normals, global_z_order, rays, radial_coeffs, tangential_coeffs,
            thin_prism_coeffs, ftheta_coeffs, lidar_coeffs, external_distortion_coeffs, rolling_shutter, viewmats_rs,
            ut_params, extra_signals, renderer_config,
        )
    # ---- features outside the path
    if with_ut or with_eval3d:
        _unsupported("with_ut/with_eval3d", "3DGUT is built for with_ut=True and with_eval3d=True together")
    for name, val in (
        ("rays", rays), ("radial_coeffs", radial_coeffs), ("tangential_coeffs", tangential_coeffs),
        ("thin_prism_coeffs", thin_prism_coeffs), ("ftheta_coeffs", ftheta_coeffs), ("lidar_coeffs", lidar_coeffs),
        ("external_distortion_coeffs", external_distortion_coeffs), ("viewmats_rs", viewmats_rs),
        ("ut_params", ut_params), ("extra_signals", extra_signals),
    ):
        if val is not None:
            _unsupported(name)
    # renderer_config selects the implementation of the eval3d rasterizer (reference rendering.py:548-556); the classic
    # path only admits the default RendererConfig_MixedBatch, which changes nothing here
    if renderer_config is not None and type(renderer_config).__name__ != "RendererConfig_MixedBatch":
        _unsupported(f"renderer_config={type(renderer_config).__name__}", "eval3d renderer variants are out of scope")
    if return_normals:
        _unsupported("return_normals")
    if _shutter_type(rolling_shutter) != RollingShutterType.GLOBAL:
        _unsupported("rolling_shutter", "a rolling shutter is built for 3DGUT (with_ut=True, with_eval3d=True)")
    if camera_model not in ("pinhole", "ortho", "fisheye"):
        _unsupported(f"camera_model={camera_model!r}", "the EWA projection is built for pinhole / ortho / fisheye")
    if render_mode not in _ALL_MODES:
        raise ValueError(f"unknown render_mode {render_mode!r}")
    if render_mode in _HIT_DISTANCE_MODES:
        _unsupported(f"render_mode={render_mode!r}", "hit-distance modes belong to the eval3d (3DGUT) renderer")
    if rasterize_mode not in ("classic", "antialiased"):
        raise ValueError(f"unknown rasterize_mode {rasterize_mode!r}")
    if sparse_grad and not packed:
        raise ValueError("sparse_grad requires packed=True")
    if sparse_grad and distributed:
        _unsupported("sparse_grad with distributed=True")
    world_size, world_rank = 1, 0
    if distributed:
        # reference: rendering.py:178-197 -- needs an initialised default group; NCCL in the reference (the CPU
        # tests of the host logic here run it over gloo)
        if not (torch.distributed.is_available() and torch.distributed.is_initialized()):
            raise ValueError("distributed=True requires an initialized default torch.distributed process group.")
        world_size, world_rank = torch.distributed.get_world_size(), torch.distributed.get_rank()
        # the reference's distributed-mode rejections (csrc/Rendering.cpp:187-232), same wording
        if len(tuple(means.shape[:-2])) != 0:
            raise ValueError("distributed=True does not support batch dimensions")
        if absgrad:
            raise ValueError("distributed=True does not support absgrad=True")
        if camera_model != "pinhole":
            raise ValueError("distributed=True only supports camera_model='pinhole'")
        if not global_z_order:
            raise ValueError("distributed=True does not support global_z_order=False")
        if colors is not None and sh_degree is None and colors.dim() == 3:
            raise ValueError("distributed=True only supports per-Gaussian colors")
    if tile_size is None:
        tile_size = 16
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")

    has_color = render_mode in _COLOR_MODES
    has_depth = render_mode in _DEPTH_MODES
    batch_dims = tuple(means.shape[:-2])
    nb = len(batch_dims)
    B = math.prod(batch_dims) if batch_dims else 1
    N = means.shape[-2]
    C = viewmats.shape[-3]
    I = B * C

    # ---- shape validation (reference rendering.py:526-556 / Rendering.cpp:97-512)
    if means.shape[-1] != 3:
        raise ValueError(f"means must be [..., N, 3], got {tuple(means.shape)}")
    if covars is None:
        if quats is None or scales is None:
            raise ValueError("either covars or (quats, scales) is required")
        if tuple(quats.shape) != batch_dims + (N, 4) or tuple(scales.shape) != batch_dims + (N, 3):
            raise ValueError(f"quats/scales shape mismatch: {tuple(quats.shape)}, {tuple(scales.shape)}")
    else:
        if tuple(covars.shape) != batch_dims + (N, 3, 3):
            raise ValueError(f"covars must be [..., N, 3, 3], got {tuple(covars.shape)}")
        quats = scales = None
        tri = ([0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2])
        covars = covars[..., tri[0], tri[1]]
    if tuple(opacities.shape) != batch_dims + (N,):
        raise ValueError(f"opacities must be [..., N], got {tuple(opacities.shape)}")
    if tuple(viewmats.shape) != batch_dims + (C, 4, 4) or tuple(Ks.shape) != batch_dims + (C, 3, 3):
        raise ValueError(f"viewmats/Ks shape mismatch: {tuple(viewmats.shape)}, {tuple(Ks.shape)}")
    if has_color:
        if colors is None:
            raise ValueError(f"render_mode={render_mode!r} needs colors")
        _check_colors(colors, sh_degree, batch_dims, C, N)
        if sh_degree is not None and colors.dtype in (torch.float16, torch.bfloat16):
            # half-precision SH storage: evaluated in fp32 on every path (as ops.spherical_harmonics does); the cast is
            # differentiable, so the gradient comes back in the storage dtype
            colors = colors.float()

    antialiased = rasterize_mode == "antialiased"

    # ---- Seam A (distributed=True): every rank projects ITS gaussians onto ALL cameras
    C_world, N_world = [C], [N]
    if distributed and world_size > 1:
        from . import distributed as gdist

        N_world = gdist.all_gather_ints(N, means.device)
        C_world = gdist.all_gather_ints(C, means.device)
        viewmats, Ks = gdist.all_gather_rows([viewmats, Ks], C_world)
        C = sum(C_world)
        if backgrounds is not None and tuple(backgrounds.shape[:-1]) != (C_world[world_rank],):
            raise ValueError("backgrounds must be [C_local, D] under distributed=True")

    # ---- packed=True: native two-pass compacting projection; everything downstream works on the [nnz, ...] rows
    # (reference rendering.py:347-353, Rendering.cpp:936-973).  Under a multi-rank distributed=True the compacted
    # rows are what Seam B exchanges (only the visible (camera, gaussian) pairs travel).
    sharded = distributed and world_size > 1
    camera_ids = gaussian_ids = batch_ids = None
    rows_out = None
    if packed:
        batch_ids, camera_ids, gaussian_ids, indptr, radii, means2d, depths, conics, compensations = fully_fused_projection(
            means, covars, quats, scales, viewmats, Ks, width, height, eps2d=eps2d, near_plane=near_plane,
            far_plane=far_plane, radius_clip=radius_clip, packed=True, sparse_grad=sparse_grad,
            calc_compensations=antialiased, camera_model=camera_model, opacities=opacities,
        )
        grow = batch_ids * N + gaussian_ids  # row of the gaussian in the flattened [B*N] parameter tensors
        # index_select: its backward is an atomic index_add (advanced indexing would sort the nnz indices)
        opac = torch.index_select(opacities.reshape(-1), 0, grow)
        if compensations is not None:
            opac = opac * compensations
        feat = None
        if has_color:
            if sh_degree is None:
                if colors.dim() == nb + 2:
                    feat = torch.index_select(colors.reshape(-1, colors.shape[-1]), 0, grow)
                else:
                    feat = torch.index_select(
                        colors.reshape(-1, colors.shape[-1]), 0, (batch_ids * C + camera_ids) * N + gaussian_ids
                    )
            else:
                feat = spherical_harmonics_rows(sh_degree, means, viewmats, colors, batch_ids, camera_ids, gaussian_ids)
                feat = torch.clamp_min(feat + 0.5, 0.0)
    else:
        # the fused projection can also count tiles and write the compositing row records, when what follows composites
        # exactly its outputs: plain RGB, input opacities (no antialiasing compensation), rows not exchanged between ranks
        if render_mode == "RGB" and not antialiased and not sharded:
            rows_out = RowSideOutputs(tile_size, math.ceil(width / float(tile_size)), math.ceil(height / float(tile_size)))
        radii, means2d, depths, conics, feat, compensations, opac = _project_dense(
            means, covars, quats, scales, opacities, colors, viewmats, Ks, width, height, sh_degree, eps2d, near_plane, far_plane,
            radius_clip, antialiased, camera_model, has_color, nb, batch_dims, C, N, rows_out=rows_out,
        )
        if rows_out is not None and rows_out.rows is None:
            rows_out = None  # the per-op projection ran: nothing precomputed

    # ---- Seam B (distributed=True): all-to-all so that each rank holds ALL gaussians projected onto ITS cameras
    if sharded and packed:
        # rows are sorted by (camera, gaussian): the rows of rank d's cameras are one contiguous range
        C_local = C_world[world_rank]
        cam0 = [sum(C_world[:d]) for d in range(world_size + 1)]
        ip = indptr.tolist()
        send = [ip[cam0[d + 1]] - ip[cam0[d]] for d in range(world_size)]
        recv = [row[world_rank] for row in gdist.all_gather_int_lists(send, means.device)]
        g0 = sum(N_world[:world_rank])  # global index of this rank's first gaussian
        ints = torch.stack([radii[:, 0], radii[:, 1], (gaussian_ids + g0).int(), camera_ids.int()], dim=-1)
        fields = [means2d, depths, conics, opac] + ([feat] if feat is not None else []) + [ints]
        got = gdist.all_to_all_rows(fields, send, recv)
        means2d, depths, conics, opac = got[0], got[1], got[2], got[3]
        if feat is not None:
            feat = got[4]
        ints = got[-1]
        radii = ints[:, :2].contiguous()
        gaussian_ids = ints[:, 2].long()
        camera_ids = ints[:, 3].long() - cam0[world_rank]
        batch_ids = torch.zeros_like(camera_ids)
        C, N = C_local, sum(N_world)
        I = C
    elif sharded:
        C_local = C_world[world_rank]
        send = [c * N for c in C_world]          # rows (camera-major) going to each camera owner
        recv = [C_local * n for n in N_world]    # rows arriving from each gaussian owner
        fields = [means2d.reshape(C * N, 2), depths.reshape(C * N), conics.reshape(C * N, 3), opac.reshape(C * N)]
        if feat is not None:
            if feat.dim() == 2:  # [N, D] shared by all cameras
                feat = torch.broadcast_to(feat[None], (C, N, feat.shape[-1]))
            fields.append(feat.reshape(C * N, feat.shape[-1]))
        fields.append(radii.reshape(C * N, 2))
        got = gdist.all_to_all_rows(fields, send, recv)
        loc = [gdist.camera_major_to_local(t, C_local, N_world) for t in got]
        means2d, depths, conics, opac = loc[0], loc[1], loc[2], loc[3]
        if feat is not None:
            feat = loc[4]
        radii = loc[-1].contiguous()
        C, N = C_local, sum(N_world)
        I = C

    # ---- tile intersection (AccuTile) + offsets
    tile_width = math.ceil(width / float(tile_size))
    tile_height = math.ceil(height / float(tile_size))
    # the S-sized sort runs on 2- / 4-byte tile ids; meta["isect_ids"] (the reference's 64-bit ids) is rebuilt from them
    # on first access
    if packed and segmented:
        raise ValueError("segmented sort is not supported for packed inputs")
    hits = isect_tiles_sorted(
        means2d, radii, depths, tile_size, tile_width, tile_height, conics=conics, opacities=opac, precounted=rows_out,
        n_images=I if packed else None, image_ids=batch_ids * C + camera_ids if packed else None,
    )
    tiles_per_gauss, flatten_ids, isect_offsets = hits.tiles_per_gauss, hits.flatten_ids, hits.isect_offsets
    isect_ids = _Lazy(hits.isect_ids)
    isect_offsets = isect_offsets.reshape(batch_dims + (C, tile_height, tile_width))

    # ---- assemble channels: [colour | depth]
    feat, backgrounds = _with_depth_channel(feat, depths, backgrounds, has_color, has_depth, batch_dims, C)

    # ---- compositing (chunked over channels, reference Rendering.cpp:1353-1447)
    n_ch = feat.shape[-1]
    if n_ch > channel_chunk:
        outs, render_alphas = [], None
        for lo in range(0, n_ch, channel_chunk):
            bg = backgrounds[..., lo : lo + channel_chunk] if backgrounds is not None else None
            rc, ra = rasterize_to_pixels(
                means2d, conics, feat[..., lo : lo + channel_chunk], opac, width, height, tile_size, isect_offsets,
                flatten_ids, backgrounds=bg, packed=packed, absgrad=absgrad,
            )
            outs.append(rc)
            if render_alphas is None:
                render_alphas = ra
        render_colors = torch.cat(outs, dim=-1)
    else:
        render_colors, render_alphas = rasterize_to_pixels_rows(
            means2d, conics, feat, opac, width, height, tile_size, isect_offsets, flatten_ids, backgrounds=backgrounds,
            packed=packed, absgrad=absgrad, _row_records=rows_out.rows if (rows_out is not None and n_ch == 3) else None,
        )

    render_colors = _normalize_expected_depth(render_colors, render_alphas, render_mode)

    meta = _Meta({
        "batch_ids": batch_ids,
        "camera_ids": camera_ids,
        "gaussian_ids": gaussian_ids,
        "radii": radii,
        "means2d": means2d,
        "depths": depths,
        "conics": conics,
        "opacities": opac,
        "tile_width": tile_width,
        "tile_height": tile_height,
        "tiles_per_gauss": tiles_per_gauss,
        "isect_ids": isect_ids,
        "flatten_ids": flatten_ids,
        "isect_offsets": isect_offsets,
        "width": width,
        "height": height,
        "tile_size": tile_size,
        "n_batches": B,
        "n_cameras": C,
    })
    return render_colors, render_alphas, meta


def _rasterization_3dgut(
    means, quats, scales, opacities, colors, viewmats, Ks, width, height, near_plane, far_plane, radius_clip, eps2d,
    sh_degree, packed, tile_size, backgrounds, render_mode, sparse_grad, rasterize_mode, channel_chunk, distributed,
    camera_model, covars, return_normals, global_z_order, rays, radial_coeffs, tangential_coeffs, thin_prism_coeffs,
    ftheta_coeffs, lidar_coeffs, external_distortion_coeffs, rolling_shutter, viewmats_rs, ut_params, extra_signals,
    renderer_config,
):
    """rasterization(with_ut=True, with_eval3d=True), after the reference's orchestrator (csrc/Rendering.cpp
    rasterization_3dgs under with_ut / with_eval3d): UT projection (no gradient) -> colours or SH -> [colour | depth]
    -> radius-box tile lists -> eval3d compositing per channel chunk -> expected depth.  Every scope check runs before
    anything touches the device."""
    # ---- the reference's own rejections of 3DGUT arguments (rendering.py:164-175, Rendering.cpp:190-357), same wording
    if distributed:
        raise ValueError("distributed=True does not support with_ut=True")
    if rasterize_mode not in ("classic", "antialiased"):
        raise ValueError(f"unknown rasterize_mode {rasterize_mode!r}")
    if rasterize_mode != "classic":
        raise ValueError(
            "3DGUT rendering only supports rasterize_mode='classic'. "
            f"Got rasterize_mode='{rasterize_mode}' with with_ut=True and with_eval3d=True."
        )
    if covars is not None:
        raise ValueError("UT and Eval3D rasterization require quats and scales, not covars")
    if quats is None or scales is None:
        raise ValueError("UT rasterization requires quats and scales")
    if packed:
        raise ValueError("Packed mode is not supported with UT")
    if sparse_grad:
        raise ValueError("Sparse grad is not supported with UT")
    if channel_chunk <= 0:
        raise ValueError("channel_chunk must be > 0")
    if tile_size is None:
        tile_size = 16
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")
    if render_mode not in _ALL_MODES:
        raise ValueError(f"unknown render_mode {render_mode!r}")

    # ---- what the 3DGUT kernels are not built for: NotImplementedError, naming the argument
    if render_mode in _HIT_DISTANCE_MODES:
        _unsupported(f"render_mode={render_mode!r}", "hit-distance modes are not built for 3DGUT")
    if return_normals:
        _unsupported("return_normals", "normals are not built for 3DGUT")
    for name, val in (("rays", rays), ("extra_signals", extra_signals)):
        if val is not None:
            _unsupported(name, "not built for 3DGUT (pinhole / fisheye / ftheta cameras, colour and depth channels)")
    if renderer_config is not None and type(renderer_config).__name__ != "RendererConfig_MixedBatch":
        _unsupported(f"renderer_config={type(renderer_config).__name__}", "3DGUT is built for RendererConfig_MixedBatch only")

    # ---- shapes and dtypes
    has_color = render_mode in _COLOR_MODES
    has_depth = render_mode in _DEPTH_MODES
    batch_dims, C, N = _ut_geometry("rasterization", means, quats, scales, viewmats, Ks)
    B = math.prod(batch_dims) if batch_dims else 1
    if tuple(opacities.shape) != batch_dims + (N,):
        raise ValueError(f"opacities must be [..., N], got {tuple(opacities.shape)}")
    n_ch = int(has_depth)
    if has_color:
        if colors is None:
            raise ValueError(f"render_mode={render_mode!r} needs colors")
        _check_colors(colors, sh_degree, batch_dims, C, N)
        if sh_degree is not None and colors.dtype in (torch.float16, torch.bfloat16):
            colors = colors.float()  # half-precision SH storage, evaluated in fp32 as on the EWA path
        if colors.dtype != torch.float32:
            raise TypeError(f"colors must be float32, got {colors.dtype}")
        if backgrounds is not None and tuple(backgrounds.shape) != batch_dims + (C, colors.shape[-1]):
            raise ValueError(f"backgrounds must be {batch_dims + (C, colors.shape[-1])}, got {tuple(backgrounds.shape)}")
        n_ch += colors.shape[-1]
    if min(channel_chunk, n_ch) > _SUPPORTED_CHANNELS[-1]:
        raise ValueError(
            f"channel_chunk={channel_chunk}: the eval3d kernels composite up to {_SUPPORTED_CHANNELS[-1]} channels per pass"
        )

    # ---- the camera, checked once for the projection and every channel chunk
    cam = _ut_camera("rasterization", viewmats, width, height, camera_model, radial_coeffs, tangential_coeffs,
                     thin_prism_coeffs, ftheta_coeffs, lidar_coeffs, external_distortion_coeffs, rolling_shutter,
                     viewmats_rs, global_z_order)
    ut = _ut_params(ut_params)

    # ---- projection through the camera model (no gradient, as in the reference)
    radii, means2d, depths, conics, _ = _project_ut(means, quats, scales, opacities, viewmats, Ks, width, height, eps2d,
                                                    near_plane, far_plane, radius_clip, False, ut, cam)
    # the SH view directions are the only path by which viewmats (and viewmats_rs) get a gradient
    feat = (_color_features(colors, sh_degree, means, viewmats, radii, batch_dims, C, N, viewmats_rs=viewmats_rs)
            if has_color else None)
    feat, backgrounds = _with_depth_channel(feat, depths, backgrounds, has_color, has_depth, batch_dims, C)
    opac = torch.broadcast_to(opacities[..., None, :], batch_dims + (C, N))

    # ---- tile lists from the radius box alone: the eval3d response is not the 2-D conic, so a conic / opacity cull
    # could drop pairs the compositing uses (the reference passes no conics here under with_ut)
    tile_width = math.ceil(width / float(tile_size))
    tile_height = math.ceil(height / float(tile_size))
    hits = isect_tiles_sorted(means2d, radii, depths, tile_size, tile_width, tile_height)
    flatten_ids = hits.flatten_ids
    isect_offsets = hits.isect_offsets.reshape(batch_dims + (C, tile_height, tile_width))

    # ---- compositing, chunked over channels; a chunk width the kernels are not built for is zero-padded
    outs, render_alphas = [], None
    for lo in range(0, feat.shape[-1], channel_chunk):
        f = feat[..., lo : lo + channel_chunk]
        bg = backgrounds[..., lo : lo + channel_chunk] if backgrounds is not None else None
        D = f.shape[-1]
        pad = next(c for c in _SUPPORTED_CHANNELS if c >= D) - D
        if pad:
            f = torch.nn.functional.pad(f, (0, pad))
            bg = torch.nn.functional.pad(bg, (0, pad)) if bg is not None else None
        rc, ra = _rasterize_eval3d(means, quats, scales, f, opac, viewmats, Ks, width, height, isect_offsets, flatten_ids,
                                   bg, None, cam)
        outs.append(rc[..., :D] if pad else rc)
        if render_alphas is None:
            render_alphas = ra
    render_colors = outs[0] if len(outs) == 1 else torch.cat(outs, dim=-1)
    render_colors = _normalize_expected_depth(render_colors, render_alphas, render_mode)

    meta = _Meta({
        "batch_ids": None,
        "camera_ids": None,
        "gaussian_ids": None,
        "radii": radii,
        "means2d": means2d,
        "depths": depths,
        "conics": conics,
        "opacities": opac,
        "tile_width": tile_width,
        "tile_height": tile_height,
        "tiles_per_gauss": hits.tiles_per_gauss,
        "isect_ids": _Lazy(hits.isect_ids),
        "flatten_ids": flatten_ids,
        "isect_offsets": isect_offsets,
        "width": width,
        "height": height,
        "tile_size": tile_size,
        "n_batches": B,
        "n_cameras": C,
    })
    return render_colors, render_alphas, meta


def _depth_to_normal(depths: Tensor, camtoworlds: Tensor, Ks: Tensor) -> Tensor:
    """Surface normals of a z-depth map [..., H, W, 1] (reference csrc/Rendering.cpp:1659-1702 depth_to_points_2dgs /
    depth_to_normal_2dgs): unproject every pixel with its unnormalised ray, take the cross product of the central
    differences of the neighbouring points, normalise, and pad the one-pixel border with zeros.  Returns [..., H, W, 3]
    in world space."""
    H, W = depths.shape[-3], depths.shape[-2]
    y, x = torch.meshgrid(
        torch.arange(H, device=depths.device, dtype=depths.dtype), torch.arange(W, device=depths.device, dtype=depths.dtype),
        indexing="ij",
    )
    fx, fy = Ks[..., 0, 0, None, None], Ks[..., 1, 1, None, None]
    cx, cy = Ks[..., 0, 2, None, None], Ks[..., 1, 2, None, None]
    dirs = torch.stack([(x - cx + 0.5) / fx, (y - cy + 0.5) / fy], dim=-1)
    dirs = torch.nn.functional.pad(dirs, (0, 1), value=1.0)  # [..., H, W, 3]
    dirs = torch.einsum("...ij,...hwj->...hwi", camtoworlds[..., :3, :3], dirs)
    points = camtoworlds[..., None, None, :3, 3] + depths * dirs
    dx = points[..., 2:, 1:-1, :] - points[..., :-2, 1:-1, :]
    dy = points[..., 1:-1, 2:, :] - points[..., 1:-1, :-2, :]
    normals = torch.linalg.cross(dx, dy, dim=-1)
    # the reference's sqrt(sum of squares); vector_norm's backward is 0 (not NaN) where the cross product vanishes
    normals = normals / torch.linalg.vector_norm(normals, dim=-1, keepdim=True).clamp_min(1e-12)
    return torch.nn.functional.pad(normals, (0, 0, 1, 1, 1, 1), value=0.0)


def rasterization_2dgs(
    means: Tensor,  # [..., N, 3]
    quats: Tensor,  # [..., N, 4]
    scales: Tensor,  # [..., N, 3]
    opacities: Tensor,  # [..., N]
    colors: Tensor,  # [..., (C,) N, D] post-activation colours, or [N, K, D] SH coefficients
    viewmats: Tensor,  # [..., C, 4, 4]
    Ks: Tensor,  # [..., C, 3, 3]
    width: int,
    height: int,
    near_plane: float = 0.01,
    far_plane: float = 1e10,
    radius_clip: float = 0.0,
    eps2d: float = 0.3,
    sh_degree: Optional[int] = None,
    packed: bool = False,
    tile_size: int = 16,
    backgrounds: Optional[Tensor] = None,
    render_mode: str = "RGB",
    sparse_grad: bool = False,
    absgrad: bool = False,
    distloss: bool = False,
    depth_mode: str = "expected",
) -> Tuple[Tensor, Tensor, Tensor, Optional[Tensor], Tensor, Tensor, Dict]:
    """Rasterize N 2D Gaussians (surfels) to C image planes, signature-compatible with the reference
    (gsplat/rendering.py:1358, orchestration csrc/Rendering.cpp:1705-1958).  Returns (render_colors
    [..., C, H, W, X], render_alphas [..., C, H, W, 1], render_normals [..., C, H, W, 3] in world space, surf_normals
    (normals of the rendered depth, world space; None unless the mode renders both colour and depth), render_distort
    [..., C, H, W, 1], render_median [..., C, H, W, 1], meta).  ``meta["gradient_2dgs"]`` is the tensor whose ``.grad``
    is the densification signal; with ``absgrad`` the backward fills ``meta["means2d"].absgrad``.  Dense rows only:
    ``packed=True`` and ``sparse_grad=True`` raise NotImplementedError."""
    if packed or sparse_grad:
        raise NotImplementedError("rasterization_2dgs: only the dense layout (packed=False) is built")
    if render_mode not in _ALL_MODES:
        raise ValueError(f"unknown render_mode {render_mode!r}")
    if render_mode in _HIT_DISTANCE_MODES:
        raise NotImplementedError(f"rasterization_2dgs(render_mode={render_mode!r}): hit-distance modes are not built")
    if depth_mode not in ("expected", "median"):
        raise ValueError(f"unknown depth_mode {depth_mode!r}")
    if tile_size != 16:
        raise ValueError(f"Unsupported tile_size {tile_size}; gsplat_b200 is built for tile_size 16")
    has_color = render_mode in _COLOR_MODES
    has_depth = render_mode in _DEPTH_MODES
    if distloss and not has_depth:
        raise ValueError("distloss requires a depth render mode")
    if means.dim() < 2 or means.shape[-1] != 3:
        raise ValueError(f"means must be [..., N, 3], got {tuple(means.shape)}")
    batch_dims = tuple(means.shape[:-2])
    nb = len(batch_dims)
    N = means.shape[-2]
    if viewmats.dim() != nb + 3:
        raise ValueError(f"viewmats must be [..., C, 4, 4], got {tuple(viewmats.shape)}")
    C = viewmats.shape[-3]
    if tuple(opacities.shape) != batch_dims + (N,):
        raise ValueError(f"opacities must be [..., N], got {tuple(opacities.shape)}")
    if has_color:
        _check_colors(colors, sh_degree, batch_dims, C, N)

    # ---- projection (ray-splat transforms), reference Rendering.cpp:1802-1814
    radii, means2d, depths, ray_transforms, normals = fully_fused_projection_2dgs(
        means, quats, scales, viewmats, Ks, width, height, eps2d=eps2d, near_plane=near_plane, far_plane=far_plane,
        radius_clip=radius_clip,
    )
    opac = torch.broadcast_to(opacities[..., None, :], batch_dims + (C, N))
    # the densification signal: the compositing backward writes its gradient here
    densify = torch.zeros_like(means2d, requires_grad=True)

    # ---- tile intersection: the radius box (no conic / opacity test), sorted by depth per tile
    tile_width = math.ceil(width / float(tile_size))
    tile_height = math.ceil(height / float(tile_size))
    hits = isect_tiles_sorted(means2d, radii, depths, tile_size, tile_width, tile_height)
    tiles_per_gauss, flatten_ids = hits.tiles_per_gauss, hits.flatten_ids
    isect_offsets = hits.isect_offsets.reshape(batch_dims + (C, tile_height, tile_width))

    # ---- channels: [colour | depth]
    feat = _color_features(colors, sh_degree, means, viewmats, radii, batch_dims, C, N) if has_color else None
    if has_depth:
        if has_color:
            feat = torch.cat((feat, depths[..., None]), dim=-1)
            if backgrounds is not None:
                backgrounds = torch.cat([backgrounds, torch.zeros_like(backgrounds[..., :1])], dim=-1)
        else:
            feat = depths[..., None]

    render_colors, render_alphas, render_normals, render_distort, render_median = rasterize_to_pixels_2dgs(
        means2d, ray_transforms, feat, opac, normals, densify, width, height, tile_size, isect_offsets, flatten_ids,
        backgrounds=backgrounds, absgrad=absgrad, distloss=distloss,
    )

    render_colors = _normalize_expected_depth(render_colors, render_alphas, render_mode)

    camtoworlds = torch.linalg.inv(viewmats)
    surf_normals = None
    if has_depth and has_color:
        depth_for_normal = render_median if depth_mode == "median" else render_colors[..., -1:]
        surf_normals = _depth_to_normal(depth_for_normal, camtoworlds, Ks).squeeze(0)
    render_normals = torch.einsum("...ij,...hwj->...hwi", camtoworlds[..., :3, :3], render_normals)

    meta = _Meta({
        "camera_ids": None,
        "gaussian_ids": None,
        "radii": radii,
        "means2d": means2d,
        "depths": depths,
        "ray_transforms": ray_transforms,
        "opacities": opac,
        "normals": normals,
        "tile_width": tile_width,
        "tile_height": tile_height,
        "tiles_per_gauss": tiles_per_gauss,
        "isect_ids": _Lazy(hits.isect_ids),
        "flatten_ids": flatten_ids,
        "isect_offsets": isect_offsets,
        "width": width,
        "height": height,
        "tile_size": tile_size,
        "n_cameras": C,
        "render_distort": render_distort,
        "gradient_2dgs": densify,
    })
    return render_colors, render_alphas, render_normals, surf_normals, render_distort, render_median, meta
