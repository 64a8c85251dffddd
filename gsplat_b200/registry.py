"""Registry-level binding (INTEGRATION.md section B, executable form): register the C ABI as the CUDA implementation
of the reference's EXISTING op schemas, so that a gsplat build keeps its ``rendering.py`` / ``_wrapper.py`` and its
registered autograd untouched and only the kernels behind ``torch.ops.gsplat.<op>`` change.

    import gsplat                      # defines the schemas (gsplat/cuda/ext.cpp:984-1089)
    import gsplat_b200.registry as r
    r.register()                       # rasterize_to_pixels_3dgs / _bwd -> libgsplat_b200.so

Covered here: the compositing pair (the path's dominant kernels).  The other ops of the table in INTEGRATION.md
follow the same pattern: argument order = schema order, outputs allocated by the caller as the reference's host code
does (csrc/Rasterization.cpp:275-365, 484-587).  Nothing is kept between forward and backward -- the backward schema
passes the forward's inputs again, so the record streams are rebuilt with gsb200_raster_pack -- which keeps the pair
re-entrant and safe on autograd worker threads.
"""
from __future__ import annotations

import torch

from ._cabi import stream as _raw_stream

from ._cabi import check, lib, ptr
from .ops import _grad_records, _prod, _split_grad_records

_libs = []


def _geom(isect_offsets, flatten_ids, colors):
    th, tw = isect_offsets.shape[-2:]
    I = isect_offsets.numel() // max(th * tw, 1)
    return I, th, tw, colors.shape[-1], flatten_ids.numel()


def _stream() -> int:
    return _raw_stream()


def rasterize_to_pixels_3dgs(means2d, conics, colors, opacities, backgrounds, masks, image_width, image_height, tile_size,
                             isect_offsets, flatten_ids, packed, absgrad):
    """Schema: ext.cpp:1079-1083 -> (renders, alphas, means2d_absgrad holder, last_ids)."""
    L = lib()
    I, th, tw, D, S = _geom(isect_offsets, flatten_ids, colors)
    dev = means2d.device
    N = means2d.shape[-2] if not packed else max((means2d.shape[0] + max(I, 1) - 1) // max(I, 1), 1)
    means2d, conics, colors, opacities = means2d.contiguous(), conics.contiguous(), colors.contiguous(), opacities.contiguous()
    img = tuple(isect_offsets.shape[:-2])
    rec = torch.empty(max(L.gsb200_raster_records_bytes(S, D, I * th * tw), 16), dtype=torch.uint8, device=dev)
    renders = torch.empty(img + (image_height, image_width, D), device=dev)
    alphas = torch.empty(img + (image_height, image_width, 1), device=dev)
    last_ids = torch.empty(img + (image_height, image_width), dtype=torch.int32, device=dev)
    m8 = None if masks is None else masks.contiguous().view(torch.uint8)
    with torch.cuda.device(dev):
        check(
            L.gsb200_raster_fwd(
                I, N, D, ptr(means2d), ptr(conics), ptr(colors), ptr(opacities), ptr(backgrounds), ptr(m8), image_width,
                image_height, tile_size, tw, th, ptr(isect_offsets.contiguous()), ptr(flatten_ids.contiguous()), S, ptr(rec),
                ptr(renders), ptr(alphas), ptr(last_ids), _stream(),
            ),
            "rasterize_to_pixels_3dgs",
        )
    holder = torch.zeros_like(means2d) if absgrad else means2d.new_empty(0)
    return renders, alphas, holder, last_ids


def rasterize_to_pixels_3dgs_bwd(means2d, conics, colors, opacities, backgrounds, masks, tile_offsets, flatten_ids,
                                 render_alphas, last_ids, image_width, image_height, tile_size, absgrad, v_render_colors,
                                 v_render_alphas, compute_v_backgrounds):
    """Schema: ext.cpp:1084-1089 -> (v_means2d_abs?, v_means2d, v_conics, v_colors, v_opacities, v_backgrounds?)."""
    L = lib()
    I, th, tw, D, S = _geom(tile_offsets, flatten_ids, colors)
    dev = means2d.device
    rows = tuple(means2d.shape[:-1])
    N = (_prod(rows) + max(I, 1) - 1) // max(I, 1)
    means2d, conics, colors, opacities = means2d.contiguous(), conics.contiguous(), colors.contiguous(), opacities.contiguous()
    offsets, fl = tile_offsets.contiguous(), flatten_ids.contiguous()
    g = _grad_records(rows, D, absgrad, dev)
    m8 = None if masks is None else masks.contiguous().view(torch.uint8)
    with torch.cuda.device(dev):
        rec = torch.empty(max(L.gsb200_raster_records_bytes(S, D, I * th * tw), 16), dtype=torch.uint8, device=dev)
        check(
            L.gsb200_raster_pack(I, D, ptr(means2d), ptr(conics), ptr(colors), ptr(opacities), tw, th, ptr(offsets), ptr(fl), S, ptr(rec), _stream()),
            "raster_pack",
        )
        check(
            L.gsb200_raster_bwd(
                I, N, D, ptr(backgrounds), ptr(m8), image_width, image_height, tile_size, tw, th, ptr(offsets), ptr(fl), S,
                ptr(rec), ptr(render_alphas.contiguous()), ptr(last_ids.contiguous()), ptr(v_render_colors.contiguous()),
                ptr(v_render_alphas.contiguous()), absgrad, ptr(g), _stream(),
            ),
            "rasterize_to_pixels_3dgs_bwd",
        )
    v_bg = None
    if compute_v_backgrounds and backgrounds is not None:
        v_bg = (v_render_colors * (1.0 - render_alphas)).sum(dim=(-3, -2))
    v_m2, v_con, v_col, v_op, v_abs = _split_grad_records(g, D, absgrad)
    v_abs = v_abs.contiguous() if absgrad else None
    return v_abs, v_m2.contiguous(), v_con.contiguous(), v_col.contiguous(), v_op.contiguous(), v_bg


def register(namespace: str = "gsplat") -> None:
    """Install the implementations above as the CUDA kernels of ``torch.ops.<namespace>.rasterize_to_pixels_3dgs``
    and ``..._bwd`` (the schemas must already be defined, i.e. the reference extension is loaded)."""
    impl = torch.library.Library(namespace, "IMPL")
    impl.impl("rasterize_to_pixels_3dgs", rasterize_to_pixels_3dgs, "CUDA")
    impl.impl("rasterize_to_pixels_3dgs_bwd", rasterize_to_pixels_3dgs_bwd, "CUDA")
    _libs.append(impl)  # the registration lives as long as the Library object
