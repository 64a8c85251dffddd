"""Float64 PyTorch-on-CPU restatement of the 2DGS (surfel) kernels of gsplat_b200/csrc/surfel.cu, the truth the GPU tests
compare against.  Same culls (near / far, degenerate ray transform, radius_clip, off-screen; float32 overflow only
approximately, see project), ``ceil`` radii, alpha
threshold, exclusive transmittance stop, median rule and L1 distortion; every gradient comes from autograd.

  project(...)       -> radii, means2d, depths, ray_transforms, normals     (differentiable)
  isect(...)         -> flatten_ids, offsets (per-tile lists sorted by depth, ties by row)
  rasterize(...)     -> dict of the compositing outputs (differentiable; vectorised per tile)
  rasterize_vjp(...) -> the same outputs and the gradients for given cotangents, one tile at a time (bounded memory)
  densify_grad(...)  -> v_densify from v_ray_transforms: (v_rt[..., 0, 2], v_rt[..., 1, 2]) * rt[..., 2, 2]
"""
from __future__ import annotations

import math
from typing import Dict

import numpy as np
import torch

f64 = torch.float64
ALPHA_THRESHOLD = 1.0 / 255.0
MAX_ALPHA = 0.99
TRANSMITTANCE_THRESHOLD = 1e-4
GAUSSIAN_EXTEND = 3.33
FILTER_INV_SQUARE = 2.0


def quat_to_rotmat(q: torch.Tensor) -> torch.Tensor:
    q = q / torch.linalg.norm(q, dim=-1, keepdim=True)
    w, x, y, z = q.unbind(-1)
    return torch.stack(
        [
            1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
            2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
            2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y),
        ],
        dim=-1,
    ).reshape(q.shape[:-1] + (3, 3))


def project(means, quats, scales, viewmats, Ks, width, height, near_plane=0.01, far_plane=1e10, radius_clip=0.0):
    """means [..., N, 3], quats [..., N, 4], scales [..., N, 3], viewmats [..., C, 4, 4], Ks [..., C, 3, 3] (float64).
    Returns radii int32 [..., C, N, 2] and means2d, depths, ray_transforms [..., C, N, 3, 3], normals, zero where culled."""
    R = viewmats[..., :3, :3]
    t = viewmats[..., :3, 3]
    Rq = quat_to_rotmat(quats)  # [..., N, 3, 3]
    one = torch.ones_like(scales[..., :1])
    RS = Rq * torch.cat([scales[..., :2], one], dim=-1)[..., None, :]  # columns s0 r0, s1 r1, r2
    RS_c = torch.einsum("...cij,...njk->...cnik", R, RS)  # [..., C, N, 3, 3]
    mc = torch.einsum("...cij,...nj->...cni", R, means) + t[..., None, :]
    T = torch.cat([RS_c[..., :2], mc[..., None]], dim=-1)
    K = torch.zeros_like(Ks)
    K[..., 0, 0], K[..., 0, 2], K[..., 1, 1], K[..., 1, 2], K[..., 2, 2] = Ks[..., 0, 0], Ks[..., 0, 2], Ks[..., 1, 1], Ks[..., 1, 2], 1.0
    M = torch.einsum("...cij,...cnjk->...cnik", K, T)  # rows M0, M1, M2
    sgn = torch.tensor([1.0, 1.0, -1.0], dtype=means.dtype)
    dist = (M[..., 2, :] * M[..., 2, :] * sgn).sum(-1)
    z = mc[..., 2]
    ok = ~((z <= near_plane) | (z >= far_plane)) & (dist != 0)
    inv = 1.0 / torch.where(ok, dist, torch.ones_like(dist))
    m2 = torch.stack([(M[..., 0, :] * M[..., 2, :] * sgn).sum(-1), (M[..., 1, :] * M[..., 2, :] * sgn).sum(-1)], -1) * inv[..., None]
    tmp = torch.stack([(M[..., 0, :] ** 2 * sgn).sum(-1), (M[..., 1, :] ** 2 * sgn).sum(-1)], -1) * inv[..., None]
    ext = (m2 * m2 - tmp).detach()
    r = torch.ceil(GAUSSIAN_EXTEND * torch.sqrt(torch.clamp_min(ext, 1e-4)))
    ok = ok & ~((r[..., 0] <= radius_clip) & (r[..., 1] <= radius_clip))
    md = m2.detach()
    off = (md[..., 0] + r[..., 0] <= 0) | (md[..., 0] - r[..., 0] >= width) | (md[..., 1] + r[..., 1] <= 0) | (md[..., 1] - r[..., 1] >= height)
    ok = ok & ~off
    # the kernel culls a row whose float32 ray transform, screen mean or depth is not finite.  This restates that only
    # for final values beyond float32's range: a row whose float32 intermediates overflow (the products in the screen
    # mean) while these values fit is culled by the kernel and kept here
    f32max = float(np.finfo(np.float32).max)
    fits = (M.detach().abs() <= f32max).all(-1).all(-1) & (md.abs() <= f32max).all(-1) & (z.detach().abs() <= f32max)
    ok = ok & fits
    radii = torch.where(ok[..., None], r, torch.zeros_like(r)).to(torch.int32)
    nrm = RS_c[..., 2]
    cosv = -(nrm * mc).sum(-1, keepdim=True)
    nrm = nrm * torch.where(cosv > 0, 1.0, -1.0)
    okf = ok.to(means.dtype)
    return (
        radii, m2 * okf[..., None], z * okf, M * okf[..., None, None], nrm * okf[..., None],
    )


def project_margins(means, quats, scales, viewmats, Ks, width, height, near_plane=0.01, far_plane=1e10):
    """Per row: the distance of the radius arguments 3.33 sqrt(ext) to the nearest integer over a float32 rounding budget
    (ext = mean2d^2 - tmp cancels: its budget is 1e-6 * (mean2d^2 + |tmp|)), so below 1 a ceil may flip; the distance
    of the off-screen tests to their thresholds in pixels; the distance of the depth to near / far."""
    with torch.no_grad():
        R, t = viewmats[..., :3, :3], viewmats[..., :3, 3]
        Rq = quat_to_rotmat(quats)
        RS = Rq * torch.cat([scales[..., :2], torch.ones_like(scales[..., :1])], -1)[..., None, :]
        RS_c = torch.einsum("...cij,...njk->...cnik", R, RS)
        mc = torch.einsum("...cij,...nj->...cni", R, means) + t[..., None, :]
        T = torch.cat([RS_c[..., :2], mc[..., None]], -1)
        K = torch.zeros_like(Ks)
        K[..., 0, 0], K[..., 0, 2], K[..., 1, 1], K[..., 1, 2], K[..., 2, 2] = Ks[..., 0, 0], Ks[..., 0, 2], Ks[..., 1, 1], Ks[..., 1, 2], 1.0
        M = torch.einsum("...cij,...cnjk->...cnik", K, T)
        sgn = torch.tensor([1.0, 1.0, -1.0], dtype=means.dtype)
        dist = (M[..., 2, :] ** 2 * sgn).sum(-1)
        m2 = torch.stack([(M[..., 0, :] * M[..., 2, :] * sgn).sum(-1), (M[..., 1, :] * M[..., 2, :] * sgn).sum(-1)], -1) / dist[..., None]
        tmp = torch.stack([(M[..., 0, :] ** 2 * sgn).sum(-1), (M[..., 1, :] ** 2 * sgn).sum(-1)], -1) / dist[..., None]
        ext = torch.clamp_min(m2 * m2 - tmp, 1e-4)
        arg = GAUSSIAN_EXTEND * torch.sqrt(ext)
        budget = GAUSSIAN_EXTEND * 1e-6 * (m2 * m2 + tmp.abs()) / (2 * torch.sqrt(ext)) + 1e-5
        ceil_margin = ((arg - torch.round(arg)).abs() / budget).min(-1).values
        r = torch.ceil(arg)
        edges = torch.stack([m2[..., 0] + r[..., 0], m2[..., 0] - r[..., 0] - width, m2[..., 1] + r[..., 1], m2[..., 1] - r[..., 1] - height], -1)
        screen_margin = edges.abs().min(-1).values
        z = mc[..., 2]
        depth_margin = torch.minimum((z - near_plane).abs(), (z - far_plane).abs())
    return ceil_margin, screen_margin, depth_margin


def isect(means2d, radii, depths, tile_size, tile_width, tile_height):
    """Radius-box tile lists of dense rows [I, N]: flatten_ids int32 (index into I * N) sorted by (image, tile, depth,
    row), offsets int32 [I, th, tw]."""
    m2 = np.asarray(means2d, np.float64).reshape(-1, means2d.shape[-2], 2)
    rad = np.asarray(radii).reshape(m2.shape[0], m2.shape[1], 2)
    dep = np.asarray(depths, np.float64).reshape(m2.shape[0], m2.shape[1])
    I, N = m2.shape[:2]
    keys, ids = [], []
    for img in range(I):
        vis = np.nonzero((rad[img] > 0).all(-1))[0]
        for n in vis:
            x, y = m2[img, n]
            rx, ry = rad[img, n]
            x0 = min(max(0, int(math.floor((x - rx) / tile_size))), tile_width)
            x1 = min(max(0, int(math.floor((x + rx) / tile_size)) + 1), tile_width)
            y0 = min(max(0, int(math.floor((y - ry) / tile_size))), tile_height)
            y1 = min(max(0, int(math.floor((y + ry) / tile_size)) + 1), tile_height)
            for ty in range(y0, y1):
                for tx in range(x0, x1):
                    keys.append((img * tile_height + ty) * tile_width + tx)
                    ids.append(img * N + n)
    keys, ids = np.asarray(keys, np.int64), np.asarray(ids, np.int64)
    if len(ids):
        order = np.lexsort((ids, dep.reshape(-1)[ids], keys))
        keys, ids = keys[order], ids[order]
    n_tiles = I * tile_height * tile_width
    offsets = np.searchsorted(keys, np.arange(n_tiles)).astype(np.int32).reshape(I, tile_height, tile_width)
    return ids.astype(np.int32), offsets


def _tile(px, py, m2, rt, op, col, nrm, bg):
    """Composite one tile.  px, py [P]; gathered gaussians m2 [K, 2], rt [K, 3, 3], op [K], col [K, D], nrm [K, 3];
    bg [D] or None.  Returns outputs per pixel and index / margin bookkeeping (no Python loop over pixels)."""
    P, K = px.shape[0], m2.shape[0]
    if K == 0:
        zero = px.new_zeros(P)
        rc = px.new_zeros(P, col.shape[-1]) + (bg[None] if bg is not None else 0.0)
        none = torch.full((P,), -1, dtype=torch.int64)
        inf = px.new_full((P,), np.inf)
        return rc, zero, px.new_zeros(P, 3), zero, zero, none, none, inf, inf, None
    hu = px[:, None, None] * rt[None, :, 2, :] - rt[None, :, 0, :]  # [P, K, 3]
    hv = py[:, None, None] * rt[None, :, 2, :] - rt[None, :, 1, :]
    s = torch.linalg.cross(hu, hv, dim=-1)
    sz = s[..., 2]
    nz = sz != 0
    szs = torch.where(nz, sz, torch.ones_like(sz))
    u, v = s[..., 0] / szs, s[..., 1] / szs
    g3 = u * u + v * v
    d = m2[None] - torch.stack([px, py], -1)[:, None, :]
    g2 = FILTER_INV_SQUARE * (d * d).sum(-1)
    sigma = 0.5 * torch.minimum(g3, g2)
    raw = op[None] * torch.exp(-sigma)
    alpha = torch.clamp_max(raw, MAX_ALPHA)
    ok = nz & (sigma >= 0) & (alpha >= ALPHA_THRESHOLD)
    a = torch.where(ok, alpha, torch.zeros_like(alpha))
    T_after = torch.cumprod(1.0 - a, dim=1)
    T_before = torch.cat([torch.ones_like(T_after[:, :1]), T_after[:, :-1]], dim=1)
    stop = ok & (T_after <= TRANSMITTANCE_THRESHOLD)
    # gaussians at or after the first stop do not contribute
    alive = torch.cumsum(stop.to(torch.int64), dim=1) == 0
    use = ok & alive
    w = torch.where(use, a * T_before, torch.zeros_like(a))
    T_final = torch.where(use, 1.0 - a, torch.ones_like(a)).prod(dim=1)
    rc = w @ col
    if bg is not None:
        rc = rc + T_final[:, None] * bg[None]
    ra = 1.0 - T_final
    rn = w @ nrm
    depth = col[:, -1]
    wd = w * depth[None]
    # L1 distortion: sum_i 2 w_i (d_i (1 - T_i) - sum_{j<i} w_j d_j)
    excl_wd = torch.cumsum(wd, dim=1) - wd
    dist = (2.0 * (wd * (1.0 - T_before) - w * excl_wd)).sum(1)
    # median: the last contributor whose T before it is > 0.5
    med_mask = use & (T_before > 0.5)
    ar = torch.arange(K)
    med_k = torch.where(med_mask, ar[None], torch.full_like(ar[None], -1)).max(1).values
    has_med = med_k >= 0
    med = torch.where(has_med, depth[med_k.clamp_min(0)], torch.zeros_like(ra))
    last_k = torch.where(use, ar[None], torch.full_like(ar[None], -1)).max(1).values
    with torch.no_grad():
        big = torch.full_like(alpha, np.inf)
        considered = alive | (torch.cumsum(stop.to(torch.int64), 1) - stop.to(torch.int64) == 0)  # up to the first stop
        m_alpha = torch.where(considered & nz, (alpha - ALPHA_THRESHOLD).abs() / ALPHA_THRESHOLD, big)
        m_term = torch.where(considered & ok, (T_before * (1 - alpha) - TRANSMITTANCE_THRESHOLD).abs() / TRANSMITTANCE_THRESHOLD, big)
        m_med = torch.where(use, (T_before - 0.5).abs() / 0.5, big)
        margin = torch.stack([m_alpha.min(1).values, m_term.min(1).values, m_med.min(1).values], -1).min(-1).values
        m_branch = torch.where(use, (g3 - g2).abs() / (g3 + g2 + 1e-300), big).min(1).values
        m_clamp = torch.where(use, (raw - MAX_ALPHA).abs(), big).min(1).values
    # what the absolute screen-mean gradient needs: per pair, the 2-D kernel's d alpha / d means2d (zero on the other
    # branch and where alpha is clamped)
    screen = use & (g2 < g3) & (raw <= MAX_ALPHA)
    dalpha_dxy = torch.where(screen[..., None], (op[None] * torch.exp(-sigma))[..., None] * (-FILTER_INV_SQUARE) * d, torch.zeros_like(d))
    return rc, ra, rn, dist, med, last_k, med_k, margin, torch.minimum(m_branch, m_clamp), (a, dalpha_dxy.detach())


def _tiles(W, H, tile_size, offsets, flatten_ids):
    I, th, tw = offsets.shape
    off = np.concatenate([offsets.reshape(-1).astype(np.int64), [len(flatten_ids)]])
    for t in range(I * th * tw):
        img, rem = divmod(t, th * tw)
        ty, tx = divmod(rem, tw)
        ys, xs = np.meshgrid(np.arange(ty * tile_size, min((ty + 1) * tile_size, H)), np.arange(tx * tile_size, min((tx + 1) * tile_size, W)), indexing="ij")
        ys, xs = ys.reshape(-1), xs.reshape(-1)
        if len(ys) == 0:
            continue
        yield t, img, ys, xs, int(off[t]), int(off[t + 1])


_OUT_NAMES = ("render_colors", "render_alphas", "render_normals", "render_distort", "render_median")


def _run(means2d, rt, colors, opacities, normals, W, H, tile_size, offsets, flatten_ids, backgrounds, masks, cot):
    image_dims = tuple(offsets.shape[:-2])
    I, N, D = int(np.prod(image_dims)) if image_dims else 1, means2d.shape[-2], colors.shape[-1]
    off = np.asarray(offsets).reshape(I, *offsets.shape[-2:])
    fl = np.asarray(flatten_ids).astype(np.int64)
    m2f, rtf, opf = means2d.reshape(I * N, 2), rt.reshape(I * N, 3, 3), opacities.reshape(I * N)
    colf, nrmf = colors.reshape(I * N, D), normals.reshape(I * N, 3)
    bgf = None if backgrounds is None else backgrounds.reshape(I, D)
    mk = None if masks is None else np.asarray(masks).reshape(I, -1)
    z = lambda *s: torch.zeros(s, dtype=f64)  # noqa: E731
    outs = [z(I, H, W, D), z(I, H, W, 1), z(I, H, W, 3), z(I, H, W, 1), z(I, H, W, 1)]
    last_ids = np.zeros((I, H, W), np.int64)
    median_ids = np.zeros((I, H, W), np.int64)
    margin = np.full((I, H, W), np.inf)
    grad_margin = np.full((I, H, W), np.inf)
    leaves = (means2d, rt, colors, opacities, normals) + ((backgrounds,) if backgrounds is not None else ())
    grads = [torch.zeros_like(x) for x in leaves] if cot is not None else None
    absgrad = torch.zeros(I * N, 2, dtype=f64)
    for t, img, ys, xs, s0, s1 in _tiles(W, H, tile_size, off, fl):
        where = (torch.tensor(img).expand(len(ys)), torch.as_tensor(ys), torch.as_tensor(xs))
        if mk is not None and not mk[img, t - img * off.shape[1] * off.shape[2]]:
            # a masked tile shows the background and nothing else
            if bgf is not None:
                outs[0] = outs[0].index_put(where, (bgf[img].detach() if cot is not None else bgf[img]).expand(len(ys), D))
                if cot is not None and cot[0] is not None:
                    grads[5].reshape(I, D)[img] += cot[0].reshape(I, H, W, D)[img, ys, xs].sum(0)
            continue
        ids = torch.as_tensor(fl[s0:s1])
        px = torch.as_tensor(xs, dtype=f64) + 0.5
        py = torch.as_tensor(ys, dtype=f64) + 0.5
        if cot is not None:
            with torch.enable_grad():
                loc = [x.detach().requires_grad_(True) for x in leaves]
                lm2, lrt, lcol, lop, lnrm = (x.reshape((I * N,) + x.shape[len(image_dims) + 1 :]) for x in loc[:5])
                lbg = loc[5].reshape(I, D)[img] if backgrounds is not None else None
                res = _tile(px, py, lm2[ids], lrt[ids], lop[ids], lcol[ids], lnrm[ids], lbg)
                loss = 0.0
                for k, val in enumerate(res[:5]):
                    c = cot[k]
                    if c is None:
                        continue
                    cc = c.reshape(I, H, W, -1)[img, ys, xs]
                    loss = loss + (val.reshape(cc.shape) * cc).sum()
                if torch.is_tensor(loss) and loss.requires_grad:
                    a_pairs, dxy = res[9]
                    gs = torch.autograd.grad(loss, loc + [a_pairs], allow_unused=True)
                    for g_acc, g in zip(grads, gs[:-1]):
                        if g is not None:
                            g_acc += g
                    if gs[-1] is not None:  # |per-pixel screen-mean gradient|, summed per gaussian
                        absgrad.index_add_(0, ids, (gs[-1][..., None] * dxy).abs().sum(0))
            res = tuple(r.detach() if torch.is_tensor(r) else r for r in res)
        else:
            bg = bgf[img] if bgf is not None else None
            res = _tile(px, py, m2f[ids], rtf[ids], opf[ids], colf[ids], nrmf[ids], bg)
        for k in range(5):
            val = res[k]
            outs[k] = outs[k].index_put(where, val.reshape(len(ys), -1))
        lk, mkk = res[5].numpy(), res[6].numpy()
        last_ids[img, ys, xs] = np.where(lk >= 0, s0 + lk, 0)
        median_ids[img, ys, xs] = np.where(mkk >= 0, s0 + mkk, 0)
        margin[img, ys, xs] = res[7].numpy()
        grad_margin[img, ys, xs] = res[8].numpy()
    pix = image_dims + (H, W)
    out = {n: o.reshape(pix + o.shape[-1:]) for n, o in zip(_OUT_NAMES, outs)}
    out.update(last_ids=last_ids.reshape(pix), median_ids=median_ids.reshape(pix), margins=margin.reshape(pix),
               grad_margins=grad_margin.reshape(pix))
    if grads is not None:
        names = ("v_means2d", "v_ray_transforms", "v_colors", "v_opacities", "v_normals", "v_backgrounds")
        out.update({n: g for n, g in zip(names, grads)})
        out["v_densify"] = densify_grad(out["v_ray_transforms"], rt.detach())
        out["absgrad"] = absgrad.reshape(means2d.shape)
    return out


def rasterize(means2d, ray_transforms, colors, opacities, normals, width, height, tile_size, offsets, flatten_ids,
              backgrounds=None, masks=None) -> Dict[str, torch.Tensor]:
    """Differentiable compositing of dense rows ([..., N, *], float64) over the tile lists (offsets [..., th, tw],
    flatten_ids).  Returns render_colors / _alphas / _normals / _distort / _median (tensors) and last_ids, median_ids,
    margins (the smallest relative distance of a pixel's threshold decisions: alpha, stop, median) and grad_margins (kernel branch and alpha clamp, where the gradient is discontinuous), as numpy arrays."""
    return _run(means2d, ray_transforms, colors, opacities, normals, width, height, tile_size, offsets, flatten_ids,
                backgrounds, masks, None)


def rasterize_vjp(means2d, ray_transforms, colors, opacities, normals, width, height, tile_size, offsets, flatten_ids,
                  cotangents, backgrounds=None, masks=None) -> Dict[str, torch.Tensor]:
    """rasterize() plus the gradients of sum(output * cotangent) (cotangents: the five outputs' in order, None = no
    gradient), taken with autograd one tile at a time: v_means2d, v_ray_transforms, v_colors, v_opacities, v_normals,
    v_densify, absgrad (the sum over pixels of |d loss_pixel / d means2d|) and, with backgrounds, v_backgrounds."""
    return _run(means2d, ray_transforms, colors, opacities, normals, width, height, tile_size, offsets, flatten_ids,
                backgrounds, masks, list(cotangents))


def densify_grad(v_ray_transforms: torch.Tensor, ray_transforms: torch.Tensor) -> torch.Tensor:
    return v_ray_transforms[..., :2, 2] * ray_transforms[..., 2:3, 2]


def depth_to_normal(depths, camtoworlds, Ks):
    """Float64 restatement of the surface normals of a z-depth map (gsplat_b200.rendering._depth_to_normal)."""
    H, W = depths.shape[-3], depths.shape[-2]
    y, x = torch.meshgrid(torch.arange(H, dtype=f64), torch.arange(W, dtype=f64), indexing="ij")
    dirs = torch.stack([(x - Ks[..., 0, 2, None, None] + 0.5) / Ks[..., 0, 0, None, None],
                        (y - Ks[..., 1, 2, None, None] + 0.5) / Ks[..., 1, 1, None, None], torch.ones_like(x).expand(Ks.shape[:-2] + (H, W))], -1)
    dirs = torch.einsum("...ij,...hwj->...hwi", camtoworlds[..., :3, :3], dirs)
    pts = camtoworlds[..., None, None, :3, 3] + depths * dirs
    n = torch.linalg.cross(pts[..., 2:, 1:-1, :] - pts[..., :-2, 1:-1, :], pts[..., 1:-1, 2:, :] - pts[..., 1:-1, :-2, :], dim=-1)
    n = n / torch.linalg.vector_norm(n, dim=-1, keepdim=True).clamp_min(1e-12)
    return torch.nn.functional.pad(n, (0, 0, 1, 1, 1, 1))
