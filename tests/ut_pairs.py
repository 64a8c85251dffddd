"""A float64 pair walk for the 3DGUT queries: per pixel, the (pixel, gaussian) pairs oracle/ut.py's eval3d_render
composites, with their weights, built on its pixel_rays and eval3d_alpha so that both take the same decisions."""
import torch

from oracle.ut import ALPHA_T, F64, MAX_ALPHA, T_STOP, eval3d_alpha, pixel_rays


def eval3d_pairs(means, quats, scales, opacities, pose, cam, isect_offsets, flatten_ids, C, N, image_index,
                 transmittances=None):
    """The pair walk of one image in float64: per pixel, the list entries eval3d_render composites, front to back, from
    the pixel's transmittance (``transmittances`` [H, W], or 1), with the same rays (pixel_rays), responses
    (eval3d_alpha), skip and stop rules.  Arguments as oracle.ut.eval3d_render's.  Returns a dict of [H*W, L] arrays
    over the longest tile list L of the image -- ``ids`` (flatten id, -1 past the pixel's pairs), ``weights`` (alpha * T before
    the pair, 0 past them) -- and of [H*W] arrays: ``count``, ``T`` (the final transmittance) and ``margins`` (the
    smallest relative distance of any decision taken at the pixel from its threshold, as eval3d_render's)."""
    H, W = cam.H, cam.W
    th, tw = isect_offsets.shape[-2:]
    offs = isect_offsets.reshape(-1).tolist()
    n_isects = len(flatten_ids)
    ends = [offs[image_index * th * tw + t + 1] if image_index * th * tw + t + 1 < len(offs) else n_isects
            for t in range(th * tw)]
    L = max([e - offs[image_index * th * tw + t] for t, e in enumerate(ends)] + [0])
    ro, rd, rok = pixel_rays(pose, cam)
    T0 = torch.ones(H * W, dtype=F64) if transmittances is None else torch.as_tensor(transmittances, dtype=F64).reshape(-1)
    out_ids = torch.full((H * W, L), -1, dtype=torch.long)
    out_w = torch.zeros(H * W, L, dtype=F64)
    count = torch.zeros(H * W, dtype=torch.long)
    T_out = T0.clone()
    margins = torch.full((H * W,), float("inf"), dtype=F64)
    for ty in range(th):
        for tx in range(tw):
            tile = image_index * th * tw + ty * tw + tx
            ys = torch.arange(ty * 16, min(ty * 16 + 16, H))
            xs = torch.arange(tx * 16, min(tx * 16 + 16, W))
            s, e = offs[tile], ends[ty * tw + tx]
            if len(ys) == 0 or len(xs) == 0 or e <= s:
                continue
            pid = (ys[:, None] * W + xs[None, :]).reshape(-1)
            ids = torch.as_tensor(flatten_ids[s:e], dtype=torch.long)
            bn = (ids // (C * N)) * N + ids % N
            alpha, hit_t, raw = eval3d_alpha(means[bn], quats[bn], scales[bn], opacities[ids], ro[pid], rd[pid])
            use = (hit_t >= 0) & (alpha >= ALPHA_T) & rok[pid][:, None]
            am = torch.where(use, alpha, torch.zeros_like(alpha))
            Tin = T0[pid][:, None] * torch.cumprod(torch.cat([torch.ones(len(pid), 1, dtype=F64), 1 - am], 1), 1)
            stop = use & (Tin[:, 1:] <= T_STOP)
            alive = torch.cumsum(stop.to(torch.int64), 1) == 0
            pair = use & alive
            rank = torch.cumsum(pair.to(torch.int64), 1) - 1
            r, k = torch.nonzero(pair, as_tuple=True)
            out_ids[pid[r], rank[r, k]] = ids[k]
            out_w[pid[r], rank[r, k]] = (am * Tin[:, :-1])[r, k]
            count[pid] = pair.sum(1)
            T_out[pid] = T0[pid] * torch.prod(torch.where(pair, 1 - am, torch.ones_like(am)), 1)
            m_alpha = (alpha - ALPHA_T).abs() / ALPHA_T
            m_hit = hit_t.abs() / (hit_t.abs().max() + 1e-30)
            m_T = (Tin[:, 1:] - T_STOP).abs() / T_STOP
            m_clamp = (raw - MAX_ALPHA).abs() / MAX_ALPHA
            live = torch.cat([torch.ones(len(pid), 1, dtype=torch.bool), alive[:, :-1]], 1) & rok[pid][:, None]
            mm = torch.minimum(torch.minimum(m_alpha, m_clamp), torch.where(use, m_T, torch.full_like(m_T, float("inf"))))
            mm = torch.minimum(mm, torch.where(raw >= ALPHA_T, m_hit * 1e3, torch.full_like(m_hit, float("inf"))))
            mm = torch.where(live, mm, torch.full_like(mm, float("inf")))
            margins[pid] = mm.min(1).values
    return dict(ids=out_ids, weights=out_w, count=count, T=T_out, margins=margins)
