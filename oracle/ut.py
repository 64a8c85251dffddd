"""Float64 PyTorch restatement of the 3DGUT operators (test infrastructure; never imported by gsplat_b200): the OpenCV
pinhole and fisheye camera models with their Newton unprojection, the unscented-transform projection and the
compositing that evaluates each gaussian in 3-D along the pixel's ray.  Differentiable by autograd where the kernels
are (the compositing in means, quats, scales, colors, opacities and backgrounds).

Written from the algorithm: sigma points mean +- sqrt(3 + lambda) * s_i * R[:, i], lambda = alpha^2 (3 + kappa) - 3,
weights lambda / (3 + lambda) (+ 1 - alpha^2 + beta for the covariance) and 1 / (2 (3 + lambda)); a sigma point is
valid when it projects in front of the camera inside the image grown by the margin factor (pinhole with distortion:
also radial factor > 0.8; fisheye: also below the model's maximum angle); the row is valid when any point is (all,
with require_all_sigma_points_valid).  The ray response of a gaussian is exp(-|g x a|^2 / 2) with a = M (o - mu),
g = M d / |M d|, M = S^-1 R^T, zero when the closest approach lies behind the origin.
"""
from __future__ import annotations

import math

import torch

F64 = torch.float64
ALPHA_T, MAX_ALPHA, T_STOP, EXTEND, MIN_COMP = 1.0 / 255.0, 0.99, 1e-4, 3.33, 0.005
UT_DEFAULTS = dict(alpha=0.1, beta=2.0, kappa=0.0, in_image_margin_factor=0.1, require_all_sigma_points_valid=False)


class Camera:
    """One camera: kind 'pinhole' / 'fisheye', K [3, 3], coefficient vectors (None = absent), image size."""

    def __init__(self, kind, K, W, H, radial=None, tangential=None, thin=None):
        K = torch.as_tensor(K, dtype=F64)
        self.kind, self.W, self.H = kind, int(W), int(H)
        self.fx, self.fy, self.cx, self.cy = (float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]))
        f = lambda v, n: [0.0] * n if v is None else [float(x) for x in torch.as_tensor(v).reshape(-1)]  # noqa: E731
        self.distorted = kind == "pinhole" and not (radial is None and tangential is None and thin is None)
        self.k = f(radial, 6 if kind == "pinhole" else 4)
        self.p, self.s = f(tangential, 2), f(thin, 4)
        if kind == "fisheye":
            self.max_angle = self._fisheye_max_angle()
            max_nd = max(self.W / 2.0 / self.fx, self.H / 2.0 / self.fy)
            self.inv_slope = self.max_angle / max_nd

    def _fisheye_max_angle(self):
        k1, k2, k3, k4 = self.k
        # f'(theta) = 1 + 3 k1 t^2 + 5 k2 t^4 + 7 k3 t^6 + 9 k4 t^8: its first positive root bounds the monotone range
        roots = [r for r in __import__("numpy").roots([9 * k4, 7 * k3, 5 * k2, 3 * k1, 1.0]) if abs(r.imag) < 1e-9 and r.real > 0]
        ma = math.sqrt(min(r.real for r in roots)) if roots else float("inf")
        mdx, mdy = max(self.W - self.cx, self.cx), max(self.H - self.cy, self.cy)
        max_r = math.hypot(mdx, mdy)
        return min(ma, max(max_r / self.fx, max_r / self.fy))

    def _fe(self, t):
        t2 = t * t
        k = self.k
        return t * (1 + t2 * (k[0] + t2 * (k[1] + t2 * (k[2] + t2 * k[3]))))

    def _dfe(self, t):
        t2 = t * t
        k = self.k
        return 1 + t2 * (3 * k[0] + t2 * (5 * k[1] + t2 * (7 * k[2] + t2 * 9 * k[3])))

    def project(self, pc, margin):
        """camera-frame points [..., 3] -> (uv [..., 2], valid [...]); invalid points keep the value the transform
        averages ((0, 0) behind the camera)."""
        x, y, z = pc[..., 0], pc[..., 1], pc[..., 2]
        front = z > 0
        zs = torch.where(front, z, torch.ones_like(z))
        if self.kind == "pinhole":
            xn, yn = x / zs, y / zs
            ok = torch.ones_like(front)
            if self.distorted:
                k, p, s = self.k, self.p, self.s
                r2 = xn * xn + yn * yn
                num = 1 + r2 * (k[0] + r2 * (k[1] + r2 * k[2]))
                den = 1 + r2 * (k[3] + r2 * (k[4] + r2 * k[5]))
                icd = torch.where(den.abs() > 1e-8, num / den, torch.zeros_like(den))
                a1 = 2 * xn * yn
                dx = p[0] * a1 + p[1] * (r2 + 2 * xn * xn) + r2 * (s[0] + r2 * s[1])
                dy = p[0] * (r2 + 2 * yn * yn) + p[1] * a1 + r2 * (s[2] + r2 * s[3])
                xn, yn = icd * xn + dx, icd * yn + dy
                ok = icd > 0.8
            u, v = xn * self.fx + self.cx, yn * self.fy + self.cy
        else:
            rxy = torch.sqrt(x * x + y * y).clamp_min(torch.finfo(torch.float32).eps)
            th_full = torch.atan2(rxy, z)
            th = torch.minimum(th_full, torch.full_like(th_full, self.max_angle))
            delta = self._fe(th) / rxy
            ok = (delta > 0) & (th_full < self.max_angle)
            front = front & (delta > 0)
            u, v = self.fx * delta * x + self.cx, self.fy * delta * y + self.cy
        mx, my = self.W * margin, self.H * margin
        inb = (u >= -mx) & (u < self.W + mx) & (v >= -my) & (v < self.H + my)
        uv = torch.stack([torch.where(front, u, torch.zeros_like(u)), torch.where(front, v, torch.zeros_like(v))], -1)
        return uv, front & ok & inb

    def unproject(self, u, v):
        """image points -> (unit camera rays [..., 3], valid), the distortion inverted by Newton iteration."""
        u, v = torch.as_tensor(u, dtype=F64), torch.as_tensor(v, dtype=F64)
        x0, y0 = (u - self.cx) / self.fx, (v - self.cy) / self.fy
        if self.kind == "pinhole":
            x, y, ok = x0.clone(), y0.clone(), torch.ones_like(x0, dtype=torch.bool)
            if self.distorted:
                k, p, s = self.k, self.p, self.s
                ok = torch.zeros_like(ok)
                for _ in range(20):  # float64 converges well inside the kernels' 5 float32 steps
                    r = x * x + y * y
                    al = 1 + r * (k[0] + r * (k[1] + r * k[2]))
                    be = 1 + r * (k[3] + r * (k[4] + r * k[5]))
                    d = al / be
                    fx = d * x + 2 * p[0] * x * y + p[1] * (r + 2 * x * x) + s[0] * r + s[1] * r * r - x0
                    fy = d * y + 2 * p[1] * x * y + p[0] * (r + 2 * y * y) + s[2] * r + s[3] * r * r - y0
                    d_r = ((k[0] + r * (2 * k[1] + 3 * k[2] * r)) * be - al * (k[3] + r * (2 * k[4] + 3 * k[5] * r))) / (be * be)
                    fxx = d + 2 * x * d_r * x + 2 * p[0] * y + 6 * p[1] * x + 2 * x * (s[0] + 2 * s[1] * r)
                    fxy = 2 * y * d_r * x + 2 * p[0] * x + 2 * p[1] * y + 2 * y * (s[0] + 2 * s[1] * r)
                    fyx = 2 * x * d_r * y + 2 * p[1] * y + 2 * p[0] * x + 2 * x * (s[2] + 2 * s[3] * r)
                    fyy = d + 2 * y * d_r * y + 2 * p[1] * x + 6 * p[0] * y + 2 * y * (s[2] + 2 * s[3] * r)
                    det = fxy * fyx - fxx * fyy
                    sx, sy = (fx * fyy - fy * fxy) / det, (fy * fxx - fx * fyx) / det
                    live = (d > 0) & (det.abs() >= 1e-12) & ~ok
                    x, y = torch.where(live, x + sx, x), torch.where(live, y + sy, y)
                    ok = ok | (live & (sx.abs() < 1e-12) & (sy.abs() < 1e-12))
            d = torch.stack([x, y, torch.ones_like(x)], -1)
            return d / d.norm(dim=-1, keepdim=True), ok
        delta = torch.sqrt(x0 * x0 + y0 * y0)
        t = self.inv_slope * delta
        for _ in range(30):
            t = t - (self._fe(t) - delta) / self._dfe(t)
        ok = (t >= 0) & (t < self.max_angle) & ((self._fe(t) - delta).abs() < 1e-9)
        sc = torch.where(delta >= 1e-6, torch.sin(t) / delta.clamp_min(1e-300), torch.zeros_like(t))
        d = torch.stack([sc * x0, sc * y0, torch.where(delta >= 1e-6, torch.cos(t), torch.ones_like(t))], -1)
        return d, ok


def quat_to_rotmat(q):
    q = q / q.norm(dim=-1, keepdim=True)
    w, x, y, z = q.unbind(-1)
    return torch.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y),
    ], -1).reshape(q.shape[:-1] + (3, 3))


def ut_projection(means, quats, scales, opacities, viewmat, cam: Camera, eps2d=0.3, near_plane=0.01, far_plane=1e10,
                  radius_clip=0.0, ut=None):
    """One camera, N gaussians.  Returns dict of float64 radii [N, 2] (0: culled), means2d, depths, conics,
    compensations, the unrounded radii and the margins of the decisions that cull a row (for threshold tests)."""
    ut = dict(UT_DEFAULTS, **(ut or {}))
    means, quats, scales = (torch.as_tensor(t, dtype=F64) for t in (means, quats, scales))
    vm = torch.as_tensor(viewmat, dtype=F64)
    R, t = vm[:3, :3], vm[:3, 3]
    a, kap = ut["alpha"], ut["kappa"]
    lam = a * a * (3 + kap) - 3
    w_m = [lam / (3 + lam)] + [1 / (2 * (3 + lam))] * 6
    w_c = [lam / (3 + lam) + 1 - a * a + ut["beta"]] + [1 / (2 * (3 + lam))] * 6
    Rq = quat_to_rotmat(quats)
    delta = math.sqrt(3 + lam) * Rq * scales[:, None, :]  # column i = spread * s_i * R[:, i]
    pts = torch.stack([means] + [means + delta[..., i] for i in range(3)] + [means - delta[..., i] for i in range(3)], 1)
    pc = pts @ R.T + t
    uv, valid = cam.project(pc, ut["in_image_margin_factor"])
    wm, wc = torch.tensor(w_m, dtype=F64), torch.tensor(w_c, dtype=F64)
    mean2d = (wm[None, :, None] * uv).sum(1)
    du = uv - mean2d[:, None]
    cov = (wc[None, :, None, None] * du[..., :, None] * du[..., None, :]).sum(1)
    ok = valid.all(1) if ut["require_all_sigma_points_valid"] else valid.any(1)
    zc = means @ R.T[:, 2] + t[2]
    eps = torch.finfo(torch.float32).eps
    ok = ok & (zc >= near_plane) & (zc <= far_plane)
    ok = ok & ((quats * quats).sum(-1).abs() >= eps) & (scales.abs() >= eps).all(-1)
    det_o = cov[:, 0, 0] * cov[:, 1, 1] - cov[:, 0, 1] ** 2
    c00, c11, c01 = cov[:, 0, 0] + eps2d, cov[:, 1, 1] + eps2d, cov[:, 0, 1]
    det = c00 * c11 - c01 * c01
    comp = torch.sqrt((det_o / det).clamp_min(MIN_COMP * MIN_COMP))
    ok = ok & (det > 0) & (c00 >= 0) & (c11 >= 0)
    extend = torch.full_like(det, EXTEND)
    if opacities is not None:
        op = torch.as_tensor(opacities, dtype=F64) * comp
        ok = ok & (op >= ALPHA_T)
        extend = torch.minimum(extend, torch.sqrt(2 * torch.log((op / ALPHA_T).clamp_min(1.0))))
    hb = 0.5 * (c00 + c11)
    r1 = extend * torch.sqrt((hb + torch.sqrt((hb * hb - det).clamp_min(0.01))).clamp_min(0))
    rxf = torch.minimum(extend * torch.sqrt(c00.clamp_min(0)), r1)
    ryf = torch.minimum(extend * torch.sqrt(c11.clamp_min(0)), r1)
    rx, ry = torch.ceil(rxf), torch.ceil(ryf)
    ok = ok & ~((rx <= radius_clip) & (ry <= radius_clip))
    ok = ok & ~((mean2d[:, 0] + rx <= 0) | (mean2d[:, 0] - rx >= cam.W) | (mean2d[:, 1] + ry <= 0) | (mean2d[:, 1] - ry >= cam.H))
    z = torch.zeros_like(det)
    conics = torch.stack([c11 / det, -c01 / det, c00 / det], -1)
    return {
        "valid": ok,
        "radii": torch.where(ok[:, None], torch.stack([rx, ry], -1), torch.zeros(len(ok), 2, dtype=F64)),
        "radii_unrounded": torch.stack([rxf, ryf], -1),
        "means2d": torch.where(ok[:, None], mean2d, torch.zeros_like(mean2d)),
        "depths": torch.where(ok, zc, z),
        "conics": torch.where(ok[:, None], conics, torch.zeros_like(conics)),
        "compensations": torch.where(ok, comp, z),
        "sigma_valid": valid,
    }


def pixel_rays(viewmat, cam: Camera):
    """World rays of every pixel centre: origins [H*W, 3], unit directions [H*W, 3], valid [H*W]."""
    vm = torch.as_tensor(viewmat, dtype=F64)
    R, t = vm[:3, :3], vm[:3, 3]
    jj, ii = torch.meshgrid(torch.arange(cam.W, dtype=F64), torch.arange(cam.H, dtype=F64), indexing="xy")
    d, ok = cam.unproject(jj.reshape(-1) + 0.5, ii.reshape(-1) + 0.5)
    o = -(R.T @ t)
    return o.expand(d.shape), d @ R, ok


def eval3d_alpha(means, quats, scales, opacities, ro, rd):
    """alpha [P, L] and the raw margins (hit_t, o * resp) of P rays against L gaussians."""
    Rq = quat_to_rotmat(quats)
    M = Rq.transpose(-1, -2) / scales[:, :, None]  # [L, 3, 3] rows R[:, i] / s_i
    a = torch.einsum("lij,plj->pli", M, ro[:, None, :] - means[None])
    b = torch.einsum("lij,pj->pli", M, rd)
    g = b / b.norm(dim=-1, keepdim=True)
    hit_t = -(g * a).sum(-1)
    c = torch.cross(g, a, dim=-1)
    resp = torch.exp(-0.5 * (c * c).sum(-1))
    raw = opacities[None] * resp
    alpha = torch.clamp(raw, max=MAX_ALPHA)
    return alpha, hit_t, raw


def eval3d_render(means, quats, scales, colors, opacities, viewmat, cam: Camera, isect_offsets, flatten_ids, C, N,
                  image_index, background=None, mask=None):
    """Composites one image (index image_index of the [I] = [B*C] images) from its tile lists, front to back.  means /
    quats / scales [B*N, *], colors [I*N, D], opacities [I*N] (float64 tensors, autograd flows through).  Returns
    (render_colors [H, W, D], render_alphas [H, W, 1], margins [H, W]: the smallest distance of any decision taken at the
    pixel from its threshold, relative)."""
    H, W, D = cam.H, cam.W, colors.shape[-1]
    th, tw = isect_offsets.shape[-2:]
    offs = isect_offsets.reshape(-1).tolist()
    n_isects = len(flatten_ids)
    ro, rd, rok = pixel_rays(viewmat, cam)
    out_c = [[None] * W for _ in range(H)]
    img = torch.zeros(H, W, D, dtype=F64)
    alp = torch.zeros(H, W, 1, dtype=F64)
    margins = torch.full((H, W), float("inf"), dtype=F64)
    rows_c, rows_a = [], []
    bg = background
    for ty in range(th):
        for tx in range(tw):
            tile = image_index * th * tw + ty * tw + tx
            ys = torch.arange(ty * 16, min(ty * 16 + 16, H))
            xs = torch.arange(tx * 16, min(tx * 16 + 16, W))
            if len(ys) == 0 or len(xs) == 0:
                continue
            pid = (ys[:, None] * W + xs[None, :]).reshape(-1)
            if mask is not None and not bool(mask[ty, tx]):
                cols = bg.expand(len(pid), D) if bg is not None else torch.zeros(len(pid), D, dtype=F64)
                rows_c.append((pid, cols, torch.zeros(len(pid), 1, dtype=F64)))
                continue
            s = offs[tile]
            e = offs[tile + 1] if tile + 1 < len(offs) else n_isects
            ids = torch.as_tensor(flatten_ids[s:e], dtype=torch.long)
            if len(ids) == 0:
                T = torch.ones(len(pid), dtype=F64)
                acc = torch.zeros(len(pid), D, dtype=F64)
            else:
                bn = (ids // (C * N)) * N + ids % N
                alpha, hit_t, raw = eval3d_alpha(means[bn], quats[bn], scales[bn], opacities[ids], ro[pid], rd[pid])
                use = (hit_t >= 0) & (alpha >= ALPHA_T) & rok[pid][:, None]
                am = torch.where(use, alpha, torch.zeros_like(alpha))
                one_m = 1 - am
                Tin = torch.cumprod(torch.cat([torch.ones(len(pid), 1, dtype=F64), one_m], 1), 1)
                # the first pair whose transmittance would fall to 1e-4 ends the pixel and does not contribute
                stop = use & (Tin[:, 1:] <= T_STOP)
                alive = torch.cumsum(stop.to(torch.int64), 1) == 0
                w = am * Tin[:, :-1] * alive
                acc = w @ colors[ids]
                last = torch.where(alive, one_m, torch.ones_like(one_m))
                T = torch.prod(last, 1)
                with torch.no_grad():
                    m_alpha = ((alpha - ALPHA_T).abs() / ALPHA_T)
                    m_hit = hit_t.abs() / (hit_t.abs().max() + 1e-30)
                    m_T = (Tin[:, 1:] - T_STOP).abs() / T_STOP
                    m_clamp = (raw - MAX_ALPHA).abs() / MAX_ALPHA
                    live = torch.cat([torch.ones(len(pid), 1, dtype=torch.bool), alive[:, :-1]], 1) & rok[pid][:, None]
                    mm = torch.minimum(torch.minimum(m_alpha, m_clamp), torch.where(use, m_T, torch.full_like(m_T, float("inf"))))
                    mm = torch.minimum(mm, torch.where(raw >= ALPHA_T, m_hit * 1e3, torch.full_like(m_hit, float("inf"))))
                    mm = torch.where(live, mm, torch.full_like(mm, float("inf")))
                    margins.view(-1)[pid] = mm.min(1).values
            cols = acc + (T[:, None] * bg[None] if bg is not None else 0)
            rows_c.append((pid, cols, (1 - T)[:, None]))
    del out_c
    flat_c = img.reshape(-1, D).clone()
    flat_a = alp.reshape(-1, 1).clone()
    for pid, cols, a in rows_c:
        flat_c = flat_c.index_put((pid,), cols)
        flat_a = flat_a.index_put((pid,), a)
    return flat_c.reshape(H, W, D), flat_a.reshape(H, W, 1), margins
