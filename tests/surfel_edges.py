"""Adversarial sweep for the 2DGS (surfel) kernels of gsplat_b200/csrc/surfel.cu and its float64 truth (no GPU needed).

Projection rows are built in the camera space of the sweep's first camera and mapped to world space through its pose;
every row carries its class: near / far plane, dist ~ 0 (the camera close to the surfel's plane: dist = M2 . (1, 1, -1)
. M2, the denominator of the screen mean), the ceil of 3.33 sqrt(ext) next to an integer, the 1e-4 floor of ext,
radius_clip, the four off-screen tests, radii of 2^31 or more, the sign of cosv (the normal flip), unnormalised
quaternions and bulk rows.  Every row has a non-zero scales[..., 2], which the kernels must ignore.

Compositing is checked on five screen-space images (means2d, ray transforms, normals, colours, opacities), each
45 x 37 (3 x 3 tiles, partial in both directions) with every tile listing every surfel of its image in depth order,
built from dyadic numbers so that float32 evaluates their decisions exactly: g3 == g2 at every pixel (the kernel
choice), T == 0.5 before a surfel (the median rule), next_T == float32(1e-4) (the transmittance stop), a surfel whose
alpha is clamped at 0.99 on every pixel, and a sub-pixel surfel drawn by the screen-space filter alone.  A sweep of
single surfels and depth-sorted stacks with per-pixel float64 budgets is not part of this module.

The truth is oracle/surfel.py in float64 on the float32 inputs; every threshold is the float32 value the kernels compare
with.  Budgets: every quantity is re-evaluated at N_PERTURB seeded relative perturbations of the float32 inputs of
4 * 2^-24; its budget is 4x the largest deviation plus a few ulp of its own magnitude (of the sum of the absolute values
of its terms where it cancels: dist, ext, the screen mean, cosv).  A row or pixel is
*decided* when every margin on its path exceeds its budget.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import surfel

f64 = torch.float64
ULP = 2.0**-24
INT32_MAX = 2**31 - 1
N_PERTURB = 6


def F32(v):
    return float(np.float32(v))


NEAR, FAR = F32(0.01), F32(100.0)
EXTEND = F32(3.33)
FLOOR = F32(1e-4)
ALPHA_TH = F32(np.float32(1.0) / np.float32(255.0))
MAX_ALPHA = F32(0.99)
T_TH = F32(1e-4)
RCLIP = 3.0
W, H = 320, 240  # projection image
IW, IH = 45, 37  # compositing images: 3 x 3 tiles, partial in both directions


def _rot(axis, angle):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K


def _camera(fx, fy, cx, cy, R, t):
    vm = np.eye(4)
    vm[:3, :3], vm[:3, 3] = R, t
    vm = vm.astype(np.float32)
    if R[2, 2] == 1.0:
        vm[2, :] = (0.0, 0.0, 1.0, 0.0)  # an exact depth row
    return vm, np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)


# cam0: off-centre principal point, fx != fy, rotated about the optical axis; cam1: the second camera of the C = 2 runs
CAMS = (
    _camera(500.0, 560.0, 150.5, 130.25, _rot((0, 0, 1), 0.3), (0.2, -0.1, 0.0)),
    _camera(420.0, 420.0, 160.0, 120.0, _rot((0.3, 1.0, 0.2), 0.12), (0.1, 0.05, 0.3)),
)


def camera_arrays(C):
    return (np.ascontiguousarray(np.stack([CAMS[c][0] for c in range(C)])),
            np.ascontiguousarray(np.stack([CAMS[c][1] for c in range(C)])))


def _quat_rot(q):
    q = q / np.sqrt((q * q).sum(-1, keepdims=True))
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    return np.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y),
    ], -1).reshape(q.shape[:-1] + (3, 3))


def _quantities(means, quats, scales, viewmats, Ks):
    """float64 decision quantities [C, N] of the projection and their term sizes (for the budgets)"""
    with np.errstate(all="ignore"):
        Rq = _quat_rot(quats)
        a, b, n = Rq[..., 0] * scales[:, :1], Rq[..., 1] * scales[:, 1:2], Rq[..., 2]
        R, t = viewmats[:, :3, :3], viewmats[:, :3, 3]
        ca, cb, cn = (np.einsum("cij,nj->cni", R, v) for v in (a, b, n))
        mc = np.einsum("cij,nj->cni", R, means) + t[:, None, :]
        Tc = np.stack([ca, cb, mc], -1)  # [C, N, 3 (xyz), 3 (ca cb mc)]
        fx, fy, cx, cy = (Ks[:, i, j][:, None, None] for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
        T0, T1, T2 = fx * Tc[..., 0, :] + cx * Tc[..., 2, :], fy * Tc[..., 1, :] + cy * Tc[..., 2, :], Tc[..., 2, :]
        sg = np.array([1.0, 1.0, -1.0])
        dist = (T2 * T2 * sg).sum(-1)
        dist_abs = (T2 * T2).sum(-1)
        m2 = np.stack([(T0 * T2 * sg).sum(-1), (T1 * T2 * sg).sum(-1)], -1) / dist[..., None]
        m2_abs = np.stack([np.abs(T0 * T2).sum(-1), np.abs(T1 * T2).sum(-1)], -1) / np.abs(dist)[..., None]
        m2_abs = m2_abs + np.abs(m2) * (dist_abs / np.abs(dist))[..., None]  # the error of 1 / dist, relative
        tmp = np.stack([(T0 * T0 * sg).sum(-1), (T1 * T1 * sg).sum(-1)], -1) / dist[..., None]
        ext = m2 * m2 - tmp
        ext_abs = m2 * m2 + np.stack([(T0 * T0).sum(-1), (T1 * T1).sum(-1)], -1) / np.abs(dist)[..., None]
        arg = EXTEND * np.sqrt(np.maximum(FLOOR, ext))
        cosv = -(cn * mc).sum(-1)
        cosv_abs = np.abs(cn * mc).sum(-1)
        z = mc[..., 2]
        z_abs = np.abs(np.einsum("cj,nj->cnj", R[:, 2], means)).sum(-1) + np.abs(t[:, 2])[:, None]
    return dict(z=z, z_abs=z_abs, dist=dist, dist_abs=dist_abs, m2=m2, m2_abs=m2_abs, ext=ext, ext_abs=ext_abs, arg=arg,
                cosv=cosv, cosv_abs=cosv_abs)


# ------------------------------------------------------------------------------------------------------------------
# projection rows
class _Rows:
    def __init__(self, rng):
        self.rng, self.rows = rng, []
        vm = CAMS[0][0].astype(np.float64)
        self.R, self.t = vm[:3, :3], vm[:3, 3]

    def add(self, cls, pc, s0, s1, quat=None):
        rng = self.rng
        if quat is None:
            quat = rng.standard_normal(4)
            quat /= np.linalg.norm(quat)
        mean = self.R.T @ (np.asarray(pc, np.float64) - self.t)
        self.rows.append((cls, mean, np.asarray(quat, np.float64), np.array([s0, s1, rng.uniform(0.01, 3.0)])))

    def arrays(self):
        f = lambda k: np.ascontiguousarray(np.array([r[k] for r in self.rows], np.float64).astype(np.float32))  # noqa: E731
        return dict(cls=np.array([r[0] for r in self.rows]), means=f(1), quats=f(2), scales=f(3))


def _facing_quat(tilt, axis_angle, roll):
    """a world quaternion whose normal makes an angle `tilt` with camera 0's optical axis (through the pose), tilted
    about the camera-frame axis (cos axis_angle, sin axis_angle, 0) after a roll about the optical axis"""
    R0 = CAMS[0][0][:3, :3].astype(np.float64)
    Rc = _rot((math.cos(axis_angle), math.sin(axis_angle), 0.0), tilt) @ _rot((0, 0, 1), roll)
    Rw = R0.T @ Rc
    w = math.sqrt(max(1e-12, 1 + Rw[0, 0] + Rw[1, 1] + Rw[2, 2])) / 2
    if w < 1e-3:  # no accurate quaternion from this branch of the conversion: a rotation about a nearby axis instead
        return _facing_quat(tilt, axis_angle, roll + 0.5)
    return np.array([w, (Rw[2, 1] - Rw[1, 2]) / (4 * w), (Rw[0, 2] - Rw[2, 0]) / (4 * w), (Rw[1, 0] - Rw[0, 1]) / (4 * w)])


def _facing(rng, tilt):
    return _facing_quat(tilt, rng.uniform(0, 2 * math.pi), rng.uniform(0, 2 * math.pi))


def _solve(f, lo, hi, target, iters=200):
    """bisection for f(x) = target on [lo, hi] (f monotone)"""
    flo = f(lo) - target
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        fm = f(mid) - target
        if (fm > 0) == (flo > 0):
            lo, flo = mid, fm
        else:
            hi = mid
    return 0.5 * (lo + hi)


def _row_q(pc, quat, s0, s1):
    """decision quantities of one row under camera 0 (camera-space centre pc)"""
    vm, K = CAMS[0]
    vm64 = vm.astype(np.float64)
    mean = vm64[:3, :3].T @ (np.asarray(pc, np.float64) - vm64[:3, 3])
    q = _quantities(mean[None], np.asarray(quat, np.float64)[None], np.array([[s0, s1, 1.0]]), vm64[None], K.astype(np.float64)[None])
    return {k: v[0, 0] for k, v in q.items()}


def make_rows(seed=20261016, n_each=10, n_bulk=64):
    rng = np.random.RandomState(seed)
    r = _Rows(rng)
    fx, fy = float(CAMS[0][1][0, 0]), float(CAMS[0][1][1, 1])

    def on_screen(z, spread=0.2):
        return np.array([rng.uniform(-spread, spread) * z, rng.uniform(-spread, spread) * z, z])

    cx, cy = float(CAMS[0][1][0, 2]), float(CAMS[0][1][1, 2])

    def near_corner(z, lo, hi):
        # a camera-space centre that projects at (lo .. hi) pixels from the image origin, where ext = m2^2 - tmp
        # cancels least
        return np.array([(rng.uniform(lo, hi) - cx) / fx * z, (rng.uniform(lo, hi) - cy) / fy * z, z])

    # near / far: a few ulp to 1e-3 relative around the planes (the depth row of camera 0 is exact)
    for plane in (NEAR, FAR):
        for i in range(n_each):
            d = (1e-6, -1e-6, 1e-5, -1e-5, 1e-4, -1e-4, 1e-3, -1e-3, 0.0, 3e-7)[i % 10]
            z = plane * (1 + d)
            r.add("near" if plane == NEAR else "far", on_screen(z), z * 0.02, z * 0.03, quat=_facing(rng, 0.3))
    # dist == 0 exactly, and dist ~ 0: the world quaternion (1, 1, 1, 1) / 2 has the exact rotation whose second
    # column is (0, 0, 1), and camera 0's depth row is exactly (0, 0, 1, 0), so T2 = (0, s1, z) in float32 as in
    # float64 and dist = s1^2 - z^2: zero for s1 == z (the kernels cull the row), a chosen relative distance otherwise
    for i in range(n_each):
        z = F32(rng.uniform(1.0, 5.0))
        r.add("dist==0", on_screen(z, 0.05), rng.uniform(0.01, 0.1) * z, z, quat=(0.5, 0.5, 0.5, 0.5))
    for i in range(2 * n_each):
        z = F32(rng.uniform(1.0, 5.0))
        rel = (5e-1, -5e-1, 3e-1, -3e-1, 2e-1, -2e-1, 1e-1, -1e-1, 1e-2, -1e-2)[i % 10]
        r.add("dist~0", on_screen(z, 0.05), rng.uniform(0.01, 0.1) * z, z * math.sqrt(1 + rel), quat=(0.5, 0.5, 0.5, 0.5))
    # ceil: 3.33 sqrt(ext) within 3e-2 .. 1e-4 of an integer, on both sides (rows whose bisection misses are skipped)
    n_ceil = 0
    for i in range(6 * n_each):
        if n_ceil == 2 * n_each:
            break
        z = rng.uniform(0.5, 10.0)
        q = _facing(rng, rng.uniform(0.0, 1.0))
        on = near_corner(z, 15.0, 40.0)
        k = int(rng.randint(1, 12))
        eps = (3e-2, -3e-2, 1e-2, -1e-2, 3e-3, -3e-3, 1e-3, -1e-3, 1e-4, -1e-4)[n_ceil % 10]
        an = rng.uniform(0.3, 1.0)
        f = lambda s: _row_q(on, q, s, an * s)["arg"].max()  # noqa: E731
        s = _solve(f, 1e-6 * z, 10.0 * z, k + eps)
        if abs(f(s) - (k + eps)) > 1e-7:
            continue
        r.add("ceil", on, s, an * s, quat=q)
        n_ceil += 1
    # the 1e-4 floor of ext: sub-pixel surfels whose ext is around 1e-4
    for i in range(2 * n_each):
        z = rng.uniform(0.5, 10.0)
        q = _facing(rng, rng.uniform(0.0, 0.8))
        on = near_corner(z, 1.0, 3.0)
        rel = (0.5, 2.0, 0.9, 1.1, 0.97, 1.03, 0.99, 1.01, 0.1, 10.0)[i % 10]
        f = lambda s: _row_q(on, q, s, 0.7 * s)["ext"].max()  # noqa: E731
        s = _solve(f, 1e-9 * z, 1e-1 * z, FLOOR * rel)
        r.add("floor", on, s, 0.7 * s, quat=q)
    # radius_clip (RCLIP = 3): max radius 2, 3 (culled: fr <= radius_clip) and 4
    for i in range(2 * n_each):
        z = rng.uniform(0.5, 10.0)
        q = _facing(rng, rng.uniform(0.0, 0.6))
        on = on_screen(z)
        target = (2.5, 2.9, 3.0 - 0.3, 3.5, 3.9, 2.2)[i % 6]
        an = rng.uniform(0.3, 1.0)
        f = lambda s: _row_q(on, q, s, an * s)["arg"].max()  # noqa: E731
        s = _solve(f, 1e-6 * z, 10.0 * z, target)
        r.add("radius_clip", on, s, an * s, quat=q)
    # off-screen: m2 +- radius against 0, W, H, 1e-2 .. 1e-5 pixels inside and outside
    for i in range(4 * n_each):
        side = i % 4
        z = rng.uniform(1.0, 10.0)
        q = _facing(rng, rng.uniform(0.0, 0.8))
        s = rng.uniform(0.002, 0.03) * z
        d = (1e-2, -1e-2, 1e-3, -1e-3, 1e-4, -1e-4, 3e-5, -3e-5)[(i // 4) % 8]
        other = on_screen(z)

        def edge(x, side=side, z=z, q=q, s=s, other=other):
            pc = other.copy()
            pc[side // 2] = x
            qq = _row_q(pc, q, s, 0.8 * s)
            fr = math.ceil(qq["arg"][side // 2])
            m = qq["m2"][side // 2]
            return m + fr if side % 2 == 0 else m - fr - (W if side // 2 == 0 else H)

        x = _solve(lambda x: edge(x), -3.0 * z, 3.0 * z, d)
        pc = other.copy()
        pc[side // 2] = x
        r.add("offscreen", pc, s, 0.8 * s, quat=q)
    # radii of 2^31 or more: face-on, scales 1e7 at z = 2 (ext ~ 1e19 fits float32; rx saturates to INT32_MAX)
    for _ in range(n_each):
        r.add("radius>=2^31", on_screen(2.0, 0.05), 1e7, 1e7 * rng.uniform(0.5, 1.0), quat=_facing(rng, 0.0))
    # the sign of cosv: the surfel's plane passes close to the camera centre; the tilt is solved so that cosv is a
    # chosen fraction of the sum of its terms' absolute values, on both sides of the flip
    for i in range(2 * n_each):
        z = rng.uniform(1.0, 5.0)
        on = on_screen(z, 0.05)
        rel = (1e-2, -1e-2, 1e-3, -1e-3, 1e-4, -1e-4, 1e-5, -1e-5, 1e-6, -1e-6)[i % 10]
        ax, roll = rng.uniform(0, 2 * math.pi), rng.uniform(0, 2 * math.pi)

        def cosv_rel(tilt, on=on, ax=ax, roll=roll):
            qq = _row_q(on, _facing_quat(tilt, ax, roll), 0.05, 0.02)
            return qq["cosv"] / qq["cosv_abs"]

        lo, hi = math.pi / 2 - 0.3, math.pi / 2 + 0.3
        if (cosv_rel(lo) - rel) * (cosv_rel(hi) - rel) > 0:
            continue
        t = _solve(cosv_rel, lo, hi, rel)
        r.add("cosv", on, 0.05 * z, 0.02 * z, quat=_facing_quat(t, ax, roll))
    # unnormalised quaternions (norms 1e-3 .. 1e3)
    for _ in range(2 * n_each):
        z = rng.uniform(0.5, 10.0)
        r.add("quat_norm", on_screen(z), 0.02 * z, 0.01 * z, quat=rng.standard_normal(4) * 10.0 ** rng.uniform(-3, 3))
    for _ in range(n_bulk):
        z = 10.0 ** rng.uniform(-0.3, 1.3)
        r.add("bulk", on_screen(z, 0.4), z * 10.0 ** rng.uniform(-3, -1), z * 10.0 ** rng.uniform(-3, -1))
    return r.arrays()


CLASS_MIN = {"near": 10, "far": 10, "dist==0": 8, "dist~0": 10, "ceil": 10, "floor": 10, "radius_clip": 10, "offscreen": 20,
             "radius>=2^31": 8, "cosv": 10, "quat_norm": 10, "bulk": 32}


def subset(rows, idx):
    return {k: np.ascontiguousarray(v[idx]) for k, v in rows.items()}


def _perturb(arrs, k):
    """float64 copies of the float32 inputs; k > 0: relative perturbation of 4 ulp (seeded)"""
    out = {key: np.asarray(v, np.float64) for key, v in arrs.items()}
    if k:
        rng = np.random.RandomState(1000 + k)
        out = {key: v * (1.0 + 4.0 * ULP * rng.uniform(-1, 1, v.shape)) for key, v in out.items()}
    return out


def _spread(base, vals):
    with np.errstate(invalid="ignore"):
        return np.nan_to_num(np.max([np.abs(v - base) for v in vals], 0), nan=np.inf)


def _project64(p, radius_clip, grad=False):
    t = {k: torch.tensor(p[k], dtype=f64, requires_grad=grad) for k in ("means", "quats", "scales", "viewmats", "Ks")}
    out = surfel.project(t["means"], t["quats"], t["scales"], t["viewmats"], t["Ks"], W, H, NEAR, FAR, radius_clip)
    return t, out


class Truth:
    pass


def truth(rows, C, radius_clip=0.0):
    """float64 truth of the rows under the first C cameras: radii, means2d, depths, ray_transforms, normals [C, N, *],
    their budgets, decided [C, N] and the class of each row."""
    vm, Ks = camera_arrays(C)
    arrs = dict(means=rows["means"], quats=rows["quats"], scales=rows["scales"], viewmats=vm, Ks=Ks)
    qs, outs = [], []
    for k in range(N_PERTURB + 1):
        p = _perturb(arrs, k)
        qs.append(_quantities(p["means"], p["quats"], p["scales"], p["viewmats"], p["Ks"]))
        with np.errstate(all="ignore"):
            outs.append([o.detach().numpy() for o in _project64(p, radius_clip)[1]])
    q, sp = qs[0], {key: _spread(qs[0][key], [x[key] for x in qs[1:]]) for key in qs[0]}
    beta = lambda key, ab, u=8.0: 4.0 * sp[key] + u * ULP * np.abs(ab)  # noqa: E731
    with np.errstate(all="ignore"):
        b_z = beta("z", q["z_abs"])
        depth_ok = (np.abs(q["z"] - NEAR) > b_z) & (np.abs(q["z"] - FAR) > b_z)
        in_depth = ~((q["z"] <= NEAR) | (q["z"] >= FAR))
        dist_ok = np.abs(q["dist"]) > beta("dist", q["dist_abs"])
        b_ext = beta("ext", q["ext_abs"], 16.0)
        sq = np.sqrt(np.maximum(FLOOR, q["ext"]))
        b_arg = 4.0 * sp["arg"] + EXTEND * b_ext / (2 * sq) + 8 * ULP * q["arg"]
        floored = q["ext"] < FLOOR
        frac_ok = np.abs(q["arg"] - np.round(q["arg"])) > b_arg
        ceil_ok = np.where(floored, np.abs(q["ext"] - FLOOR) > b_ext, frac_ok | (q["arg"] - b_arg > 2.0**31))
        ceil_ok = ceil_ok.all(-1)
        fr = np.ceil(q["arg"])
        b_m2 = beta("m2", q["m2_abs"], 16.0)
        edges = np.stack([q["m2"][..., 0] + fr[..., 0], q["m2"][..., 0] - fr[..., 0] - W, q["m2"][..., 1] + fr[..., 1],
                          q["m2"][..., 1] - fr[..., 1] - H], -1)
        off_ok = (np.abs(edges) > np.repeat(b_m2, 2, -1)).all(-1)
        cos_ok = np.abs(q["cosv"]) > beta("cosv", q["cosv_abs"])
    # the oracle's margins: its ceil budget (1e-6 of the terms of ext) must also hold
    ceil_m, screen_m, depth_m = (x.numpy() for x in surfel.project_margins(
        *(torch.tensor(v, dtype=f64) for v in (rows["means"], rows["quats"], rows["scales"], vm, Ks)), W, H, NEAR, FAR))
    ceil_ok &= (ceil_m > 1.0) | (q["arg"] - b_arg > 2.0**31).all(-1)
    # dist exactly 0 is decided: the rows built for it are exact in float32 (see make_rows), and the kernels cull them
    dist_zero = q["dist"] == 0
    decided = depth_ok & (~in_depth | dist_zero | (dist_ok & ceil_ok & off_ok & cos_ok & (screen_m > 0) & (depth_m > 0)))
    radii, m2, dep, rt, nrm = outs[0]
    # radii: the float64 ceil, saturated like cvt.rzi.s32.f32
    vis = (radii != 0).all(-1)
    radii = np.where(vis[..., None], np.minimum(fr, INT32_MAX), 0).astype(np.int64)
    tr = Truth()
    tr.cls, tr.decided, tr.vis, tr.q = rows["cls"], decided, vis, q
    tr.radii, tr.means2d, tr.depths, tr.ray_transforms, tr.normals = radii, m2, dep, rt, nrm
    with np.errstate(all="ignore"):
        Mabs = np.abs(rt)
        tr.beta = dict(
            means2d=4.0 * _spread(m2, [o[1] for o in outs[1:]]) + 16 * ULP * q["m2_abs"],
            depths=4.0 * _spread(dep, [o[2] for o in outs[1:]]) + 8 * ULP * q["z_abs"],
            ray_transforms=4.0 * _spread(rt, [o[3] for o in outs[1:]]) + 16 * ULP * Mabs.max(-1, keepdims=True) * 4,
            normals=4.0 * _spread(nrm, [o[4] for o in outs[1:]]) + 16 * ULP,
        )
    tr.inputs = arrs
    return tr


def describe(rows, tr, c, n):
    return (f"row {n} (class {tr.cls[n]}, camera {c}, mean={rows['means'][n].tolist()}, quat={rows['quats'][n].tolist()}, "
            f"scale={rows['scales'][n].tolist()})")


def check_projection(rows, tr, radii, means2d, depths, ray_transforms, normals, what):
    """float32 forward outputs [C, N, *] against the truth on decided rows; returns failure messages"""
    msgs = []
    dec = tr.decided
    radii = np.asarray(radii).astype(np.int64)
    bad = dec & (radii != tr.radii).any(-1)
    if bad.any():
        c, n = np.argwhere(bad)[0]
        msgs.append(f"{what}: {int(bad.sum())} decided rows with wrong radii, e.g. {describe(rows, tr, c, n)}: "
                    f"got {radii[c, n].tolist()}, truth {tr.radii[c, n].tolist()}")
    culled = (radii == 0).all(-1)
    for name, got in (("means2d", means2d), ("depths", depths), ("ray_transforms", ray_transforms), ("normals", normals)):
        got = np.asarray(got, np.float64)
        ref, b = getattr(tr, name), tr.beta[name]
        g, r_ = got.reshape(got.shape[:2] + (-1,)), ref.reshape(ref.shape[:2] + (-1,))
        bb = np.broadcast_to(b.reshape(b.shape[:2] + (-1,)), g.shape)
        with np.errstate(invalid="ignore"):
            bad = dec & tr.vis & ~(np.abs(g - r_) <= bb).all(-1)
        bad_c = culled & (g != 0).any(-1)
        if bad.any():
            c, n = np.argwhere(bad)[0]
            msgs.append(f"{what}: {int(bad.sum())} decided rows with {name} out of budget, e.g. {describe(rows, tr, c, n)}: "
                        f"got {g[c, n].tolist()}, truth {r_[c, n].tolist()}, beta {bb[c, n].tolist()}")
        if bad_c.any():
            c, n = np.argwhere(bad_c)[0]
            msgs.append(f"{what}: {int(bad_c.sum())} culled rows with non-zero {name}, e.g. {describe(rows, tr, c, n)}")
    return msgs


def undecided_report(tr):
    """per class: (rows, undecided (camera, row) pairs, pairs)"""
    out = {}
    for k in np.unique(tr.cls):
        sel = tr.cls == k
        out[str(k)] = (int(sel.sum()), int((~tr.decided[:, sel]).sum()), int(tr.decided[:, sel].size))
    return out


def cotangents(shape_lead, seed=0):
    rng = np.random.RandomState(seed)
    return dict(means2d=rng.standard_normal(shape_lead + (2,)), depths=rng.standard_normal(shape_lead),
                ray_transforms=rng.standard_normal(shape_lead + (3, 3)), normals=rng.standard_normal(shape_lead + (3,)))


def grad_truth(rows, tr, radius_clip, cot):
    """float64 gradients for the cotangents `cot` [C, N, *] (zeroed off the decided visible rows; returned as float32,
    which is what the kernels get): v_means, v_quats, v_scales [N, *], v_viewmats [C, 4, 4], and their budgets:
    4x the spread over the perturbations + 64 ulp of the surfel's largest gradient of that kind; v_viewmats: the l1 of
    the per-row budgets of its shares + 64 ulp of the l1 of the shares."""
    keep = tr.decided & tr.vis
    cot32 = {k: (v * keep.reshape(keep.shape + (1,) * (v.ndim - 2))).astype(np.float32) for k, v in cot.items()}
    N = rows["means"].shape[0]
    res = []
    for k in range(N_PERTURB + 1):
        p = _perturb(tr.inputs, k)
        # one row per batch element, so that the viewmats gradient of each row (its share) is known
        pb = dict(means=p["means"][:, None], quats=p["quats"][:, None], scales=p["scales"][:, None],
                  viewmats=np.broadcast_to(p["viewmats"][None], (N,) + p["viewmats"].shape).copy(),
                  Ks=np.broadcast_to(p["Ks"][None], (N,) + p["Ks"].shape).copy())
        with np.errstate(all="ignore"):
            t, out = _project64(pb, radius_clip, grad=True)
        loss = 0.0
        for name, o in zip(("means2d", "depths", "ray_transforms", "normals"), out[1:]):
            c = torch.tensor(np.swapaxes(cot32[name], 0, 1), dtype=f64)[:, :, None]  # [N, C, 1, ...]
            loss = loss + (o * c).sum()
        g = torch.autograd.grad(loss, [t["means"], t["quats"], t["scales"], t["viewmats"]])
        res.append(dict(v_means=g[0][:, 0].numpy(), v_quats=g[1][:, 0].numpy(), v_scales=g[2][:, 0].numpy(),
                        shares=g[3].numpy().reshape(N, -1)))
    grads, betas = {}, {}
    for key in ("v_means", "v_quats", "v_scales"):
        base = res[0][key]
        grads[key] = base
        betas[key] = 4.0 * _spread(base, [r[key] for r in res[1:]]) + 64 * ULP * np.abs(base).max(-1, keepdims=True)
    sh = res[0]["shares"]
    b_sh = 4.0 * _spread(sh, [r["shares"] for r in res[1:]]) + 64 * ULP * np.abs(sh).max(-1, keepdims=True)
    C = tr.decided.shape[0]
    grads["v_viewmats"] = sh.sum(0).reshape(C, 4, 4)
    betas["v_viewmats"] = (b_sh.sum(0) + 64 * ULP * np.abs(sh).sum(0)).reshape(C, 4, 4)
    return grads, betas, cot32


def check_grads(rows, tr, got, ref, beta, what):
    msgs = []
    for k, g in got.items():
        g = np.asarray(g, np.float64)
        with np.errstate(invalid="ignore"):
            bad = ~(np.abs(g - ref[k]) <= beta[k])
        if k != "v_viewmats":
            bad = bad.any(-1)
        if bad.any():
            i = tuple(np.argwhere(bad)[0])
            who = describe(rows, tr, 0, i[0]) if k != "v_viewmats" else f"entry {i}"
            msgs.append(f"{what}: {int(bad.sum())} {k} out of budget, e.g. {who}: got {g[i].tolist()}, truth "
                        f"{ref[k][i].tolist()}, beta {beta[k][i].tolist()}")
    return msgs


# ------------------------------------------------------------------------------------------------------------------
# compositing: exact ties in screen space
def _rt(a, b, c, d, x, y):
    """ray transform [[a, b, x], [c, d, y], [0, 0, 1]]: screen mean (x, y), (u, v) = [[a, b], [c, d]]^-1 (x - px, y - py)"""
    return np.array([[a, b, x], [c, d, y], [0.0, 0.0, 1.0]], np.float32)


# next_T == float32(1e-4) exactly after the fifth surfel of the stop image, at its centre pixel (alpha == opacity
# there, since g3 == g2 == 0 and exp(-0) == 1): found by a search over float32 opacities
STOP_OPACITIES = (0.9, 0.9, 0.9, 0.899, 0.009901762)


def tie_images(D=3, seed=5):
    """Five 45 x 37 images whose decisions fall exactly on a threshold, in float32 as in float64 (dyadic inputs):
      0 "branch": one surfel with g3 == g2 at every pixel: (u, v) = (p + q, p - q), so u^2 + v^2 = 2 (p^2 + q^2);
      1 "median": opacities 0.5, 0.25 centred on pixel (10, 12): T == 0.5 exactly before the second surfel;
      2 "stop": STOP_OPACITIES centred on pixel (30, 20): next_T == float32(1e-4) exactly at the fifth surfel;
      3 "clamp": one surfel of opacity 1 so large that raw alpha > 0.99 on every pixel;
      4 "filter": a sub-pixel surfel, (u, v) = 64 (p, q), so g3 = 2048 g2 > g2 at every pixel: the screen-space filter.
    Returns dense [5, 5, *] inputs, flatten_ids / isect_offsets listing every surfel of an image on each of its
    tiles (depth order) and the centre pixel (x, y) of each image."""
    rng = np.random.RandomState(seed)
    I, N = 5, 5
    m2 = np.zeros((I, N, 2), np.float32)
    rt = np.zeros((I, N, 3, 3), np.float32)
    op = np.zeros((I, N), np.float32)
    counts = [1, 2, 5, 1, 1]
    centres = [(20, 17), (10, 12), (30, 20), (22, 18), (12, 9)]
    x, y = 20.25, 17.75
    m2[0, 0], rt[0, 0], op[0, 0] = (x, y), _rt(0.5, 0.5, 0.5, -0.5, x, y), 0.8
    for n, o in enumerate((0.5, 0.25)):
        m2[1, n], rt[1, n], op[1, n] = (10.5, 12.5), _rt(4.0, 0.0, 0.0, 4.0, 10.5, 12.5), o
    for n, o in enumerate(STOP_OPACITIES):
        m2[2, n], rt[2, n], op[2, n] = (30.5, 20.5), _rt(8.0, 0.0, 0.0, 8.0, 30.5, 20.5), o
    m2[3, 0], rt[3, 0], op[3, 0] = (22.5, 18.5), _rt(1024.0, 0.0, 0.0, 1024.0, 22.5, 18.5), 1.0
    m2[4, 0], rt[4, 0], op[4, 0] = (12.25, 9.75), _rt(1.0 / 64, 0.0, 0.0, 1.0 / 64, 12.25, 9.75), 0.9
    colors = rng.random_sample((I, N, D)).astype(np.float32)
    colors[..., -1] = np.arange(1, N + 1, dtype=np.float32)[None] * 0.5 + 1.0  # depth channel, increasing
    nrm = rng.standard_normal((I, N, 3)).astype(np.float32)
    ids, offs = [], []
    for i in range(I):
        for _ in range(9):
            offs.append(len(ids))
            ids.extend(i * N + n for n in range(counts[i]))
    return dict(means2d=m2, ray_transforms=rt, opacities=op, colors=colors, normals=nrm,
                flatten_ids=np.array(ids, np.int32), isect_offsets=np.array(offs, np.int32).reshape(I, 3, 3),
                counts=counts, centres=centres)


def stop_chain_float32():
    """(index of the last contributor, T after it) of the stop image's centre pixel, evaluated like the kernel"""
    f = np.float32
    T, last = f(1.0), -1
    for k, o in enumerate(STOP_OPACITIES):
        nxt = f(T * f(f(1.0) - f(min(f(MAX_ALPHA), f(o)))))
        if nxt <= f(T_TH):
            break
        T, last = nxt, k
    return last, T


# ------------------------------------------------------------------------------------------------------------------
# the non-finite hazard: finite inputs whose float32 projection overflows
def overflow_rows(n=12, seed=9):
    """surfels facing camera 0 with scales 1e37 .. 3e38: fx * scale overflows float32 for any fx above 34, so M0 / M1
    hold inf and the screen mean is inf * 0 = NaN in float32 (the float64 values are finite but beyond float32's range)"""
    rng = np.random.RandomState(seed)
    r = _Rows(rng)
    for i in range(n):
        z = rng.uniform(1.0, 5.0)
        s = (1e37, 3e37, 3e38)[i % 3]
        pc = np.array([rng.uniform(-0.2, 0.2) * z, rng.uniform(-0.2, 0.2) * z, z])
        r.add("overflow", pc, s, s * rng.uniform(0.5, 1.0), quat=_facing(rng, 0.0) if i % 2 else (1.0, 0.0, 0.0, 0.0))
    return r.arrays()


def ext_overflow_rows(n=12, seed=11):
    """surfels facing camera 0 with scales 1e19 .. 1e21: the ray transform (about fx * scale) fits float32 but
    its square in ext = m2^2 - tmp overflows, so the float32 radius is not the float64 one: ext is +-inf or NaN"""
    rng = np.random.RandomState(seed)
    r = _Rows(rng)
    for i in range(n):
        z = rng.uniform(1.0, 5.0)
        s = (1e19, 1e20, 1e21)[i % 3]
        pc = np.array([rng.uniform(-0.2, 0.2) * z, rng.uniform(-0.2, 0.2) * z, z])
        r.add("ext_overflow", pc, s, s * rng.uniform(0.5, 1.0), quat=(1.0, 0.0, 0.0, 0.0) if i % 2 else _facing(rng, 0.0))
    return r.arrays()


def radii_float32(rows, C):
    """the projection's radii [C, N, 2] evaluated in float32 with the kernel's order of operations (no culls), for
    rows whose outcome float32 overflow decides: ceil(3.33 sqrt(fmax(1e-4, ext))), saturated to INT32_MAX; and whether
    the screen mean and the ray transform are finite [C, N]"""
    f = np.float32
    vm, Ks = camera_arrays(C)
    with np.errstate(all="ignore"):
        q = rows["quats"].astype(f)
        q = q * (f(1) / np.sqrt((q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3] + q[:, 0] * q[:, 0])))[:, None]
        Rq = _quat_rot(q.astype(np.float64)).astype(f)
        s = rows["scales"].astype(f)
        a, b, mean = Rq[..., 0] * s[:, :1], Rq[..., 1] * s[:, 1:2], rows["means"].astype(f)
        R, t = vm[:, :3, :3], vm[:, :3, 3]
        app = lambda v: (R[:, None, :, 0] * v[None, :, None, 0] + R[:, None, :, 1] * v[None, :, None, 1]  # noqa: E731
                         + R[:, None, :, 2] * v[None, :, None, 2])
        ca, cb, mc = app(a), app(b), app(mean) + t[:, None, :]
        out = []
        fx, fy, cx, cy = (Ks[:, i, j][:, None] for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
        T0 = [fx * v[..., 0] + cx * v[..., 2] for v in (ca, cb, mc)]
        T1 = [fy * v[..., 1] + cy * v[..., 2] for v in (ca, cb, mc)]
        T2 = [v[..., 2] for v in (ca, cb, mc)]
        dist = T2[0] * T2[0] + T2[1] * T2[1] - T2[2] * T2[2]
        inv = f(1) / dist
        fs = (inv, inv, -inv)
        for T in (T0, T1):
            m = fs[0] * T[0] * T2[0] + fs[1] * T[1] * T2[1] + fs[2] * T[2] * T2[2]
            e = m * m - (fs[0] * T[0] * T[0] + fs[1] * T[1] * T[1] + fs[2] * T[2] * T[2])
            fr = np.ceil(f(EXTEND) * np.sqrt(np.fmax(f(FLOOR), e)))
            out.append(np.where(fr >= 2.0**31, INT32_MAX, np.nan_to_num(fr, nan=0.0, posinf=0.0).astype(np.int64)))
            finite = np.isfinite(m) & np.isfinite(np.stack(T0 + T1 + T2)).all(0) if len(out) == 1 else finite & np.isfinite(m)
    return np.stack(out, -1), finite
