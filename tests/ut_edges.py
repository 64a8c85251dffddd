"""Adversarial sweep for the 3DGUT projection of gsplat_b200/csrc/ut.cu (ut_project_kernel through camera.cuh) and its
float64 truth (no GPU needed).  Global shutter; the perfect pinhole, a strongly distorted pinhole and a fisheye lens.

Rows are built in the camera space of one pose and mapped to world space through it: a quarter turn about the optical
axis (exact in float32) with a dyadic translation, an off-centre principal point and fx != fy.  Every row carries its
class: bulk, a sigma point on or near the margin edge (in_margin is half-open), a sigma point at z = 0 or behind the
camera, a sigma point's radial factor icD at or near 0.8 (distorted pinhole), a sigma point's angle near max_angle with
a negative k1 that ends the fisheye's monotone range inside the image, near / far planes, degenerate quaternions and
scales, a UT covariance that is not positive definite (the centre covariance weight is negative), opacity *
compensation near 1/255, the ceil of the radius and radius_clip near an integer, the four off-screen tests, and finite
inputs whose float32 transform overflows (the kernel must cull them).

Exact UT: alpha = 1, kappa = 1, beta = 0 give spread 2 and weights 1/4, 1/4, 1/8.  With the identity quaternion,
dyadic means and scales, power-of-two focal lengths and a dyadic principal point, the undistorted transform is exact in
float32, so the tie rows sit exactly on their threshold in float32 as in float64: a sigma point at u == -W m (valid),
at u == W + W m (invalid) and at z == 0 (behind).  A distorted sigma point whose icD is exactly float32(0.8)
on a lens with k1 = float32(0.8) - 1 at x / z == 1 is exact too.  The truth takes a tie as decided only under the exact
UT on the lens it is built for.

The truth is oracle.ut.ut_projection in float64 on the float32 inputs, with the UT parameters, planes, eps2d and
radius_clip at their float32 values.  Budgets: every decision quantity is re-evaluated under N_PERTURB seeded relative
perturbations of 4 * 2^-24 of every float32 input; its budget is 4x the largest deviation plus the float32 rounding of
its terms.  The UT mean and covariance are weighted sums that cancel (with the default parameters the centre weight is
-99 and the others 16.7), so their rounding is propagated from the sums of the absolute values of their terms:
    e_m2  = sum_k |w_k| e_u_k + 4 ulp sum_k |w_k u_k| + sum_k |w_k - w32_k| |u_k|
    e_cov = sum_k |wc_k| (2 |du_k| e_u_k + e_u_k^2) + 2 |sum_k wc_k du_k| e_m2 + |sum_k wc_k| e_m2^2
            + 2 e_m2 sum_k |wc_k| e_u_k + 4 ulp sum_k |wc_k| du_k^2
(the kernel's m2 error is common to every du_k = u_k - m2, so it enters through sum_k wc_k du_k and sum_k wc_k)
and det, det_orig, the compensation, the radius and the conic follow by first-order propagation.  A row is *decided*
when every margin on its path exceeds its budget: the degenerate and depth tests, each sigma point's validity as far as
the any / all rule needs it, then det, c00, c11, the opacity threshold, both ceils and the four off-screen tests.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np
import torch

from oracle import ut as U

f64 = torch.float64
f32 = np.float32
ULP = 2.0**-24
N_PERTURB = 6
FLT_EPS = float(np.finfo(np.float32).eps)
FLT_MAX = float(np.finfo(np.float32).max)


def F32(v):
    return float(np.float32(v))


ALPHA_TH = F32(f32(1.0) / f32(255.0))
EXTEND = F32(3.33)
MIN_COMP = F32(0.005)
FAR = 100.0
W, H = 320, 240

# a quarter turn about the optical axis and a dyadic translation: camera = R world + t, exact in float32
VM = np.array([[0, -1, 0, 0.25], [1, 0, 0, -0.125], [0, 0, 1, 0.5], [0, 0, 0, 1]], np.float32)

LENSES = {
    "pinhole": dict(kind="pinhole", f=(256.0, 512.0), coeffs={}),
    # k1 = float32(0.8) - 1 (exact): a sigma point at x / z == 1, y == 0 has icD == 1 + k1 == float32(0.8) exactly, in
    # float32 as in float64
    "distorted": dict(kind="pinhole", f=(128.0, 160.0),
                      coeffs=dict(radial=(F32(f32(0.8) - f32(1)), 0.0, 0.0, 0.0, 0.0, 0.0), tangential=(2.0**-7, -(2.0**-8)))),
    "fisheye": dict(kind="fisheye", f=(100.0, 112.0), coeffs=dict(radial=(-0.2, 0.0, 0.0, 0.0))),
}
CX, CY = 150.5, 130.25
COEFF_KEYS = {"radial": "radial_coeffs", "tangential": "tangential_coeffs", "thin": "thin_prism_coeffs"}

EXACT_UT = (1.0, 0.0, 1.0)  # alpha, beta, kappa
DEFAULT_UT = (0.1, 2.0, 0.0)
OTHER_UT = (0.5, 2.0, 1.0)
# beta < -(1 - alpha^2): the covariance's centre weight is below the mean's, so the UT covariance can be indefinite
NEG_BETA_UT = (0.1, -3.0, 0.0)
# (name, (alpha, beta, kappa), in_image_margin_factor, require_all, eps2d, radius_clip, near_plane)
PARAM_SETS = [
    ("default", DEFAULT_UT, 0.1, False, 0.3, 0.0, 0.01),
    ("default/all/m0.5/eps0", DEFAULT_UT, 0.5, True, 0.0, 0.0, 0.01),
    ("default/m0/clip3", DEFAULT_UT, 0.0, False, 0.3, 3.0, 0.01),
    ("exact/m0", EXACT_UT, 0.0, False, 0.3, 0.0, 0.01),
    ("exact/all/m0", EXACT_UT, 0.0, True, 0.3, 0.0, 0.01),
    ("exact/all/m0.5", EXACT_UT, 0.5, True, 0.3, 0.0, 0.01),
    ("exact/m0.5/eps0/near0.5", EXACT_UT, 0.5, False, 0.0, 0.0, 0.5),
    ("exact/all/m0.1/clip3", EXACT_UT, 0.1, True, 0.3, 3.0, 0.01),
    ("other/all/m0.1/clip3", OTHER_UT, 0.1, True, 0.3, 3.0, 0.01),
    ("other/m0/eps0/near0.5", OTHER_UT, 0.0, False, 0.0, 0.0, 0.5),
    ("negbeta/m0.5/eps0", NEG_BETA_UT, 0.5, False, 0.0, 0.0, 0.01),
]


def params(name):
    n, ut, m, req, eps2d, clip, near = next(p for p in PARAM_SETS if p[0] == name)
    return dict(name=n, ut=ut, margin=m, require_all=req, eps2d=eps2d, clip=clip, near=near)


def ut_namespace(P):
    a, b, k = P["ut"]
    return SimpleNamespace(alpha=a, beta=b, kappa=k, in_image_margin_factor=P["margin"],
                           require_all_sigma_points_valid=P["require_all"])


def K_of(lens):
    fx, fy = LENSES[lens]["f"]
    return np.array([[fx, 0, CX], [0, fy, CY], [0, 0, 1]], np.float32)


def camera(lens, K=None, coeffs=None):
    spec = LENSES[lens]
    K = K_of(lens) if K is None else K
    co = spec["coeffs"] if coeffs is None else coeffs
    return U.Camera(spec["kind"], np.asarray(K, np.float64), W, H,
                    **{k: [F32(x) for x in np.asarray(v).reshape(-1)] for k, v in co.items()})


def weights32(ut):
    """the kernel's float32 UT weights: (spread, w_mean0, w_cov0, w_rest)"""
    a, b, k = (f32(x) for x in ut)
    lam = f32(f32(a * a) * f32(f32(3) + k)) - f32(3)
    spread = np.sqrt(f32(f32(3) + lam))
    w_m0 = f32(lam / f32(f32(3) + lam))
    w_c0 = f32(w_m0 + f32(f32(f32(1) - f32(a * a)) + b))
    w_r = f32(f32(1) / f32(f32(2) * f32(f32(3) + lam)))
    return float(spread), float(w_m0), float(w_c0), float(w_r)


def weights64(ut):
    a, b, k = (F32(x) for x in ut)
    lam = a * a * (3 + k) - 3
    return math.sqrt(3 + lam), lam / (3 + lam), lam / (3 + lam) + 1 - a * a + b, 1 / (2 * (3 + lam))


# ------------------------------------------------------------------------------------------------------------------
# the decision quantities
def _rotmat(q):
    return U.quat_to_rotmat(q)


def quantities(means, quats, scales, opac, vm, cam, P, K=None):
    """float64 decision quantities of N rows (float64 tensors / arrays) under one camera and parameter set: per sigma
    point z, u, v, icD, th_full, validity [N, 7]; the UT mean, covariance, det_orig, det, compensation, op, the
    unrounded radii, zc, |q|^2 and min |s|; and their float32 rounding estimates (e_*)."""
    means, quats, scales, vm = (torch.as_tensor(np.asarray(x, np.float64)) for x in (means, quats, scales, vm))
    opac = torch.as_tensor(np.asarray(opac, np.float64))
    spread, wm0, wc0, wr = weights64(P["ut"])
    _, wm0_32, wc0_32, wr_32 = weights32(P["ut"])
    Rq = _rotmat(quats)
    off = spread * Rq * scales[:, None, :]
    pts = torch.stack([means] + [means + off[..., i] for i in range(3)] + [means - off[..., i] for i in range(3)], 1)
    R, t = vm[:3, :3], vm[:3, 3]
    pc = pts @ R.T + t
    pc_abs = pts.abs() @ R.T.abs() + t.abs()
    uv, valid = cam.project(pc, P["margin"])
    u, v = uv[..., 0], uv[..., 1]
    x, y, z = pc[..., 0], pc[..., 1], pc[..., 2]
    zs = torch.where(z > 0, z, torch.ones_like(z))
    nan = torch.full_like(z, float("nan"))
    icd, th = nan, nan
    if cam.kind == "pinhole" and cam.distorted:
        r2 = (x / zs) ** 2 + (y / zs) ** 2
        k = cam.k
        num = 1 + r2 * (k[0] + r2 * (k[1] + r2 * k[2]))
        den = 1 + r2 * (k[3] + r2 * (k[4] + r2 * k[5]))
        icd = num / den
    if cam.kind == "fisheye":
        th = torch.atan2(torch.sqrt(x * x + y * y), z)
    wm = torch.tensor([wm0] + [wr] * 6, dtype=f64)
    wc = torch.tensor([wc0] + [wr] * 6, dtype=f64)
    dwm = torch.tensor([abs(wm0 - wm0_32)] + [abs(wr - wr_32)] * 6, dtype=f64)
    dwc = torch.tensor([abs(wc0 - wc0_32)] + [abs(wr - wr_32)] * 6, dtype=f64)
    m2 = (wm[None, :, None] * uv).sum(1)
    du = uv - m2[:, None]
    cov = (wc[None, :, None, None] * du[..., :, None] * du[..., None, :]).sum(1)
    c00, c01, c11 = cov[:, 0, 0], cov[:, 0, 1], cov[:, 1, 1]
    # float32 rounding of the sigma points' image points: a few ulp of the image point and of the principal point,
    # and of the camera-frame terms carried to the image (relative to z)
    fxy = torch.tensor([cam.fx, cam.fy], dtype=f64)
    rel = pc_abs[..., :2] / zs.abs()[..., None] + pc_abs[..., 2:] * (pc[..., :2].abs() / zs[..., None] ** 2)
    e_uv = 4 * ULP * (uv.abs() + torch.tensor([CX, CY], dtype=f64) + fxy * rel)
    if cam.kind == "fisheye" or cam.distorted:
        e_uv = e_uv * 4
    e_m2 = (wm.abs()[None, :, None] * e_uv).sum(1) + 4 * ULP * (wm.abs()[None, :, None] * uv.abs()).sum(1) \
        + (dwm[None, :, None] * uv.abs()).sum(1)
    # du_k = u_k - m2: the error of m2 is common to every point, and sum_k wc_k du_k is small (sum_k wm_k du_k = 0)
    # the kernel's du_k - (its m2 error) enters c as sum_k wc_k (du_k + d_k - d_m)^2: the common d_m is weighted by
    # sum_k wc_k du_k (small, sum_k wm_k du_k = 0) and sum_k wc_k (about 4), the per-point d_k by |wc_k|
    sw = (wc[None, :, None] * du).sum(1).abs()
    swc = abs(float(wc.sum()))
    ew = (wc.abs()[None, :, None] * e_uv).sum(1)
    e_c = (wc.abs()[None, :, None] * (2 * du.abs() * e_uv + e_uv * e_uv)).sum(1) + 2 * sw * e_m2 + swc * e_m2 * e_m2 \
        + 2 * ew * e_m2 + 4 * ULP * (wc.abs()[None, :, None] * du * du).sum(1) + (dwc[None, :, None] * du * du).sum(1)
    e_c00, e_c11 = e_c[:, 0], e_c[:, 1]
    e_c01 = (wc.abs()[None] * (du[..., 0].abs() * e_uv[..., 1] + du[..., 1].abs() * e_uv[..., 0]
                               + e_uv[..., 0] * e_uv[..., 1])).sum(1) \
        + sw[:, 0] * e_m2[:, 1] + sw[:, 1] * e_m2[:, 0] + swc * e_m2[:, 0] * e_m2[:, 1] \
        + ew[:, 0] * e_m2[:, 1] + ew[:, 1] * e_m2[:, 0] \
        + 4 * ULP * (wc.abs()[None] * (du[..., 0] * du[..., 1]).abs()).sum(1) + (dwc[None] * (du[..., 0] * du[..., 1]).abs()).sum(1)
    eps2d = F32(P["eps2d"])
    det_o = c00 * c11 - c01 * c01
    e_det_o = c11.abs() * e_c00 + c00.abs() * e_c11 + 2 * c01.abs() * e_c01 + 4 * ULP * (c00 * c11).abs() + 4 * ULP * c01 * c01
    a00, a11 = c00 + eps2d, c11 + eps2d
    det = a00 * a11 - c01 * c01
    e_det = a11.abs() * e_c00 + a00.abs() * e_c11 + 2 * c01.abs() * e_c01 + 4 * ULP * ((a00 * a11).abs() + c01 * c01)
    with np.errstate(all="ignore"):
        ratio = det_o / det
        e_ratio = e_det_o / det.abs() + det_o.abs() * e_det / det**2 + 4 * ULP * ratio.abs()
        comp = torch.sqrt(ratio.clamp_min(MIN_COMP * MIN_COMP))
        e_comp = torch.where(ratio > MIN_COMP * MIN_COMP, e_ratio / (2 * comp), torch.zeros_like(comp)) + 4 * ULP * comp
        op = opac * comp
        e_op = opac * e_comp + 4 * ULP * op
        lg = torch.log((op / ALPHA_TH).clamp_min(1.0))
        e2 = torch.sqrt(2 * lg)
        ext = torch.minimum(e2, torch.full_like(e2, EXTEND))
        e_ext = torch.where(e2 < EXTEND, (e_op / op) / e2.clamp_min(1e-30) + 8 * ULP * e2, torch.zeros_like(e2))
        hb = 0.5 * (a00 + a11)
        e_hb = 0.5 * (e_c00 + e_c11) + 2 * ULP * hb.abs()
        arg = hb * hb - det
        targ = torch.sqrt(arg.clamp_min(0.01))
        e_targ = torch.where(arg > 0.01, (2 * hb.abs() * e_hb + e_det + 4 * ULP * (hb * hb + det.abs())) / (2 * targ),
                             torch.zeros_like(targ)) + 2 * ULP * targ
        s1 = (hb + targ).clamp_min(0)
        r1 = ext * torch.sqrt(s1)
        e_r1 = e_ext * torch.sqrt(s1) + ext * (e_hb + e_targ) / (2 * torch.sqrt(s1)) + 8 * ULP * r1
        rxa, rya = ext * torch.sqrt(a00.clamp_min(0)), ext * torch.sqrt(a11.clamp_min(0))
        e_rxa = e_ext * torch.sqrt(a00.clamp_min(0)) + ext * e_c00 / (2 * torch.sqrt(a00.clamp_min(0))) + 8 * ULP * rxa
        e_rya = e_ext * torch.sqrt(a11.clamp_min(0)) + ext * e_c11 / (2 * torch.sqrt(a11.clamp_min(0))) + 8 * ULP * rya
        rxf = torch.minimum(rxa, r1)
        ryf = torch.minimum(rya, r1)
        e_rx = torch.where(rxa < r1, e_rxa, e_r1)
        e_ry = torch.where(rya < r1, e_rya, e_r1)
        conic = torch.stack([a11 / det, -c01 / det, a00 / det], -1)
        e_conic = torch.stack([e_c11, e_c01, e_c00], -1) / det.abs()[:, None] + conic.abs() * (e_det / det.abs())[:, None] \
            + 4 * ULP * conic.abs()
    zc = means @ R[2] + t[2]
    e_zc = 8 * ULP * ((means.abs() @ R[2].abs()) + t[2].abs())
    qn2 = (quats * quats).sum(-1)
    return dict(z=z, e_z=8 * ULP * pc_abs[..., 2], u=u, v=v, e_u=e_uv[..., 0], e_v=e_uv[..., 1], icd=icd, th=th,
                valid=valid, pc=pc, m2=m2, e_m2=e_m2, c00=a00, c11=a11, c01=c01, e_c00=e_c00, e_c11=e_c11,
                det=det, e_det=e_det, det_o=det_o, comp=comp, e_comp=e_comp, op=op, e_op=e_op, rxf=rxf, ryf=ryf,
                e_rx=e_rx, e_ry=e_ry, conic=conic, e_conic=e_conic, zc=zc, e_zc=e_zc, qn2=qn2,
                smin=scales.abs().min(-1).values, ext=ext)


# ------------------------------------------------------------------------------------------------------------------
# rows
def _world(pc):
    """camera-frame point -> world point through VM (exact for dyadic points)"""
    R, t = VM[:3, :3].astype(np.float64), VM[:3, 3].astype(np.float64)
    return R.T @ (np.asarray(pc, np.float64) - t)


# with the identity world quaternion, the sigma points' camera-frame offsets: world axis 0 is camera +y, axis 1
# camera -x, axis 2 camera +z; sigma point k (1..3: +axis k-1, 4..6: -axis k-4)
CAM_AXIS_POINT = {"+x": (5, 1), "-x": (2, 1), "+y": (1, 0), "-y": (4, 0), "+z": (3, 2), "-z": (6, 2)}


class Rows:
    def __init__(self, rng):
        self.rng, self.rows = rng, []

    def add(self, cls, pc, scales, quat=(1.0, 0.0, 0.0, 0.0), opacity=0.9, exact=False):
        self.rows.append((cls, _world(pc), np.asarray(quat, np.float64), np.asarray(scales, np.float64), opacity, exact))

    def arrays(self):
        f = lambda k: np.ascontiguousarray(np.array([r[k] for r in self.rows], np.float64).astype(np.float32))  # noqa: E731
        return dict(cls=np.array([r[0] for r in self.rows]), means=f(1), quats=f(2), scales=f(3), opacities=f(4),
                    exact=np.array([r[5] for r in self.rows], bool))


def _rand_quat(rng):
    q = rng.standard_normal(4)
    return q / np.linalg.norm(q)


def _solve(f, lo, hi, target, iters=100):
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


def _row_q(lens, pc, scales, quat, opacity, P):
    q = quantities(_world(pc)[None], np.asarray(quat, np.float64)[None], np.asarray(scales, np.float64)[None],
                   np.array([opacity]), VM, camera(lens), P)
    return {k: (v[0] if torch.is_tensor(v) and v.dim() > 0 else v) for k, v in q.items()}


K1 = LENSES["distorted"]["coeffs"]["radial"][0]


def make_rows(lens, seed=20261019):
    rng = np.random.RandomState(seed + len(lens))
    r = Rows(rng)
    cam = camera(lens)
    fx, fy = LENSES[lens]["f"]
    P0 = params("default")

    def on_screen(z, spread=0.8):
        # a camera-frame point imaged inside the central part of the image (pinhole guess; fine for every lens here)
        u, v = CX + rng.uniform(-spread, spread) * 0.4 * W, CY + rng.uniform(-spread, spread) * 0.4 * H
        if LENSES[lens]["kind"] == "fisheye":
            return np.array([(u - CX) / fx * z * 0.6, (v - CY) / fy * z * 0.6, z])
        return np.array([(u - CX) / fx * z, (v - CY) / fy * z, z])

    for _ in range(48):
        z = 10.0 ** rng.uniform(0.0, 1.3)
        s = z * 10.0 ** rng.uniform(-3, -1.3, 3)
        r.add("bulk", on_screen(z), s, _rand_quat(rng), rng.uniform(0.05, 1.0))
    # margin edges: exact ties under the exact UT (perfect pinhole), for margin factors 0 and 0.5
    if lens == "pinhole":
        for m in (0.0, 0.5):
            for side in ("+x", "-x", "+y", "-y"):
                z, s = 2.0, 1.0 / 16
                ax = 0 if side[1] == "x" else 1
                f, c, n = (fx, CX, W) if ax == 0 else (fy, CY, H)
                edge = n + n * m if side[0] == "+" else -n * m
                e = (edge - c) * z / f
                pc = np.array([0.0, 0.0, z])
                pc[ax] = e - 2 * s if side[0] == "+" else e + 2 * s
                r.add("margin", pc, (s, s, s), exact=True)
                for d in (0.25, -0.25, 0.01, -0.01):  # near the edge in pixels (spread 2 of the exact UT)
                    pc2 = pc.copy()
                    pc2[ax] += d * z / f
                    r.add("margin", pc2, (s, s, s))
        # a sigma point at z == 0 (exact), and behind the camera
        for i in range(4):
            s2 = 0.25
            pc = on_screen(2.0, 0.5)
            pc = np.round(pc * 64) / 64
            pc[2] = 2 * s2
            r.add("behind", pc, (1.0 / 32, 1.0 / 64, s2), exact=True)
            pc[2] = 1.5 * s2
            r.add("behind", pc, (1.0 / 32, 1.0 / 64, s2))
    else:
        for i in range(8):
            z = rng.uniform(1.0, 4.0)
            s2 = z / (0.2 + 0.1 * i) / weights64(DEFAULT_UT)[0]
            r.add("behind", on_screen(z, 0.5), (z * 0.01, z * 0.01, s2), (1.0, 0.0, 0.0, 0.0))
    if lens == "distorted":
        # the +x sigma point (spread 2 * 1/32) at (1, 0, 1): icD == float32(0.8) exactly; the other six have smaller
        # x / z and icD > 0.8
        for i in range(2):
            r.add("icd", (1.0 - 1.0 / 16, 0.0, 1.0), (1.0 / 64, 1.0 / 32, 1.0 / 64), exact=True)
        # near icD == 0.8 on the +x sigma point under the default UT
        spread = weights64(DEFAULT_UT)[0]
        for d in (1e-2, -1e-2, 1e-3, -1e-3, 1e-4, -1e-4, 3e-3, -3e-3):
            r2 = (1 - (0.8 + d)) / -K1
            phi = rng.uniform(0, 2 * math.pi)
            s = 0.02
            z = rng.uniform(1.0, 3.0)
            pt = np.array([math.sqrt(r2) * math.cos(phi) * z, math.sqrt(r2) * math.sin(phi) * z, z])
            pc = pt.copy()
            pc[0] -= spread * s  # the +x sigma point at pt
            r.add("icd", pc, (s * 0.5, s, s * 0.5))
    if lens == "fisheye":
        ma = cam.max_angle
        spread = weights64(DEFAULT_UT)[0]
        for d in (1e-2, -1e-2, 1e-3, -1e-3, 1e-4, -1e-4, 3e-3, -3e-3, 3e-2, -3e-2):
            th = ma * (1 + d)
            phi = rng.uniform(0, 2 * math.pi)
            z = rng.uniform(1.0, 3.0)
            pt = np.array([math.tan(th) * math.cos(phi) * z, math.tan(th) * math.sin(phi) * z, z])
            s = 0.01
            pc = pt.copy()
            pc[2] -= spread * s  # the +z sigma point at pt
            r.add("max_angle", pc, (s * 0.5, s * 0.5, s))
    # near / far planes (both near planes of the parameter sets)
    for plane in (0.01, 0.5, FAR):
        for d in (1e-3, -1e-3, 1e-5, -1e-5, 1e-6, -1e-6):
            zz = F32(plane) * (1 + d)
            r.add("near" if plane < 1 else "far", on_screen(zz, 0.3), (zz * 0.02, zz * 0.03, zz * 0.02), _rand_quat(rng))
    # degenerate: |q|^2 around FLT_EPSILON, one |s| around FLT_EPSILON
    for f in (0.25, 4.0):
        q = _rand_quat(rng) * math.sqrt(f * FLT_EPS)
        r.add("degenerate", on_screen(3.0), (0.05, 0.05, 0.05), q)
        r.add("degenerate", on_screen(3.0), (0.05, f * FLT_EPS, 0.05), _rand_quat(rng))
    # a UT covariance that is not positive definite: large gaussians close to the camera under a negative beta with
    # eps2d = 0, kept when the float64 det_orig or c00 is negative
    P_np = params("negbeta/m0.5/eps0")
    n_np = 0
    for _ in range(400):
        if n_np >= 10:
            break
        z = rng.uniform(0.5, 2.0)
        pc = on_screen(z, 0.6)
        s = z * rng.uniform(0.1, 1.0, 3)
        q = _rand_quat(rng)
        qq = _row_q(lens, pc, s, q, 0.9, P_np)
        if float(qq["det_o"]) < 0 or float(qq["c00"]) < 0:
            r.add("nonpd", pc, s, q)
            n_np += 1
    # opacity * compensation near 1/255 (default parameters)
    for d in (1e-2, -1e-2, 1e-3, -1e-3, 1e-4, -1e-4, 3e-5, -3e-5):
        z = rng.uniform(2.0, 8.0)
        pc, s, q = on_screen(z), z * 10.0 ** rng.uniform(-3, -2.5, 3), _rand_quat(rng)
        comp = float(_row_q(lens, pc, s, q, 0.5, P0)["comp"])
        r.add("opacity", pc, s, q, ALPHA_TH / comp * (1 + d))
    # ceil: the radius near an integer (default parameters); radius_clip: near 3
    for cls, targets in (("ceil", (5 + 1e-2, 5 - 1e-2, 9 + 1e-3, 9 - 1e-3, 14 + 1e-4, 14 - 1e-4, 21 + 3e-3, 21 - 3e-3)),
                         ("radius_clip", (3 + 1e-2, 3 - 1e-2, 3 + 1e-3, 3 - 1e-3, 2.5, 3.5, 3 + 1e-4, 3 - 1e-4))):
        for tg in targets:
            z = rng.uniform(2.0, 8.0)
            pc, q, an = on_screen(z, 0.5), _rand_quat(rng), rng.uniform(0.3, 1.0, 3)
            f = lambda s, pc=pc, q=q, an=an: float(_row_q(lens, pc, s * an, q, 0.9, P0)["rxf"])  # noqa: E731
            s = _solve(f, 1e-5 * z, 0.3 * z, tg)
            r.add(cls, pc, s * an, q, 0.9)
    # off-screen: m2 +- radius against 0, W, 0, H (default parameters)
    for i in range(16):
        side = i % 4
        z = rng.uniform(2.0, 8.0)
        q, s = _rand_quat(rng), z * rng.uniform(0.002, 0.01) * np.array([1.0, 0.8, 0.6])
        d = (1e-1, -1e-1, 1e-3, -1e-3)[i // 4]
        other = on_screen(z, 0.3)
        ax = side // 2

        def edge(x, other=other, q=q, s=s, side=side, ax=ax):
            pc = other.copy()
            pc[ax] = x
            qq = _row_q(lens, pc, s, q, 0.9, P0)
            fr = math.ceil(float(qq["rxf"] if ax == 0 else qq["ryf"]))
            m = float(qq["m2"][ax])
            return m + fr if side % 2 == 0 else m - fr - (W if ax == 0 else H)

        lim = 0.6 * z if LENSES[lens]["kind"] == "fisheye" else 1.2 * z
        lo, hi = (-lim, 0.0) if side % 2 == 0 else (0.0, lim)
        if (edge(lo) - d) * (edge(hi) - d) > 0:
            continue
        x = _solve(edge, lo, hi, d, 60)
        pc = other.copy()
        pc[ax] = x
        r.add("offscreen", pc, s, q)
    # finite inputs whose float32 transform overflows (pinhole: the fisheye clamps the angle, so its image points of
    # far sigma points stay finite)
    for sc in ((1e37, 1e38, 3e38) if LENSES[lens]["kind"] == "pinhole" else ()):
        # one axis across the view: its sigma points' image coordinates are beyond float32's range
        r.add("overflow", on_screen(3.0), (sc, 0.1, 0.1), (1.0, 0.0, 0.0, 0.0))
        r.add("overflow", on_screen(3.0), (0.1, sc, 0.1), (1.0, 0.0, 0.0, 0.0))
    return r.arrays()


CLASSES = {
    "pinhole": ("bulk", "margin", "behind", "near", "far", "degenerate", "nonpd", "opacity", "ceil", "radius_clip",
                "offscreen", "overflow"),
    "distorted": ("bulk", "behind", "icd", "near", "far", "degenerate", "nonpd", "opacity", "ceil", "radius_clip",
                  "offscreen", "overflow"),
    "fisheye": ("bulk", "behind", "max_angle", "near", "far", "degenerate", "nonpd", "opacity", "ceil", "radius_clip"),
}


# ------------------------------------------------------------------------------------------------------------------
# truth
def _perturb(arrs, k):
    out = {key: np.asarray(v, np.float64) for key, v in arrs.items()}
    if k:
        rng = np.random.RandomState(1000 + k)
        out = {key: v * (1.0 + 4.0 * ULP * rng.uniform(-1, 1, v.shape)) for key, v in out.items()}
    return out


def _spread(base, vals):
    base = np.asarray(base, np.float64)
    with np.errstate(invalid="ignore"):
        return np.nan_to_num(np.max([np.abs(np.asarray(v, np.float64) - base) for v in vals], 0), nan=np.inf, posinf=np.inf)


def _n(t):
    return t.detach().numpy() if torch.is_tensor(t) else np.asarray(t)


class Truth:
    pass


def truth(rows, lens, P):
    """float64 truth of the rows under one lens and parameter set: the oracle's outputs, their budgets, decided [N],
    visible [N], and the margins behind the decision."""
    spec = LENSES[lens]
    K = K_of(lens)
    co = {k: np.asarray(v, np.float32) for k, v in spec["coeffs"].items()}
    arrs = dict(means=rows["means"], quats=rows["quats"], scales=rows["scales"], opacities=rows["opacities"], vm=VM, K=K,
                **{"co_" + k: v for k, v in co.items()})
    qs = []
    for k in range(N_PERTURB + 1):
        p = _perturb(arrs, k)
        cam = camera(lens, p["K"], {c: p["co_" + c] for c in co})
        with np.errstate(all="ignore"):
            qs.append({key: _n(v) for key, v in quantities(p["means"], p["quats"], p["scales"], p["opacities"], p["vm"],
                                                            cam, P).items()})
    q = qs[0]
    sp = lambda key: _spread(q[key], [x[key] for x in qs[1:]])  # noqa: E731
    b = lambda key, e: 4.0 * sp(key) + q[e]  # noqa: E731
    near = F32(P["near"])
    with np.errstate(all="ignore"):
        b_zc = b("zc", "e_zc")
        degenerate = (np.abs(q["qn2"]) < FLT_EPS) | (q["smin"] < FLT_EPS)
        deg_ok = (np.abs(q["qn2"] - FLT_EPS) > 8 * ULP * q["qn2"])  # |s| < FLT_EPSILON is exact
        in_depth = (q["zc"] >= near) & (q["zc"] <= FAR)
        depth_ok = (np.abs(q["zc"] - near) > b_zc) & (np.abs(q["zc"] - FAR) > b_zc)
        # the tie rows are exact under the exact UT only: the undistorted pinhole for the margin and z == 0 ties, the
        # distorted pinhole's icD == 0.8 tie
        exact_ut = P["ut"] == EXACT_UT
        exact = rows["exact"][:, None] & exact_ut & (lens == "pinhole")
        exact_icd = rows["exact"][:, None] & exact_ut & (lens == "distorted")
        # each sigma point: the margin of every test of its validity
        b_z = b("z", "e_z")
        z_ok = (np.abs(q["z"]) > b_z) | (exact & (q["z"] == 0))
        mx, my = F32(f32(W) * f32(P["margin"])), F32(f32(H) * f32(P["margin"]))
        b_u, b_v = b("u", "e_u"), b("v", "e_v")
        edge_ok = ((np.minimum(np.abs(q["u"] + mx), np.abs(q["u"] - W - mx)) > b_u)
                   & (np.minimum(np.abs(q["v"] + my), np.abs(q["v"] - H - my)) > b_v)) | exact
        pt_ok = z_ok & (edge_ok | (q["z"] <= 0))
        if spec["kind"] == "pinhole" and "radial" in co:
            b_icd = 4.0 * sp("icd") + 16 * ULP * (1 + np.abs(q["icd"]))
            pt_ok &= (np.abs(q["icd"] - F32(0.8)) > b_icd) | (exact_icd & (q["icd"] == F32(0.8))) | (q["z"] <= 0)
        if spec["kind"] == "fisheye":
            ma = camera(lens).max_angle
            b_th = 4.0 * sp("th") + 32 * ULP * ma
            pt_ok &= (np.abs(q["th"] - ma) > b_th) | (q["z"] <= 0)
        valid = q["valid"]
        if P["require_all"]:
            pts_ok = ((~valid) & pt_ok).any(1) | pt_ok.all(1)
            ut_valid = valid.all(1)
        else:
            pts_ok = (valid & pt_ok).any(1) | pt_ok.all(1)
            ut_valid = valid.any(1)
        det_ok = np.abs(q["det"]) > b("det", "e_det")
        c_ok = (np.abs(q["c00"]) > b("c00", "e_c00")) & (np.abs(q["c11"]) > b("c11", "e_c11"))
        pd = (q["det"] > 0) & (q["c00"] >= 0) & (q["c11"] >= 0)
        b_op = b("op", "e_op")
        op_ok = np.abs(q["op"] - ALPHA_TH) > b_op
        op_keep = q["op"] >= ALPHA_TH
        b_rx, b_ry = b("rxf", "e_rx"), b("ryf", "e_ry")
        ceil_ok = (np.abs(q["rxf"] - np.round(q["rxf"])) > b_rx) & (np.abs(q["ryf"] - np.round(q["ryf"])) > b_ry)
        rx, ry = np.ceil(q["rxf"]), np.ceil(q["ryf"])
        clipped = (rx <= F32(P["clip"])) & (ry <= F32(P["clip"]))
        b_m2 = 4.0 * sp("m2") + q["e_m2"]
        edges = np.stack([q["m2"][:, 0] + rx, q["m2"][:, 0] - rx - W, q["m2"][:, 1] + ry, q["m2"][:, 1] - ry - H], -1)
        off = (edges[:, 0] <= 0) | (edges[:, 1] >= 0) | (edges[:, 2] <= 0) | (edges[:, 3] >= 0)
        off_ok = (np.abs(edges) > np.repeat(b_m2, 2, -1)).all(-1)
        # the float32 transform overflows where any float64 image point or covariance term is beyond float32's range
        overflow = ~np.isfinite(q["u"]).all(1) | (np.abs(np.stack([q["u"], q["v"]])) > FLT_MAX / 512).any((0, 2)) \
            | (np.abs(q["c00"]) > FLT_MAX / 512) | (np.abs(q["c11"]) > FLT_MAX / 512) | (np.abs(q["det"]) > FLT_MAX / 512)
        live = ~degenerate & in_depth
        vis = live & ut_valid & pd & op_keep & ~clipped & ~off & ~overflow
        tail = ceil_ok & (clipped | off_ok)
        after_pd = op_ok & (~op_keep | tail)
        after_ut = det_ok & c_ok & (~pd | after_pd)
        decided = deg_ok & (degenerate | (depth_ok & (~in_depth | overflow | (pts_ok & (~ut_valid | after_ut)))))
    # the oracle's outputs
    cam = camera(lens)
    a, be, ka = P["ut"]
    o = U.ut_projection(rows["means"], rows["quats"], rows["scales"], rows["opacities"], VM.astype(np.float64), cam,
                        eps2d=F32(P["eps2d"]), near_plane=near, far_plane=FAR, radius_clip=F32(P["clip"]),
                        ut=dict(alpha=F32(a), beta=F32(be), kappa=F32(ka), in_image_margin_factor=F32(P["margin"]),
                                require_all_sigma_points_valid=P["require_all"]))
    tr = Truth()
    tr.cls, tr.decided, tr.vis, tr.q, tr.P, tr.lens = rows["cls"], decided, vis, q, P, lens
    tr.oracle_valid = _n(o["valid"]) & ~overflow
    tr.radii = np.where(vis[:, None], np.stack([rx, ry], -1), 0).astype(np.int64)
    tr.means2d = np.where(vis[:, None], _n(o["means2d"]), 0)
    tr.depths = np.where(vis, _n(o["depths"]), 0)
    tr.conics = np.where(vis[:, None], _n(o["conics"]), 0)
    tr.compensations = np.where(vis, _n(o["compensations"]), 0)
    tr.beta = dict(means2d=b_m2, depths=b_zc, conics=4.0 * sp("conic") + q["e_conic"], compensations=b("comp", "e_comp"))
    tr.margins = dict(pts_ok=pts_ok, det_ok=det_ok, c_ok=c_ok, op_ok=op_ok, ceil_ok=ceil_ok, off_ok=off_ok,
                      depth_ok=depth_ok, overflow=overflow, ut_valid=ut_valid, pd=pd)
    return tr


def describe(rows, tr, n):
    return (f"row {n} (class {tr.cls[n]}, lens {tr.lens}, params {tr.P['name']}, mean={rows['means'][n].tolist()}, "
            f"quat={rows['quats'][n].tolist()}, scale={rows['scales'][n].tolist()}, opacity={float(rows['opacities'][n])})")


def check_projection(rows, tr, radii, means2d, depths, conics, comps, what):
    """float32 outputs [N, *] against the truth on decided rows; returns failure messages"""
    msgs = []
    dec = tr.decided
    radii = np.asarray(radii).astype(np.int64)
    bad = dec & (radii != tr.radii).any(-1)
    if bad.any():
        n = np.argwhere(bad)[0][0]
        msgs.append(f"{what}: {int(bad.sum())} decided rows with wrong radii, e.g. {describe(rows, tr, n)}: "
                    f"got {radii[n].tolist()}, truth {tr.radii[n].tolist()}")
    culled = (radii == 0).all(-1)
    for name, got in (("means2d", means2d), ("depths", depths), ("conics", conics), ("compensations", comps)):
        got = np.asarray(got, np.float64)
        ref, b = getattr(tr, name), tr.beta[name]
        g, r_ = got.reshape(len(got), -1), ref.reshape(len(ref), -1)
        bb = np.broadcast_to(np.asarray(b).reshape(len(got), -1), g.shape)
        with np.errstate(invalid="ignore"):
            bad = dec & tr.vis & ~(np.abs(g - r_) <= bb).all(-1)
        bad_c = culled & (g != 0).any(-1)
        if bad.any():
            n = np.argwhere(bad)[0][0]
            msgs.append(f"{what}: {int(bad.sum())} decided rows with {name} out of budget, e.g. {describe(rows, tr, n)}: "
                        f"got {g[n].tolist()}, truth {r_[n].tolist()}, beta {bb[n].tolist()}")
        if bad_c.any():
            n = np.argwhere(bad_c)[0][0]
            msgs.append(f"{what}: {int(bad_c.sum())} culled rows with non-zero {name}, e.g. {describe(rows, tr, n)}")
    return msgs


# ceilings on the undecided share of the bulk rows and of all rows, per lens, under the exact and the other UT and under
# the default and the negative-beta UT (whose centre weight of -99 amplifies float32 rounding about 100x; the distorted
# lenses carry larger image-point budgets)
UNDECIDED_MAX = {
    "pinhole": dict(bulk=(0.1, 0.3), rows=(0.2, 0.45)),
    "distorted": dict(bulk=(0.1, 0.8), rows=(0.2, 0.7)),
    "fisheye": dict(bulk=(0.1, 0.95), rows=(0.2, 0.8)),
}


def undecided_ceiling_msgs(tr):
    """the undecided shares of tr against UNDECIDED_MAX; returns failure messages"""
    k = 0 if tr.P["ut"] in (EXACT_UT, OTHER_UT) else 1
    lim = UNDECIDED_MAX[tr.lens]
    bulk = tr.cls == "bulk"
    out = []
    for what, sel in (("bulk", bulk), ("rows", np.ones_like(bulk))):
        share = float((~tr.decided[sel]).mean())
        if share > lim[what][k]:
            out.append(f"{tr.lens} {tr.P['name']}: {share:.2f} of the {what} undecided, ceiling {lim[what][k]}")
    return out


def undecided_report(tr):
    """per class: (rows, undecided rows, decided visible rows)"""
    out = {}
    for k in np.unique(tr.cls):
        sel = tr.cls == k
        out[str(k)] = (int(sel.sum()), int((~tr.decided[sel]).sum()), int((tr.decided & tr.vis)[sel].sum()))
    return out
