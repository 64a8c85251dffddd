"""Float64 restatement of the FTheta camera of 3DGUT (test infrastructure), a camera model for oracle/ut.py's
projection and compositing and for the rolling-shutter oracle in tests/ut_rs_oracle.py.

FTheta: a ray at angle theta from the optical axis lands at the pixel distance delta = fw(theta) from the principal
point, fw the forward polynomial (angle -> pixel distance); bw, the backward polynomial (pixel distance -> angle), is
calibrated together with it.  The reference polynomial (reference_poly 0: bw, 1: fw) is evaluated directly, the other
direction inverts it by three Newton steps starting from the other polynomial, stopping early once a step is below
1e-6.  The image offset is [[c, d], [e, 1]] times the radial offset delta * (x, y) / |(x, y)|, about the principal
point Ks (cx, cy) + 0.5.  Projection: no z > 0 requirement; theta is clamped to max_angle and a point is valid below
max_angle, inside the image grown by the margin; the Newton convergence flag is ignored.  Unprojection: invalid where
the linear map is singular (|c - e d| < 1e-8) or, with the forward polynomial as the reference, where the last Newton
step stays at or above 1e-6.

Depth order: with global_z_order=False the near / far cull and the depth take the distance |mean_c| from the camera
centre (the mid-frame pose under a rolling shutter) instead of z.

The calibrations of tests/golden/ftheta_calibrations.json are scaled to an image s times as wide by ``scaled``:
principal point * s, forward coefficient k * s, backward coefficient k * s^-k."""
from __future__ import annotations

import json
import math
import os

import torch

from oracle import ut as U
from oracle.ut import F64
from tests import ut_rs_oracle as R8

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALIBRATIONS = os.path.join(ROOT, "tests", "golden", "ftheta_calibrations.json")
PIXELDIST_TO_ANGLE, ANGLE_TO_PIXELDIST = 0, 1
NEWTON_STEPS, NEWTON_TOL = 3, 1e-6
FLT_EPS = float(torch.finfo(torch.float32).eps)


def calibrations():
    """{name: calibration dict} of tests/golden/ftheta_calibrations.json at native resolution."""
    with open(CALIBRATIONS) as f:
        return {k: v for k, v in json.load(f).items() if not k.startswith("_")}


def scaled(cal, width):
    """The calibration for an image `width` pixels wide: principal point * s, forward coefficient k * s, backward
    coefficient k * s^-k, s = width / native width.  Returns (params dict, principal point (cx, cy), (W, H))."""
    W0, H0 = cal["resolution"]
    s = width / W0
    fw = [c * s for c in cal["angle_to_pixeldist_poly"]]
    bw = [c * s ** (-k) for k, c in enumerate(cal["pixeldist_to_angle_poly"])]
    pp = (cal["principal_point"][0] * s, cal["principal_point"][1] * s)
    params = dict(pixeldist_to_angle_poly=bw, angle_to_pixeldist_poly=fw, max_angle=float(cal["max_angle"]),
                  linear_cde=list(cal["linear_cde"]))
    return params, pp, (int(width), int(round(H0 * s)))


def poly(c, x):
    y = torch.zeros_like(x)
    for k in reversed(c):
        y = y * x + k
    return y


def dpoly(c):
    return [k * c[k] for k in range(1, len(c))]


def newton(ref, approx, y):
    """x with ref(x) = y: three Newton steps from approx(y), each element stopping once its step is below 1e-6.
    Returns (x, converged, |last step|)."""
    d = dpoly(ref)
    x = poly(approx, y)
    live = torch.ones_like(x, dtype=torch.bool)
    step = torch.full_like(x, math.inf)
    for _ in range(NEWTON_STEPS):
        dx = (poly(ref, x) - y) / poly(d, x)
        x = torch.where(live, x - dx, x)
        step = torch.where(live, dx.abs(), step)
        live = live & ~(dx.abs() < NEWTON_TOL)
    return x, ~live, step


class FThetaCamera:
    """One FTheta camera: the shared parameters (dict with the five fields of FThetaCameraDistortionParameters), its
    principal point from K (cx, cy), the image size.  ``last_step`` after unproject: each pixel's last Newton step
    (forward reference), for tests that exclude pixels at the 1e-6 convergence threshold."""

    def __init__(self, params, K, W, H):
        K = torch.as_tensor(K, dtype=F64)
        self.W, self.H = int(W), int(H)
        self.cx, self.cy = float(K[0, 2]) + 0.5, float(K[1, 2]) + 0.5
        self.ref = int(params["reference_poly"])
        self.bw = [float(x) for x in params["pixeldist_to_angle_poly"]]
        self.fw = [float(x) for x in params["angle_to_pixeldist_poly"]]
        self.max_angle = float(params["max_angle"])
        self.c, self.d, self.e = (float(x) for x in params["linear_cde"])
        self.last_step = None

    def delta_of_angle(self, th):
        if self.ref == ANGLE_TO_PIXELDIST:
            return poly(self.fw, th)
        return newton(self.bw, self.fw, th)[0]

    def project(self, pc, margin):
        """camera-frame points [..., 3] -> (uv [..., 2], valid [...]); an invalid point keeps its image point."""
        x, y, z = pc[..., 0], pc[..., 1], pc[..., 2]
        rxy = torch.sqrt(x * x + y * y)
        rxy = torch.where(rxy <= 0, torch.full_like(rxy, FLT_EPS), rxy)
        th_full = torch.atan2(rxy, z)
        th = torch.minimum(th_full, torch.full_like(th_full, self.max_angle))
        delta = self.delta_of_angle(th)
        ix, iy = delta * (x / rxy), delta * (y / rxy)
        u = self.c * ix + self.d * iy + self.cx
        v = self.e * ix + iy + self.cy
        mx, my = self.W * margin, self.H * margin
        inb = (u >= -mx) & (u < self.W + mx) & (v >= -my) & (v < self.H + my)
        return torch.stack([u, v], -1), inb & (th_full < self.max_angle)

    def unproject(self, u, v):
        """image points -> (unit camera rays [..., 3], valid)."""
        u, v = torch.as_tensor(u, dtype=F64), torch.as_tensor(v, dtype=F64)
        x, y = u - self.cx, v - self.cy
        det = self.c - self.e * self.d
        if abs(det) < 1e-8:
            z = torch.zeros_like(x)
            self.last_step = z
            return torch.stack([z, z, torch.ones_like(x)], -1), torch.zeros_like(x, dtype=torch.bool)
        ux, uy = (x - self.d * y) / det, (-self.e * x + self.c * y) / det
        delta = torch.sqrt(ux * ux + uy * uy)
        if self.ref == PIXELDIST_TO_ANGLE:
            th, ok = poly(self.bw, delta), torch.ones_like(delta, dtype=torch.bool)
            self.last_step = torch.zeros_like(delta)
        else:
            th, ok, self.last_step = newton(self.fw, self.bw, delta)
        big = delta >= 1e-6
        sc = torch.where(big, torch.sin(th) / torch.where(big, delta, torch.ones_like(delta)), torch.zeros_like(delta))
        d = torch.stack([sc * ux, sc * uy, torch.where(big, torch.cos(th), torch.ones_like(th))], -1)
        return d, ok


def ut_projection(means, quats, scales, opacities, viewmat, cam, eps2d=0.3, near_plane=0.01, far_plane=1e10,
                  radius_clip=0.0, ut=None, global_z_order=True, viewmat_rs=None, shutter=R8.GLOBAL):
    """The UT projection (oracle.ut, tests/ut_rs_oracle) in either depth order: with global_z_order=False the near /
    far cull and the depth take |mean_c| (at the mid-frame pose under a rolling shutter)."""
    if global_z_order:
        return R8.ut_projection(means, quats, scales, opacities, viewmat, cam, eps2d, near_plane, far_plane, radius_clip,
                                ut, viewmat_rs=viewmat_rs, shutter=shutter)
    out = R8.ut_projection(means, quats, scales, opacities, viewmat, cam, eps2d, -math.inf, math.inf, radius_clip, ut,
                           viewmat_rs=viewmat_rs, shutter=shutter)
    m = torch.as_tensor(means, dtype=F64)
    if shutter == R8.GLOBAL:
        vm = torch.as_tensor(viewmat, dtype=F64)
        R, t = vm[:3, :3], vm[:3, 3]
    else:
        Rs, ts = R8.ShutterPoses(viewmat, viewmat_rs).at(torch.tensor([0.5], dtype=F64))
        R, t = Rs[0], ts[0]
    dist = (m @ R.T + t).norm(dim=-1)
    keep = out["valid"] & (dist >= near_plane) & (dist <= far_plane)
    for k in ("radii", "means2d", "conics"):
        out[k] = torch.where(keep[:, None], out[k], torch.zeros_like(out[k]))
    out["compensations"] = torch.where(keep, out["compensations"], torch.zeros_like(dist))
    out["depths"] = torch.where(keep, dist, torch.zeros_like(dist))
    out["valid"] = keep
    return out


def eval3d_render(*args, **kw):
    """oracle.ut.eval3d_render under either shutter, through tests/ut_rs_oracle (any camera with unproject)."""
    return R8.eval3d_render(*args, **kw)


__all__ = ["FThetaCamera", "calibrations", "scaled", "ut_projection", "eval3d_render", "U"]
