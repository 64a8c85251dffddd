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

FTheta: a ray at angle theta from the optical axis lands at the pixel distance delta = fw(theta) from the principal
point, fw the forward polynomial (angle -> pixel distance); bw, the backward polynomial (pixel distance -> angle), is
calibrated together with it.  The reference polynomial (reference_poly 0: bw, 1: fw) is evaluated directly, the other
direction inverts it by three Newton steps starting from the other polynomial, stopping early once a step is below
1e-6.  The image offset is [[c, d], [e, 1]] times the radial offset delta * (x, y) / |(x, y)|, about the principal
point Ks (cx, cy) + 0.5.  Projection: no z > 0 requirement; theta is clamped to max_angle and a point is valid below
max_angle, inside the image grown by the margin; the Newton convergence flag is ignored.  Unprojection: invalid where
the linear map is singular (|c - e d| < 1e-8) or, with the forward polynomial as the reference, where the last Newton
step stays at or above 1e-6.  With global_z_order=False the near / far cull and the depth take the distance |mean_c|
from the camera centre instead of z.

Rolling shutter: every image row (or column) is exposed at its own pose, the start pose (viewmat) and the end pose
(viewmat_rs) interpolated at the row's relative frame time, translation linearly and rotation by slerp of the poses'
quaternions (taken from the rotation blocks from their largest component).  A sigma point is projected by a fixed-point
iteration on its frame time, starting from the start pose's projection if it is valid, else the end pose's; a pixel's
ray leaves at its row's pose; the depth and the near / far cull take the mid-frame pose; the SH view directions are
taken from the mean of the two camera positions.  The projection, the rays and the compositing take either a view
matrix (global shutter) or a ShutterPoses.
"""
from __future__ import annotations

import math

import torch

F64 = torch.float64
FLT_EPS = float(torch.finfo(torch.float32).eps)
ALPHA_T, MAX_ALPHA, T_STOP, EXTEND, MIN_COMP = 1.0 / 255.0, 0.99, 1e-4, 3.33, 0.005
UT_DEFAULTS = dict(alpha=0.1, beta=2.0, kappa=0.0, in_image_margin_factor=0.1, require_all_sigma_points_valid=False)
# rolling shutter: ids as the reference's RollingShutterType
TOP_TO_BOTTOM, LEFT_TO_RIGHT, BOTTOM_TO_TOP, RIGHT_TO_LEFT, GLOBAL = 0, 1, 2, 3, 4
RS_ITERATIONS = 10
# FTheta
PIXELDIST_TO_ANGLE, ANGLE_TO_PIXELDIST = 0, 1
NEWTON_STEPS, NEWTON_TOL = 3, 1e-6
# pinhole validity: the radial factor above 0.8, compared at float32(0.8) as the kernels do
ICD_MIN = float(torch.tensor(0.8, dtype=torch.float32))


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
                ok = icd > ICD_MIN
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

    def unproject(self, u, v, rule="converged"):
        """image points -> (unit camera rays [..., 3], valid), the distortion inverted by Newton iteration.  rule
        "converged": iterate float64 to convergence.  rule "reference": replay the kernels' rule in float64 (pinhole:
        at most 5 steps, giving up at icD <= 0 or |det| < 1e-6, converged once both steps are below 1e-6; fisheye: at
        most 20 steps, converged once the step is below 1e-6, invalid at t < 0 or t >= max_angle) and keep in
        ``self.trace`` what each decision compared, per step [steps, ...] (NaN once a point has stopped)."""
        u, v = torch.as_tensor(u, dtype=F64), torch.as_tensor(v, dtype=F64)
        x0, y0 = (u - self.cx) / self.fx, (v - self.cy) / self.fy
        if rule == "reference":
            return self._unproject_reference(x0, y0)
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

    def _unproject_reference(self, x0, y0):
        nan = torch.full_like(x0, math.nan)
        trace = {}

        def rec(key, live, val):
            trace.setdefault(key, []).append(torch.where(live, val, nan))

        if self.kind == "pinhole":
            x, y = x0.clone(), y0.clone()
            ok = torch.full_like(x0, not self.distorted, dtype=torch.bool)
            live = torch.full_like(ok, self.distorted)
            k, p, s = self.k, self.p, self.s
            for _ in range(5 if self.distorted else 0):
                r2 = x * x + y * y
                num = 1 + r2 * (k[0] + r2 * (k[1] + r2 * k[2]))
                den = 1 + r2 * (k[3] + r2 * (k[4] + r2 * k[5]))
                icd = num / den
                rec("icd", live, icd)
                live = live & (icd > 0)
                dicd = ((k[0] + r2 * (2 * k[1] + 3 * r2 * k[2])) - icd * (k[3] + r2 * (2 * k[4] + 3 * r2 * k[5]))) / den
                gx, gy = s[0] + 2 * s[1] * r2, s[2] + 2 * s[3] * r2
                Dx = icd * x + p[0] * 2 * x * y + p[1] * (r2 + 2 * x * x) + r2 * (s[0] + r2 * s[1])
                Dy = icd * y + p[0] * (r2 + 2 * y * y) + p[1] * 2 * x * y + r2 * (s[2] + r2 * s[3])
                J0 = icd + 2 * x * x * dicd + 2 * p[0] * y + 6 * p[1] * x + 2 * x * gx
                J1 = 2 * x * y * dicd + 2 * p[0] * x + 2 * p[1] * y + 2 * y * gx
                J2 = 2 * x * y * dicd + 2 * p[0] * x + 2 * p[1] * y + 2 * x * gy
                J3 = icd + 2 * y * y * dicd + 6 * p[0] * y + 2 * p[1] * x + 2 * y * gy
                det = J0 * J3 - J1 * J2
                rec("det", live, det)
                rec("jinv", live, torch.maximum(J3.abs() + J1.abs(), J0.abs() + J2.abs()) / det.abs())  # |J^-1|_inf
                live = live & (det.abs() >= 1e-6)
                ex, ey = x0 - Dx, y0 - Dy
                sx, sy = (J3 * ex - J1 * ey) / det, (J0 * ey - J2 * ex) / det
                x, y = torch.where(live, x + sx, x), torch.where(live, y + sy, y)
                step = torch.maximum(sx.abs(), sy.abs())
                rec("step", live, step)
                conv = live & (step < 1e-6)
                ok, live = ok | conv, live & ~conv
            self.trace = {key: torch.stack(v) for key, v in trace.items()}
            d = torch.stack([x, y, torch.ones_like(x)], -1)
            return d / d.norm(dim=-1, keepdim=True), ok
        delta = torch.sqrt(x0 * x0 + y0 * y0)
        t = self.inv_slope * delta
        live = torch.ones_like(delta, dtype=torch.bool)
        for _ in range(20):
            dx = (self._fe(t) - delta) / self._dfe(t)
            t = torch.where(live, t - dx, t)
            rec("step", live, dx.abs())
            live = live & ~(dx.abs() < 1e-6)
        self.trace = {key: torch.stack(v) for key, v in trace.items()}
        self.trace["t"] = t
        ok = ~live & (t >= 0) & (t < self.max_angle)
        big = delta >= 1e-6
        sc = torch.where(big, torch.sin(t) / torch.where(big, delta, torch.ones_like(delta)), torch.zeros_like(t))
        d = torch.stack([sc * x0, sc * y0, torch.where(big, torch.cos(t), torch.ones_like(t))], -1)
        return torch.where(ok[..., None], d, torch.tensor([0.0, 0.0, 1.0], dtype=F64)), ok


def quat_to_rotmat(q):
    q = q / q.norm(dim=-1, keepdim=True)
    w, x, y, z = q.unbind(-1)
    return torch.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y),
    ], -1).reshape(q.shape[:-1] + (3, 3))


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


def quat_from_rotmat(R):
    """Unit quaternion (w, x, y, z) of a rotation matrix [3, 3], from its largest component."""
    R = torch.as_tensor(R, dtype=F64)
    f = torch.stack([R[0, 0] + R[1, 1] + R[2, 2], R[0, 0] - R[1, 1] - R[2, 2], R[1, 1] - R[0, 0] - R[2, 2],
                     R[2, 2] - R[0, 0] - R[1, 1]])
    big = int(torch.argmax(f))  # the first of equal maxima, as a strict > scan
    v = torch.sqrt(f[big] + 1) * 0.5
    m = 0.25 / v
    wx, wy, wz = (R[2, 1] - R[1, 2]) * m, (R[0, 2] - R[2, 0]) * m, (R[1, 0] - R[0, 1]) * m
    xy, xz, yz = (R[1, 0] + R[0, 1]) * m, (R[0, 2] + R[2, 0]) * m, (R[2, 1] + R[1, 2]) * m
    return torch.stack([(v, wx, wy, wz), (wx, v, xy, xz), (wy, xy, v, yz), (wz, xz, yz, v)][big])


def slerp(q0, q1, a):
    """Normalised slerp of two unit quaternions at a (a tensor [P], not clamped) -> [P, 4]: the short arc, a
    component-wise lerp when cos(theta) > 1 - FLT_EPSILON."""
    a = torch.as_tensor(a, dtype=F64).reshape(-1, 1)
    c = float((q0 * q1).sum())
    if c < 0:
        q1, c = -q1, -c
    if c > 1 - FLT_EPS:
        q = q0 * (1 - a) + q1 * a
    else:
        th = math.acos(c)
        q = (torch.sin((1 - a) * th) * q0 + torch.sin(a * th) * q1) / math.sin(th)
    return q / q.norm(dim=-1, keepdim=True)


def frame_time(shutter, W, H, u, v):
    """Relative frame time of image points (u, v): that of their row (or column)."""
    u, v = torch.as_tensor(u, dtype=F64), torch.as_tensor(v, dtype=F64)
    if shutter == TOP_TO_BOTTOM:
        return torch.floor(v) / (H - 1)
    if shutter == LEFT_TO_RIGHT:
        return torch.floor(u) / (W - 1)
    if shutter == BOTTOM_TO_TOP:
        return (H - torch.ceil(v)) / (H - 1)
    return (W - torch.ceil(u)) / (W - 1)


class ShutterPoses:
    """A rolling-shutter camera: its start and end poses (row-major 4x4 view matrices) as quaternions and translations,
    and the shutter type; ``at(a)`` -> (R [P, 3, 3], t [P, 3]) at relative frame times a [P]: translation lerp,
    rotation slerp."""

    def __init__(self, viewmat, viewmat_rs, shutter):
        vm0, vm1 = torch.as_tensor(viewmat, dtype=F64), torch.as_tensor(viewmat_rs, dtype=F64)
        self.q0, self.q1 = quat_from_rotmat(vm0[:3, :3]), quat_from_rotmat(vm1[:3, :3])
        self.t0, self.t1 = vm0[:3, 3], vm1[:3, 3]
        self.shutter = shutter

    def at(self, a):
        a = torch.as_tensor(a, dtype=F64).reshape(-1)
        t = (1 - a)[:, None] * self.t0 + a[:, None] * self.t1
        return quat_to_rotmat(slerp(self.q0, self.q1, a)), t


def rs_project(points, cam, poses: ShutterPoses, margin):
    """World points [P, 3] -> (uv [P, 2], valid [P], edge [P]) through a rolling shutter: start from the start pose's
    projection if valid, else the end pose's (neither: invalid, at the end pose's point); then re-project at the frame
    time of the current point until that time repeats, at most 10 times.  ``edge``: a point whose row (or column)
    coordinate came within 1e-3 pixel of a boundary on the way, where float32 may pick the neighbouring row's pose."""
    P = points.shape[0]

    def proj(a):
        R, t = poses.at(a)
        return cam.project(torch.einsum("pij,pj->pi", R, points) + t, margin)

    uv0, ok0 = proj(torch.zeros(P, dtype=F64))
    uv1, ok1 = proj(torch.ones(P, dtype=F64))
    uv = torch.where(ok0[:, None], uv0, uv1)
    valid = ok0 | ok1
    live = valid.clone()
    prev = torch.full((P,), -math.inf, dtype=F64)
    coord = 1 if poses.shutter in (TOP_TO_BOTTOM, BOTTOM_TO_TOP) else 0
    edge = torch.zeros(P, dtype=torch.bool)
    for _ in range(RS_ITERATIONS):
        a = frame_time(poses.shutter, cam.W, cam.H, uv[:, 0], uv[:, 1])
        x = uv[:, coord]
        edge = edge | (live & ((x - torch.round(x)).abs() < 1e-3))
        live = live & (a != prev)
        if not bool(live.any()):
            break
        prev = torch.where(live, a, prev)
        uv_n, ok_n = proj(a)
        uv = torch.where(live[:, None], uv_n, uv)
        valid = torch.where(live, ok_n, valid)
    return uv, valid, edge


def rs_sh_viewmat(viewmat, viewmat_rs):
    """[..., 4, 4] view matrices [I | -c] with c the mean of the two poses' positions -R^T t: the camera position the
    SH view directions of a rolling-shutter camera are taken from."""
    vm0, vm1 = torch.as_tensor(viewmat, dtype=F64), torch.as_tensor(viewmat_rs, dtype=F64)
    pos = lambda vm: -torch.einsum("...ji,...j->...i", vm[..., :3, :3], vm[..., :3, 3])  # noqa: E731
    out = torch.zeros(vm0.shape, dtype=F64)
    out[..., :3, :3] = torch.eye(3, dtype=F64)
    out[..., :3, 3] = -0.5 * (pos(vm0) + pos(vm1))
    out[..., 3, 3] = 1
    return out


def ut_projection(means, quats, scales, opacities, pose, cam, eps2d=0.3, near_plane=0.01, far_plane=1e10,
                  radius_clip=0.0, ut=None, global_z_order=True):
    """One camera, N gaussians; ``pose`` a view matrix [4, 4] or a ShutterPoses.  Returns dict of float64 radii [N, 2]
    (0: culled), means2d, depths, conics, compensations, the unrounded radii, the sigma points' validity and
    ``rs_edge`` [N]: the rows with a sigma point near a row (column) boundary of a rolling shutter, where float32 may
    take the neighbouring row's pose.  Under a rolling shutter the near / far cull and the depth take the mid-frame
    pose; with global_z_order=False they take |mean_c| instead of z."""
    ut = dict(UT_DEFAULTS, **(ut or {}))
    means, quats, scales = (torch.as_tensor(t, dtype=F64) for t in (means, quats, scales))
    a, kap = ut["alpha"], ut["kappa"]
    lam = a * a * (3 + kap) - 3
    w_m = [lam / (3 + lam)] + [1 / (2 * (3 + lam))] * 6
    w_c = [lam / (3 + lam) + 1 - a * a + ut["beta"]] + [1 / (2 * (3 + lam))] * 6
    Rq = quat_to_rotmat(quats)
    delta = math.sqrt(3 + lam) * Rq * scales[:, None, :]  # column i = spread * s_i * R[:, i]
    pts = torch.stack([means] + [means + delta[..., i] for i in range(3)] + [means - delta[..., i] for i in range(3)], 1)
    margin = ut["in_image_margin_factor"]
    if isinstance(pose, ShutterPoses):
        uv, valid, edge = rs_project(pts.reshape(-1, 3), cam, pose, margin)
        uv, valid, rs_edge = uv.reshape(pts.shape[:-1] + (2,)), valid.reshape(pts.shape[:-1]), edge.reshape(pts.shape[:-1]).any(1)
        Rs, ts = pose.at(torch.tensor([0.5], dtype=F64))
        R, t = Rs[0], ts[0]
    else:
        vm = torch.as_tensor(pose, dtype=F64)
        R, t = vm[:3, :3], vm[:3, 3]
        uv, valid = cam.project(pts @ R.T + t, margin)
        rs_edge = torch.zeros(len(means), dtype=torch.bool)
    wm, wc = torch.tensor(w_m, dtype=F64), torch.tensor(w_c, dtype=F64)
    mean2d = (wm[None, :, None] * uv).sum(1)
    du = uv - mean2d[:, None]
    cov = (wc[None, :, None, None] * du[..., :, None] * du[..., None, :]).sum(1)
    ok = valid.all(1) if ut["require_all_sigma_points_valid"] else valid.any(1)
    zc = means @ R.T[:, 2] + t[2] if global_z_order else (means @ R.T + t).norm(dim=-1)
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
        "rs_edge": rs_edge,
    }


def pixel_rays(pose, cam):
    """World rays of every pixel centre: origins [H*W, 3], unit directions [H*W, 3], valid [H*W]; ``pose`` a view
    matrix or a ShutterPoses, under which each pixel's ray leaves at the pose of its row (column)."""
    jj, ii = torch.meshgrid(torch.arange(cam.W, dtype=F64), torch.arange(cam.H, dtype=F64), indexing="xy")
    u, v = jj.reshape(-1) + 0.5, ii.reshape(-1) + 0.5
    d, ok = cam.unproject(u, v)
    if isinstance(pose, ShutterPoses):
        R, t = pose.at(frame_time(pose.shutter, cam.W, cam.H, u, v))
        return -torch.einsum("pji,pj->pi", R, t), torch.einsum("pji,pj->pi", R, d), ok
    vm = torch.as_tensor(pose, dtype=F64)
    R, t = vm[:3, :3], vm[:3, 3]
    return (-(R.T @ t)).expand(d.shape), d @ R, ok


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


def eval3d_render(means, quats, scales, colors, opacities, pose, cam, isect_offsets, flatten_ids, C, N, image_index,
                  background=None, mask=None):
    """Composites one image (index image_index of the [I] = [B*C] images, seen from ``pose``, a view matrix or a
    ShutterPoses) from its tile lists, front to back.  means /
    quats / scales [B*N, *], colors [I*N, D], opacities [I*N] (float64 tensors, autograd flows through).  Returns
    (render_colors [H, W, D], render_alphas [H, W, 1], margins [H, W]: the smallest distance of any decision taken at the
    pixel from its threshold, relative)."""
    H, W, D = cam.H, cam.W, colors.shape[-1]
    th, tw = isect_offsets.shape[-2:]
    offs = isect_offsets.reshape(-1).tolist()
    n_isects = len(flatten_ids)
    ro, rd, rok = pixel_rays(pose, cam)
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
