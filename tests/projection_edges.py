"""Adversarial sweep for the projection and tile-intersection stages, and its float64 truth (no GPU needed).

Every visibility decision of a frame is taken by the projection (near / far plane, det_blur > 0, the opacity threshold
op * compensation >= 1/255, the radius ceil(extend * sqrt(c00)), radius_clip, the off-screen test) and by the tile
intersection (AccuTile / SNUGBOX or the radius AABB).  The sweep puts rows right at those decisions, for the pinhole,
orthographic and fisheye cameras, and tags every row with its class so that failures and undecided counts are reported
per class.  Most rows are built in camera space and mapped to world space through the camera's pose.

The truth of a row is the float64 oracle evaluated on the float32 inputs (oracle/gso.py, ``_f64``), plus the small
vectorised numpy restatement of the decision quantities below (``_quantities``), which the oracle does not return.
Every threshold in the truth is the float32 value the kernels compare with (near / far plane, eps2d, radius_clip,
1/255, 3.33, 0.005, 0.3, 1e-7): at z = float32(0.01) the kernel keeps a row that a float64 0.01 would cull.

Budgets.  Each float64 quantity is re-evaluated at 8 seeded relative perturbations of the float32 inputs of size
4 * 2^-24.  The budget beta of a quantity is 4x the largest deviation, plus the float32 / float64 difference of the
constant it is compared with, plus a few ulp of its own magnitude; fisheye quantities are widened by the documented
atan2f error (3 ulp).  Two quantities are computed exactly by the kernels and get beta = 0: pc.z when the camera's
third pose row is (0, 0, 1, 0), and the orthographic means2d when the camera is the identity with fx = fy = 1,
cx = cy = 0 (products with 0 and 1 and sums with 0 are exact in float32).  A row is *decided* when every margin on its
path through the kernel exceeds its beta (or is exact).  The same perturbation spread gives beta for each output
value; the matrix products and determinants also get a random error of their float32 rounding in the perturbed
evaluations, since perturbing the inputs alone leaves a needle's short axis exact.  Gradients are the float64 oracle
backward of the decided rows, fed that forward's conics and compensations, at the same perturbations (the world
covariance carries the random rounding error there), with one gaussian per batch element so that each row's share of
v_viewmats is known.

A radius of 2^31 or more is INT32_MAX: the kernels convert with cvt.rzi.s32.f32, which saturates (and maps NaN to 0);
the oracle converts the same way.
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

from oracle import gso

ULP = 2.0**-24
INT32_MAX = 2**31 - 1


def F32(v):
    return float(np.float32(v))


NEAR, FAR = F32(0.01), F32(100.0)
ALPHA_TH = F32(np.float32(1.0) / np.float32(255.0))
EXTEND = F32(3.33)
FLOOR = F32(np.float32(0.005) * np.float32(0.005))
CLAMP = F32(0.3)
FISHEYE_EPS = F32(1e-7)
RCLIP = 5.0  # radius_clip of the clip configuration (rows of class "radius_clip" have max(rx, ry) == 5)
N_PERTURB = 8
W, H = 640, 480


def _rot(axis, angle):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K


def _camera(model, fx, fy, cx, cy, R, t):
    vm = np.eye(4)
    vm[:3, :3], vm[:3, 3] = R, t
    vm = vm.astype(np.float32)
    if model == "pinhole" and R[2, 2] == 1.0:
        vm[2, :] = (0.0, 0.0, 1.0, 0.0)  # an exact third row: pc.z == mean.z in float32
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    exact_z = bool((vm[2] == np.array([0, 0, 1, 0], np.float32)).all())
    exact_m2 = model == "ortho" and (vm == np.eye(4, dtype=np.float32)).all() and (fx, fy, cx, cy) == (1, 1, 0, 0)
    return dict(model=model, viewmat=vm, K=K, exact_z=exact_z, exact_m2=bool(exact_m2))


# pin0: off-centre principal point (asymmetric clamp limits), fx != fy, rotated about the optical axis (a non-trivial
# pose gradient with an exact depth row); pin1: the second camera of the C = 2 runs; ortho: unit focal lengths, so that
# means2d lands on exact integers; fisheye: a wide field (theta up to pi / 2 stays on the 640 x 480 image)
CAMS = {
    "pin0": _camera("pinhole", 500.0, 560.0, 300.5, 260.25, _rot((0, 0, 1), 0.3), (0.2, -0.1, 0.0)),
    "pin1": _camera("pinhole", 420.0, 420.0, 330.0, 230.0, _rot((0.3, 1.0, 0.2), 0.12), (0.1, 0.05, 0.3)),
    "ortho": _camera("ortho", 1.0, 1.0, 0.0, 0.0, np.eye(3), (0, 0, 0)),
    "fisheye": _camera("fisheye", 200.0, 200.0, 320.0, 240.0, np.eye(3), (0, 0, 0)),
}
FAMILY_CAMS = {"pinhole": ("pin0", "pin1"), "ortho": ("ortho",), "fisheye": ("fisheye",)}


def _lims(cam):
    K = cam["K"].astype(np.float64)
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    return ((W - cx) / fx + CLAMP * 0.5 * W / fx, cx / fx + CLAMP * 0.5 * W / fx,
            (H - cy) / fy + CLAMP * 0.5 * H / fy, cy / fy + CLAMP * 0.5 * H / fy)


# ------------------------------------------------------------------------------------------------------------------
# the sweep
class _Rows:
    def __init__(self, cam, rng):
        self.cam, self.rng, self.rows = CAMS[cam], rng, []

    def add(self, cls, pc, scale, quat=None, op=None, covar=None, world=False):
        rng = self.rng
        if quat is None:
            quat = rng.standard_normal(4)
            quat /= np.linalg.norm(quat)
        if op is None:
            op = rng.uniform(0.05, 1.0)
        pc = np.asarray(pc, np.float64)
        if world:
            mean = pc
        else:
            vm = self.cam["viewmat"].astype(np.float64)
            with np.errstate(invalid="ignore"):
                mean = vm[:3, :3].T @ (pc - vm[:3, 3])
        scale = np.broadcast_to(np.asarray(scale, np.float64), (3,))
        if covar is None:
            covar = _covar6(np.asarray(quat, np.float64), scale)
        self.rows.append((cls, mean, np.asarray(quat, np.float64), scale,
                          float(op), np.asarray(covar, np.float64)))

    def arrays(self):
        with np.errstate(over="ignore", invalid="ignore"):
            f = lambda k: np.ascontiguousarray(np.array([r[k] for r in self.rows], np.float64).astype(np.float32))  # noqa: E731
            return dict(cls=np.array([r[0] for r in self.rows]), means=f(1), quats=f(2), scales=f(3), opacities=f(4),
                        covars=f(5))


def _covar6(q, s):
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        R = _quat_rot(q[None])[0]
        M = R * s[None, :]
        c = M @ M.T
    return np.array([c[0, 0], c[0, 1], c[0, 2], c[1, 1], c[1, 2], c[2, 2]])


def _quat_rot(q):
    """[..., 4] wxyz (normalised here, as the kernels do) -> [..., 3, 3]"""
    q = q / np.sqrt((q * q).sum(-1, keepdims=True))
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    return np.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y),
    ], -1).reshape(q.shape[:-1] + (3, 3))


def _ulps(v, ks):
    """float32 neighbours of v: k steps up (k > 0) or down (k < 0)"""
    out = []
    for k in ks:
        x = np.float32(v)
        for _ in range(abs(k)):
            x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf))
        out.append(float(x))
    return out


_AXIS_QUATS = ((1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0), (0, 0, 0, 1), (math.sqrt(0.5), 0, 0, math.sqrt(0.5)),
               (0.6, 0, 0.8, 0), (0, 0.6, 0, -0.8))


def _common_classes(r, rng, fx, n_bulk, z_exact):
    """depth, covariance, opacity, degenerate and bulk rows, centred on the optical axis region of camera r"""
    def on_screen(z, spread=0.35):
        return np.array([rng.uniform(-spread, spread) * z, rng.uniform(-spread, spread) * z, z])

    # depth: exactly at / a few ulp around the near and far planes (exact when the pose's depth row is exact), and
    # z over 1e-2 .. 1e4
    for plane in (NEAR, FAR):
        for z in _ulps(plane, (-4, -3, -2, -1, 0, 1, 2, 3, 4)):
            for _ in range(3 if z_exact else 1):
                r.add("depth", on_screen(z), z * rng.uniform(0.01, 0.1))
    for z in 10.0 ** rng.uniform(-2, 4, 120):
        r.add("depth", on_screen(z), z * rng.uniform(0.003, 0.1))
    # covariance: scales 1e-6 .. 1e7 (rx beyond 2^31), anisotropy up to 1e6, axis-aligned and random rotations,
    # quaternion norms 1e-3 .. 1e3, zero components
    for i in range(700):
        # most scales keep rx below 2^22, where the float32 ceil is exact; one in six reaches rx >= 2^31
        big = i % 6 == 0
        z = rng.uniform(0.5, 2.5) if big else (rng.uniform(0.5, 20.0) if i % 4 else 2.0)
        base = 10.0 ** (rng.uniform(6.5, 7) if big else rng.uniform(-6, 3))
        an = 10.0 ** rng.uniform(0, 6) if i % 3 else 1.0
        s = base * np.array([1.0, an**-0.5, 1.0 / an])
        rng.shuffle(s)
        q = np.array(_AXIS_QUATS[i % len(_AXIS_QUATS)], np.float64) if i % 2 else rng.standard_normal(4)
        q = q * 10.0 ** rng.uniform(-3, 3)
        r.add("covariance", on_screen(z), s, quat=q, op=rng.uniform(0.1, 1.0))
    # the radius >= 2^31 probe: z = 2, scales (1e7, 1e7, 1e-3), opacity 0.9
    for _ in range(4):
        r.add("radius>=2^31", on_screen(2.0, 0.05), (1e7, 1e7, 1e-3), quat=(1, 0, 0, 0), op=0.9)
    # direct covariances (used by the covars configurations; quats / scales rows stay ordinary)
    v = rng.standard_normal((8, 3))
    for i in range(40):
        z = rng.uniform(1, 10)
        a = v[i % 8] * z * 0.05
        b = v[(i + 3) % 8] * z * 0.05
        kind = i % 5
        if kind == 0:
            c = np.outer(a, a)  # rank 1
        elif kind == 1:
            c = np.outer(a, a) + np.outer(b, b)  # rank 2
        elif kind == 2:
            c = np.outer(a, a) - 0.5 * np.outer(b, b)  # indefinite
        elif kind == 3:
            c = -np.outer(a, a) - np.eye(3) * 1e-4 * z * z  # negative definite
        else:
            c = np.outer(a, a) + np.eye(3) * 1e-3 * z * z
            c[i % 3, (i + 1) % 3] = c[(i + 1) % 3, i % 3] = (math.nan, math.inf, -math.inf, 1e30)[i // 5 % 4]
        r.add("covars", on_screen(z), z * 0.05, covar=[c[0, 0], c[0, 1], c[0, 2], c[1, 1], c[1, 2], c[2, 2]])
    # opacity: around 1/255, op * comp around 1/255 (isotropic on-axis rows, whose compensation is known in closed
    # form), extend = sqrt(2 log(255 op)) around 3.33, compensation ratios below the 0.005^2 floor
    for k in (-4, -3, -2, -1, 0, 1, 2, 3, 4):
        for op in _ulps(ALPHA_TH, (k,)) + [ALPHA_TH * (1 + 1e-4 * np.sign(k or 1) * abs(k))]:
            r.add("opacity", on_screen(rng.uniform(1, 10)), rng.uniform(0.002, 0.05), op=op)
    fxy = (CAMS_FOCAL[r.cam_name])
    for i in range(60):
        z = rng.uniform(1, 10)
        s = z / fxy[0] * 10.0 ** rng.uniform(-1.0, 0.5)
        a, b = (fxy[0] * s / z) ** 2, (fxy[1] * s / z) ** 2
        comp = math.sqrt(a * b / ((a + 0.3) * (b + 0.3)))
        d = (1e-3, -1e-3, 1e-5, -1e-5, 3e-7, -3e-7)[i % 6]
        r.add("opacity*comp", np.array([0.0, 0.0, z]), s, quat=(1, 0, 0, 0), op=min(ALPHA_TH / comp * (1 + d), 1.0))
    for d in (1e-3, -1e-3, 1e-5, -1e-5, 1e-6, -1e-6) * 4:
        op = math.exp((EXTEND * (1 + d)) ** 2 / 2) * ALPHA_TH
        r.add("extend", on_screen(rng.uniform(1, 10)), rng.uniform(0.002, 0.05), op=op)
    for _ in range(30):
        z = rng.uniform(1, 10)
        r.add("ratio_floor", on_screen(z), z * np.array([0.05, 10.0 ** rng.uniform(-9, -6), 10.0 ** rng.uniform(-9, -6)]))
    # eps2d = 0: sub-pixel gaussians and needles, whose conics are unbounded without the blur
    for _ in range(100):
        z = rng.uniform(0.5, 20)
        s = z / fx * 10.0 ** rng.uniform(-4, 0.5) * np.array([1.0, 10.0 ** rng.uniform(-3, 0), 10.0 ** rng.uniform(-3, 0)])
        r.add("eps2d=0", on_screen(z), s)
    # degenerate: NaN / inf means, zero quaternion, NaN / inf scales, NaN / negative opacity
    nan, inf = math.nan, math.inf
    for pc in ((nan, 0, 2), (0, nan, 2), (0, 0, nan), (inf, 0, 2), (0, -inf, 2), (0, 0, inf)):
        r.add("degenerate", pc, 0.05)
    for q, s, op in (((0, 0, 0, 0), 0.05, 0.5), ((1, 0, 0, 0), nan, 0.5), ((1, 0, 0, 0), inf, 0.5),
                     ((1, 0, 0, 0), (0.05, nan, 0.05), 0.5), ((nan, 0, 0, 1), 0.05, 0.5), ((1, 0, 0, 0), 0.05, nan),
                     ((1, 0, 0, 0), 0.05, -0.5), ((1, 0, 0, 0), 0.05, 0.0)):
        r.add("degenerate", on_screen(2.0), s, quat=q, op=op)
    # bulk: ordinary gaussians
    for _ in range(n_bulk):
        z = 10.0 ** rng.uniform(-0.3, 1.5)
        r.add("bulk", on_screen(z, 0.6), z * 10.0 ** rng.uniform(-3, -0.5) * 10.0 ** rng.uniform(-0.5, 0.5, 3))


CAMS_FOCAL = {k: (float(c["K"][0, 0]), float(c["K"][1, 1])) for k, c in CAMS.items()}


def _pinhole_rows(rng):
    r = _Rows("pin0", rng)
    r.cam_name = "pin0"
    fx, fy = CAMS_FOCAL["pin0"]
    _common_classes(r, rng, fx, 1300, True)
    # clamp: x/z and y/z at +-lim +- a few ulp, +-1e-3, and 1.3 .. 10x beyond the 1.3 x FOV clamp
    lxp, lxn, lyp, lyn = _lims(CAMS["pin0"])
    facs = [1 + k * ULP for k in (-4, -2, -1, 1, 2, 4)] + [1 - 1e-3, 1 + 1e-3, 1.3, 2.0, 5.0, 10.0]
    for axis in (0, 1):
        for lim, sgn in (((lxp, 1), (lxn, -1)) if axis == 0 else ((lyp, 1), (lyn, -1))):
            for f in facs:
                for rep in range(6):
                    z = rng.uniform(1, 10)
                    pc = np.array([rng.uniform(-0.3, 0.3) * z, rng.uniform(-0.3, 0.3) * z, z])
                    pc[axis] = sgn * lim * f * z
                    s = z * (10.0 ** rng.uniform(-0.3, 0.7) if f > 1.01 else 10.0 ** rng.uniform(-2, 0))
                    r.add("clamp", pc, s)
    # off-screen: the 3.33-sigma edge of an isotropic gaussian at the image border (approximately: pinhole means2d
    # rounds)
    for i in range(120):
        z = rng.uniform(1, 10)
        s = z / fx * rng.uniform(1, 30)
        rx = math.ceil(3.33 * math.sqrt((fx * s / z) ** 2 + 0.3))
        edge = i % 4
        d = rng.uniform(-1.5, 1.5)
        u = (-rx + d, W + rx + d, -rx + d, H + rx + d)[edge]
        px, py = (u, rng.uniform(0, H)) if edge < 2 else (rng.uniform(0, W), u)
        K = CAMS["pin0"]["K"].astype(np.float64)
        pc = np.array([(px - K[0, 2]) / K[0, 0] * z, (py - K[1, 2]) / K[1, 1] * z, z])
        r.add("offscreen", pc, s, quat=(1, 0, 0, 0))
    # radius_clip: isotropic on-axis rows with max(rx, ry) == RCLIP (culled by radius_clip = RCLIP) or RCLIP + 1
    for i in range(48):
        z = rng.uniform(1, 10)
        target = RCLIP + (i % 2) - rng.uniform(0.25, 0.75)
        s = z / fy * math.sqrt((target / 3.33) ** 2 - 0.3)
        r.add("radius_clip", np.array([rng.uniform(-0.05, 0.05) * z, rng.uniform(-0.05, 0.05) * z, z]), s,
              quat=(1, 0, 0, 0), op=1.0)
    return r.arrays()


def _ortho_rows(rng):
    r = _Rows("ortho", rng)
    r.cam_name = "ortho"
    _common_classes(r, rng, 1.0, 400, True)
    # off-screen, exactly: means2d = (x, y) in float32, the radius an integer R (the 3.33-sigma edge R - u,
    # u in [0.25, 0.75]) and x = -R, W + R (or y = -R, H + R) exactly, a few ulp off, or a quarter pixel off
    for i in range(200):
        R = int(rng.randint(3, 40))
        s = math.sqrt(((R - rng.uniform(0.25, 0.75)) / 3.33) ** 2 - 0.3)
        edge = i % 4
        base = (-R, W + R, -R, H + R)[edge]
        k = (0, 0, 0, 1, -1, 2, -2, 0.25, -0.25)[i // 4 % 9]
        v = base + k if isinstance(k, float) else _ulps(base, (k,))[0]
        x, y = (v, rng.uniform(0, H)) if edge < 2 else (rng.uniform(0, W), v)
        r.add("offscreen", np.array([x, y, rng.uniform(1, 10)]), s, quat=(1, 0, 0, 0), op=1.0)
    return r.arrays()


def _fisheye_rows(rng):
    r = _Rows("fisheye", rng)
    r.cam_name = "fisheye"
    _common_classes(r, rng, 200.0, 500, True)
    # exactly on the optical axis, xy_len 1e-7 .. 1e-3, x = 0 with y != 0 (and y = 0 with x != 0), theta near pi / 2
    for _ in range(24):
        z = rng.uniform(0.5, 20)
        r.add("fisheye_axis", np.array([0.0, 0.0, z]), z * rng.uniform(0.002, 0.05))
    for _ in range(80):
        z = rng.uniform(0.5, 5)
        ln, ph = 10.0 ** rng.uniform(-7, -3), rng.uniform(0, 2 * math.pi)
        r.add("fisheye_axis", np.array([ln * math.cos(ph), ln * math.sin(ph), z]), z * rng.uniform(0.002, 0.05))
    for i in range(60):
        z = rng.uniform(0.5, 5)
        v = rng.choice((-1, 1)) * 10.0 ** rng.uniform(-7, 0) * z
        r.add("fisheye_x=0", np.array([0.0, v, z]) if i % 4 else np.array([v, 0.0, z]), z * rng.uniform(0.002, 0.05))
    for _ in range(60):
        ln, ph = rng.uniform(1, 10), rng.uniform(0, 2 * math.pi)
        z = ln * 10.0 ** rng.uniform(-2.5, -0.5)
        r.add("fisheye_theta", np.array([ln * math.cos(ph), ln * math.sin(ph), max(z, 0.0101)]), ln * rng.uniform(0.002, 0.05))
    for _ in range(300):
        th, ph, d = rng.uniform(0, 1.55), rng.uniform(0, 2 * math.pi), rng.uniform(1, 10)
        pc = d * np.array([math.sin(th) * math.cos(ph), math.sin(th) * math.sin(ph), math.cos(th)])
        r.add("fisheye_wide", pc, d * 10.0 ** rng.uniform(-3, -1))
    return r.arrays()


def make_sweep(seed=20261016):
    """{family: rows}; rows holds float32 means [N, 3], quats [N, 4], scales [N, 3], covars [N, 6], opacities [N] and
    the per-row class label `cls`.  Deterministic for a seed."""
    rng = np.random.RandomState(seed)
    return dict(pinhole=_pinhole_rows(rng), ortho=_ortho_rows(rng), fisheye=_fisheye_rows(rng))


@dataclasses.dataclass(frozen=True)
class Config:
    family: str
    C: int = 1
    covars: bool = False
    opacities: bool = True
    comp: bool = False
    eps2d: float = 0.3
    radius_clip: float = 0.0

    @property
    def cams(self):
        return FAMILY_CAMS[self.family][: self.C]

    def __str__(self):
        return (f"{self.family} C={self.C} {'covars' if self.covars else 'quats'}"
                f"{' opac' if self.opacities else ''}{' comp' if self.comp else ''} eps2d={self.eps2d} clip={self.radius_clip}")

    def camera_arrays(self):
        vm = np.ascontiguousarray(np.stack([CAMS[c]["viewmat"] for c in self.cams]))
        Ks = np.ascontiguousarray(np.stack([CAMS[c]["K"] for c in self.cams]))
        return vm, Ks

    def kwargs(self):
        return dict(width=W, height=H, eps2d=F32(self.eps2d), near_plane=NEAR, far_plane=FAR,
                    radius_clip=F32(self.radius_clip), calc_compensations=self.comp,
                    camera_model=self.family)


# every dense configuration: camera x {quats / scales, covars} x {with, without opacities} x calc_compensations, plus
# radius_clip = RCLIP and eps2d = 0 (unbounded conics)
CONFIGS = [Config(f, C=2 if f == "pinhole" else 1, covars=cv, opacities=op, comp=cp)
           for f in ("pinhole", "ortho", "fisheye") for cv in (False, True) for op in (True, False) for cp in (False, True)]
CONFIGS += [Config("pinhole", radius_clip=RCLIP), Config("pinhole", eps2d=0.0), Config("pinhole")]
# configurations whose backward budgets the float32 oracle is checked against (tests/test_projection_edges_cpu.py):
# with compensation, a second camera, covariance inputs or the non-pinhole models, needles make the backward's
# float32 cancellation larger than these budgets, so their gradients are not compared
GRAD_CONFIGS = [Config("pinhole"), Config("pinhole", radius_clip=RCLIP), Config("pinhole", eps2d=0.0)]


# ------------------------------------------------------------------------------------------------------------------
# the decision quantities, restated in numpy (float64)
def _inject(A, absA, absB, rng):
    """float32 rounding of the matrix product A = X Y: a random error of up to 8 ulp of (|X| |Y|) per entry"""
    if rng is None:
        return A
    return A + 8.0 * ULP * (absA @ absB) * rng.uniform(-1.0, 1.0, A.shape)


def _quantities(p, cam, cfg, rng=None):
    """p: float64 means / quats / scales / covars / opacities; cam: float64 viewmat / K.  Mirrors project_one.  With
    `rng`, the three matrix products (covariance, world -> camera, Jacobian) also get a random error of the size of
    their float32 rounding, which perturbing the inputs alone does not produce (e.g. a needle's short axis)."""
    vm, K = p["viewmat"], p["K"]
    R, t = vm[:3, :3], vm[:3, 3]
    m = p["means"]
    with np.errstate(all="ignore"):
        pc = m @ R.T + t
        x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
        if cfg.covars:
            c6 = p["covars"]
            cov = np.stack([c6[:, 0], c6[:, 1], c6[:, 2], c6[:, 1], c6[:, 3], c6[:, 4], c6[:, 2], c6[:, 4], c6[:, 5]],
                           -1).reshape(-1, 3, 3)
        else:
            M = _quat_rot(p["quats"]) * p["scales"][:, None, :]
            cov = _inject(M @ M.transpose(0, 2, 1), np.abs(M), np.abs(M).transpose(0, 2, 1), rng)
        covc = _inject(R @ cov @ R.T, np.abs(R) @ np.abs(cov), np.abs(R).T, rng)
        fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
        N = m.shape[0]
        J = np.zeros((N, 2, 3))
        out = dict(z=z)
        if cam["model"] == "pinhole":
            lxp = (W - cx) / fx + CLAMP * (0.5 * W / fx)
            lxn = cx / fx + CLAMP * (0.5 * W / fx)
            lyp = (H - cy) / fy + CLAMP * (0.5 * H / fy)
            lyn = cy / fy + CLAMP * (0.5 * H / fy)
            rz = 1.0 / z
            xz, yz = x * rz, y * rz
            cxz = np.where(xz > -lxn, xz, -lxn)
            cxz = np.where(cxz < lxp, cxz, lxp)
            cyz = np.where(yz > -lyn, yz, -lyn)
            cyz = np.where(cyz < lyp, cyz, lyp)
            J[:, 0, 0], J[:, 1, 1] = fx * rz, fy * rz
            J[:, 0, 2], J[:, 1, 2] = -fx * (z * cxz) * rz * rz, -fy * (z * cyz) * rz * rz
            m2x, m2y = fx * x * rz + cx, fy * y * rz + cy
            out.update(clamp=np.stack([xz - lxp, xz + lxn, yz - lyp, yz + lyn], -1),
                       clamp_scale=np.stack([np.abs(xz) + lxp, np.abs(xz) + lxn, np.abs(yz) + lyp, np.abs(yz) + lyn], -1),
                       tan=np.array([0.5 * W / fx, 0.5 * W / fx, 0.5 * H / fy, 0.5 * H / fy]))
        elif cam["model"] == "ortho":
            J[:, 0, 0], J[:, 1, 1] = fx, fy
            m2x, m2y = fx * x + cx, fy * y + cy
        else:
            e = FISHEYE_EPS
            xy_len = np.sqrt(x * x + y * y) + e
            theta = np.arctan2(xy_len, z + e)
            m2x = x * fx * theta / xy_len + cx
            m2y = y * fy * theta / xy_len + cy
            x2, y2, xy = x * x + e, y * y, x * y
            x2y2 = x2 + y2
            inv = 1.0 / (x2y2 + z * z)
            b = np.arctan2(xy_len, z) / xy_len / x2y2
            a = z * inv / x2y2
            J[:, 0] = np.stack([fx * (x2 * a + y2 * b), fx * xy * (a - b), -fx * x * inv], -1)
            J[:, 1] = np.stack([fy * xy * (a - b), fy * (y2 * a + x2 * b), -fy * y * inv], -1)
        c2 = _inject(J @ covc @ J.transpose(0, 2, 1), np.abs(J) @ np.abs(covc), np.abs(J).transpose(0, 2, 1), rng)
        c00, c01, c10, c11 = c2[:, 0, 0], c2[:, 0, 1], c2[:, 1, 0], c2[:, 1, 1]
        det_orig = c00 * c11 - c01 * c10
        c00b, c11b = c00 + F32(cfg.eps2d), c11 + F32(cfg.eps2d)
        det_blur = c00b * c11b - c01 * c10
        if rng is not None:  # the rounding of the two determinants, which cancel for needles
            det_orig = det_orig + 4.0 * ULP * (np.abs(c00 * c11) + np.abs(c01 * c10)) * rng.uniform(-1, 1, N)
            det_blur = det_blur + 4.0 * ULP * (np.abs(c00b * c11b) + np.abs(c01 * c10)) * rng.uniform(-1, 1, N)
        ratio = det_orig / det_blur
        comp = np.sqrt(np.where(ratio > FLOOR, ratio, FLOOR))
        if cfg.opacities:
            opc = p["opacities"] * comp if cfg.comp else p["opacities"]
            e2 = np.sqrt(2.0 * np.log(opc / ALPHA_TH))
            extend = np.where(e2 < EXTEND, e2, EXTEND)
        else:
            opc = np.full(N, np.inf)
            extend = np.full(N, EXTEND)
        rxq, ryq = extend * np.sqrt(c00b), extend * np.sqrt(c11b)
        big = np.max(np.abs(np.concatenate([cov.reshape(N, 9), covc.reshape(N, 9), c2.reshape(N, 4), J.reshape(N, 6),
                                            (c00b * c11b)[:, None], (c01 * c10)[:, None]], -1)), -1)
        big = np.where(np.isnan(big), np.inf, big)
        conic = np.stack([c11b, -c01, c00b], -1) / det_blur[:, None]
        out.update(m2x=m2x, m2y=m2y, det_blur=det_blur, conic=conic, det_scale=np.abs(c00b * c11b) + np.abs(c01 * c10), opc=opc,
                   rxq=rxq, ryq=ryq, big=big, comp=comp, c00b=c00b, c11b=c11b)
    return out


def _perturb(rows, cfg, k):
    """float64 inputs of perturbation k (k = 0: the float32 inputs themselves)"""
    rng = np.random.RandomState(1000 + k)
    vm, Ks = cfg.camera_arrays()
    out = {}
    for name, a in (("means", rows["means"]), ("quats", rows["quats"]), ("scales", rows["scales"]),
                    ("covars", rows["covars"]), ("opacities", rows["opacities"]), ("viewmats", vm), ("Ks", Ks)):
        a = a.astype(np.float64)
        if k:
            a = a * (1.0 + 4.0 * ULP * rng.uniform(-1.0, 1.0, a.shape))
        out[name] = a
    return out


def _dev(base, vals):
    with np.errstate(invalid="ignore"):
        d = np.max(np.abs(np.stack(vals) - base[None]), 0)
    return np.where(np.isnan(d) & np.isfinite(base), np.inf, np.nan_to_num(d, nan=0.0))


@dataclasses.dataclass
class Truth:
    radii: np.ndarray  # [C, N, 2] int64
    decided: np.ndarray  # [C, N]
    why: np.ndarray  # [C, N] name of the first decision within its budget (undecided rows)
    margin: np.ndarray  # [C, N] |margin| / beta of that decision
    values: dict  # means2d, depths, conics, compensations (float64 oracle)
    beta: dict
    inputs: dict  # the float64 inputs (perturbation 0)
    cls: np.ndarray


def truth(rows, cfg):
    """float64 truth of one configuration: per (camera, row) radii, decided flag, and output values with budgets."""
    ins = [_perturb(rows, cfg, k) for k in range(N_PERTURB + 1)]
    C, N = cfg.C, rows["means"].shape[0]
    finite_in = np.isfinite(rows["means"]).all(-1) & np.isfinite(rows["opacities"] if cfg.opacities else 0.0)
    finite_in &= (np.isfinite(rows["covars"]).all(-1) if cfg.covars else
                  np.isfinite(rows["quats"]).all(-1) & np.isfinite(rows["scales"]).all(-1))
    radii = np.zeros((C, N, 2), np.int64)
    decided = np.ones((C, N), bool)
    why = np.full((C, N), "", object)
    margin = np.full((C, N), np.inf)
    spreads = []
    for c, cname in enumerate(cfg.cams):
        cam = CAMS[cname]
        qs = []
        for k, p in enumerate(ins):
            pp = dict(p, viewmat=p["viewmats"][c], K=p["Ks"][c])
            qs.append(_quantities(pp, cam, cfg, np.random.RandomState(2000 + k) if k else None))
        q0 = qs[0]
        dev = {k: _dev(q0[k], [q[k] for q in qs[1:]]) for k in q0 if k not in ("tan",)}
        spreads.append(dict(m2=np.stack([dev["m2x"], dev["m2y"]], -1), conic=dev["conic"], z=dev["z"], comp=dev["comp"]))
        fish = cam["model"] == "fisheye"
        alive = np.ones(N, bool)
        dec = np.ones(N, bool)
        w = np.full(N, "", object)
        mg = np.full(N, np.inf)

        def stage(name, m, beta, cull):
            nonlocal alive, dec
            with np.errstate(invalid="ignore"):
                ok = (np.abs(m) > beta) | (beta == 0) | (np.isnan(m) & ~finite_in)
                ratio = np.where(beta > 0, np.abs(m) / np.where(beta > 0, beta, 1.0), np.inf)
            und = alive & dec & ~ok
            w[und] = name
            mg[und] = np.nan_to_num(ratio[und], nan=0.0)
            dec &= ~und
            alive &= ~cull

        with np.errstate(invalid="ignore"):
            bz = np.zeros(N) if cam["exact_z"] else 4.0 * dev["z"]
            z = q0["z"]
            stage("near", z - NEAR, bz, z < NEAR)
            stage("far", z - FAR, bz, z > FAR)
            over = finite_in & (q0["big"] > 1e38)  # float32 overflows at 3.4e38
            stage("overflow", np.where(over, 0.0, 1.0), np.where(over, 1.0, 0.0), np.zeros(N, bool))
            fw = 12.0 * ULP if fish else 0.0
            db = q0["det_blur"]
            stage("det_blur", db, 4.0 * dev["det_blur"] + (8.0 * ULP + fw) * q0["det_scale"], ~(db > 0))
            if cfg.opacities:
                opc = q0["opc"]
                bo = 4.0 * dev["opc"] + 8.0 * ULP * np.abs(opc) + abs(ALPHA_TH - 1.0 / 255.0)
                stage("opacity", opc - ALPHA_TH, bo, opc < ALPHA_TH)
            rr = []
            for key in ("rxq", "ryq"):
                v = q0[key]
                # float32 / float64 constants: 3.33, 1/255 inside the extend; atan2f for the fisheye Jacobian
                bv = 4.0 * dev[key] + (8.0 * ULP + 2 * fw) * np.abs(v) + 1e-7 * np.abs(v)
                frac = np.abs(v - np.round(v))
                m = np.where(v >= 2.0**31, v - 2.0**31, np.where(v < 2.0**22, frac, 0.0))
                stage(key[:2], m, np.where((v < 2.0**22) | (v >= 2.0**31), bv, 1.0), np.zeros(N, bool))
                rr.append((np.where(v >= 2.0**31, INT32_MAX, np.ceil(np.nan_to_num(np.minimum(v, 2.0**31), nan=0.0))), bv))
            (rx, brx), (ry, bry) = rr
            stage("radius_clip", np.ones(N), np.zeros(N), (rx <= cfg.radius_clip) & (ry <= cfg.radius_clip))
            if cam["exact_m2"]:
                bmx = bmy = np.zeros(N)
            else:
                ax = np.abs(q0["m2x"] - float(cam["K"][0, 2])), np.abs(q0["m2y"] - float(cam["K"][1, 2]))
                bmx = 4.0 * dev["m2x"] + 4.0 * ULP * (np.abs(q0["m2x"]) + rx) + 2 * fw * ax[0] + np.where(rx >= 2**22, brx, 0)
                bmy = 4.0 * dev["m2y"] + 4.0 * ULP * (np.abs(q0["m2y"]) + ry) + 2 * fw * ax[1] + np.where(ry >= 2**22, bry, 0)
            mx, my = q0["m2x"], q0["m2y"]
            stage("offscreen x+", mx + rx, bmx, mx + rx <= 0)
            stage("offscreen x-", mx - rx - W, bmx, mx - rx >= W)
            stage("offscreen y+", my + ry, bmy, my + ry <= 0)
            stage("offscreen y-", my - ry - H, bmy, my - ry >= H)
            if cam["model"] == "pinhole":  # the Jacobian clamp picks the backward branch
                for j in range(4):
                    bc = 4.0 * dev["clamp"][:, j] + 4.0 * ULP * q0["clamp_scale"][:, j] + abs(CLAMP - 0.3) * q0["tan"][j]
                    stage("clamp", q0["clamp"][:, j], bc, np.zeros(N, bool))
        vis = alive
        radii[c, vis, 0], radii[c, vis, 1] = rx[vis], ry[vis]
        decided[c], why[c], margin[c] = dec, w, mg
    # values: the float64 oracle at the perturbations
    vals, betas = _oracle_values(rows, cfg, ins)
    # widen by the spread of the same values computed with the float32 rounding of the matrix products
    fish = cfg.family == "fisheye"
    for k, key in (("means2d", "m2"), ("conics", "conic"), ("depths", "z"), ("compensations", "comp")):
        if k in betas:
            sp = np.stack([s_[key] for s_ in spreads])
            scale = np.abs(np.nan_to_num(vals[k], nan=0.0, posinf=0.0, neginf=0.0))
            if sp.ndim == 3:
                scale = scale.max(-1, keepdims=True)
            betas[k] = betas[k] + 4.0 * sp + (8.0 + (12.0 if fish else 0.0)) * ULP * scale
    return Truth(radii, decided, why, margin, vals, betas, ins[0], rows["cls"])


def _oracle_fwd(rows, cfg, p):
    kw = cfg.kwargs()
    return gso.fully_fused_projection(
        p["means"], p["covars"] if cfg.covars else None, p["quats"], p["scales"], p["viewmats"], p["Ks"], kw["width"],
        kw["height"], kw["eps2d"], kw["near_plane"], kw["far_plane"], kw["radius_clip"], cfg.comp, kw["camera_model"],
        p["opacities"] if cfg.opacities else None,
    )


def _row_beta(base, vals, fish, axis=-1, ulps=8.0):
    """4x the perturbation spread + `ulps` ulp of the row's largest magnitude (+ the atan2f widening for fisheye)"""
    with np.errstate(invalid="ignore"):
        scale = np.max(np.abs(np.nan_to_num(base, nan=0.0, posinf=0.0, neginf=0.0)), axis=axis, keepdims=True)
    return 4.0 * _dev(base, vals) + (ulps + (12.0 if fish else 0.0)) * ULP * scale


def _oracle_values(rows, cfg, ins):
    fish = cfg.family == "fisheye"
    outs = [_oracle_fwd(rows, cfg, p) for p in ins]
    names = ("radii", "means2d", "depths", "conics", "compensations")
    vals = dict(zip(names, outs[0]))
    betas = {}
    for i, k in enumerate(names[1:], 1):
        if outs[0][i] is None:
            continue
        base = outs[0][i] if outs[0][i].ndim == 3 else outs[0][i][..., None]
        others = [(o[i] if o[i].ndim == 3 else o[i][..., None]) for o in outs[1:]]
        b = _row_beta(base, others, fish)
        betas[k] = b if outs[0][i].ndim == 3 else b[..., 0]
    return vals, betas


# ------------------------------------------------------------------------------------------------------------------
# gradients
def subset(rows, idx):
    return {k: np.ascontiguousarray(v[idx]) for k, v in rows.items()}


def cotangents(cfg, N, seed=0):
    """seeded cotangents [C, N, *] of means2d, depths, conics (and compensations)"""
    rng = np.random.RandomState(seed)
    C = cfg.C
    return dict(v_means2d=rng.standard_normal((C, N, 2)), v_depths=rng.standard_normal((C, N)),
                v_conics=rng.standard_normal((C, N, 3)),
                v_compensations=rng.standard_normal((C, N)) if cfg.comp else None)


def _cov64(p, cfg, rng):
    """world covariance [N, 6] (triu) in float64, with a random error of 16 ulp of its float32 evaluation when rng"""
    if cfg.covars:
        c6 = p["covars"]
        if rng is not None:
            d = np.sqrt(np.abs(c6[:, [0, 0, 0, 3, 3, 5]] * c6[:, [0, 3, 5, 3, 5, 5]]))
            c6 = c6 + 16.0 * ULP * d * rng.uniform(-1, 1, c6.shape)
        return c6
    with np.errstate(invalid="ignore", over="ignore"):
        M = _quat_rot(p["quats"]) * p["scales"][:, None, :]
        cov = M @ M.transpose(0, 2, 1)
        if rng is not None:
            e = 16.0 * ULP * (np.abs(M) @ np.abs(M).transpose(0, 2, 1)) * rng.uniform(-1, 1, cov.shape)
            cov = cov + 0.5 * (e + e.transpose(0, 2, 1))
    return np.ascontiguousarray(cov.reshape(-1, 9)[:, [0, 1, 2, 4, 5, 8]])


def grad_truth(rows, cfg, tr, cot):
    """float64 gradients of the decided visible rows for the cotangents `cot` (zeroed elsewhere; returned as float32,
    which is what the kernels get).  Returns (grads, betas, cot32): v_means [N, 3], v_quats [N, 4] and v_scales [N, 3]
    or v_covars [N, 6], v_viewmats [C, 4, 4] and its per-row shares v_viewmats_rows [N, C, 4, 4].

    The oracle backward runs on the world covariance (one gaussian per batch element); quats / scales gradients are
    its covariance gradient through the oracle's quat_scale_to_covar_preci_bwd.  beta: 4x the spread over the 8
    perturbations + 32 ulp of the gaussian's largest gradient of that kind (44 for fisheye); v_viewmats: the l1 of
    the per-row budgets + 64 ulp of the l1 of the shares (the order of the float32 sum)."""
    C, N = cfg.C, rows["means"].shape[0]
    keep = tr.decided & (tr.radii > 0).all(-1)
    cot32 = {k: None if v is None else (v * (keep[..., None] if v.ndim == 3 else keep)).astype(np.float32)
             for k, v in cot.items()}
    fish = cfg.family == "fisheye"
    kw = cfg.kwargs()
    res = []
    for k in range(N_PERTURB + 1):
        p = _perturb(rows, cfg, k)
        c6 = _cov64(p, cfg, np.random.RandomState(3000 + k) if k else None)
        radii, m2, dep, con, comp = gso.fully_fused_projection(
            p["means"], c6, None, None, p["viewmats"], p["Ks"], W, H, kw["eps2d"], NEAR, FAR, kw["radius_clip"], cfg.comp,
            cfg.family, p["opacities"] if cfg.opacities else None,
        )
        radii = np.where(keep[..., None], radii, 0)
        b = lambda a: np.ascontiguousarray(np.swapaxes(a, 0, 1)[:, :, None])  # [C, N, ...] -> [N, C, 1, ...]  # noqa: E731
        vmb = np.ascontiguousarray(np.broadcast_to(p["viewmats"][None], (N, C, 4, 4)))
        Kb = np.ascontiguousarray(np.broadcast_to(p["Ks"][None], (N, C, 3, 3)))
        f8 = lambda a: None if a is None else b(a.astype(np.float64))  # noqa: E731
        v_means, v_cov, _, _, v_vm = gso.fully_fused_projection_bwd(
            np.ascontiguousarray(p["means"][:, None]), np.ascontiguousarray(c6[:, None]), None, None, vmb, Kb, W, H,
            kw["eps2d"], b(radii), b(con), None if comp is None else b(comp), f8(cot32["v_means2d"]), f8(cot32["v_depths"]),
            f8(cot32["v_conics"]), f8(cot32["v_compensations"]) if cfg.comp else None, True, cfg.family,
        )
        g = dict(v_means=v_means[:, 0], v_viewmats_rows=v_vm, _vcov=np.abs(v_cov[:, 0]).max(-1), _cov=c6)
        if cfg.covars:
            g["v_covars"] = v_cov[:, 0]
        else:
            with np.errstate(invalid="ignore"):
                g["v_quats"], g["v_scales"] = gso.quat_scale_to_covar_preci_bwd(
                    p["quats"], p["scales"], True, np.ascontiguousarray(v_cov[:, 0]), None)
        res.append(g)
    # The backward's float32 terms are far larger than its result where it cancels (a needle's conic is huge along
    # its short axis): floors of 256 ulp of the term sizes, from A = the largest |v_cov| entry of the gaussian and its
    # covariance scale S2 (largest variance): v_covars ~ A, v_scales ~ A max(s), v_quats ~ A S2 / |q|,
    # v_means ~ A S2 / z (through the Jacobian's derivative), v_viewmats ~ A S2 + |v_means| |mean|.
    with np.errstate(invalid="ignore", over="ignore"):
        A = np.nan_to_num(np.max([r["_vcov"] for r in res], 0), nan=0.0, posinf=0.0)
        c6 = res[0]["_cov"]
        S2 = np.nan_to_num(np.abs(c6[:, [0, 3, 5]]).max(-1), nan=0.0, posinf=0.0)
        pcz = np.einsum("cj,nj->cn", tr.inputs["viewmats"][:, 2, :3], tr.inputs["means"]) + tr.inputs["viewmats"][:, 2, 3][:, None]
        inv_z = np.nan_to_num(np.max(np.where(keep, 1.0 / np.abs(pcz), 0.0), 0), nan=0.0, posinf=0.0)
        qn = np.sqrt((rows["quats"].astype(np.float64) ** 2).sum(-1))
        sc = np.abs(rows["scales"].astype(np.float64))
        fl = 256.0 * ULP
        floors = dict(v_means=fl * A * S2 * inv_z, v_covars=fl * A, v_scales=fl * 3.0 * A[:, None] * sc.max(-1, keepdims=True),
                      v_quats=fl * A * S2 / np.where(qn > 0, qn, 1.0))
        m_abs = np.abs(np.nan_to_num(rows["means"].astype(np.float64), nan=0.0, posinf=0.0, neginf=0.0)).max(-1)
    seen = keep.any(0)  # a gaussian without a kept row gets exactly zero
    grads, betas = {}, {}
    for k in res[0]:
        if k.startswith("_"):
            continue
        base = res[0][k]
        if k == "v_viewmats_rows":
            flat = base.reshape(N, -1)
            bro = _row_beta(flat, [r[k].reshape(N, -1) for r in res[1:]], fish, ulps=32.0)
            vm_abs = np.abs(np.nan_to_num(res[0]["v_means"], nan=0.0)).max(-1)
            bro = bro + (fl * (A * S2 + vm_abs * m_abs))[:, None]
            grads[k] = base
            grads["v_viewmats"] = base.sum(0)
            betas["v_viewmats"] = (bro.sum(0) + 64.0 * ULP * np.abs(flat).sum(0)).reshape(C, 4, 4)
            continue
        base = np.where(seen.reshape((-1,) + (1,) * (base.ndim - 1)), base, 0.0)
        grads[k] = base
        f = floors.get(k, 0.0)
        b_ = _row_beta(base, [r[k] for r in res[1:]], fish, ulps=32.0) + (f if np.ndim(f) == 2 else np.asarray(f)[:, None])
        betas[k] = np.where(seen.reshape((-1,) + (1,) * (base.ndim - 1)), b_, 0.0)
    return grads, betas, cot32


def check_grads(rows, tr, got, ref, beta, what):
    """per-gaussian gradients [N, k] and v_viewmats [C, 4, 4] against the truth; a gaussian with an undecided row
    only needs finite gradients (its cotangents are zero).  Returns failure messages."""
    msgs = []
    und = ~tr.decided.all(0)
    for k, g in got.items():
        if g is None:
            continue
        g = np.asarray(g, np.float64)
        with np.errstate(invalid="ignore"):
            if k == "v_viewmats":
                bad = ~(np.abs(g - ref[k]) <= beta[k])
                if bad.any():
                    msgs.append(f"{what}: v_viewmats out of budget at {np.argwhere(bad)[:4].tolist()}: got "
                                f"{g[bad][:4].tolist()}, truth {ref[k][bad][:4].tolist()}, beta {beta[k][bad][:4].tolist()}")
                continue
            bad = (~(np.abs(g - ref[k]) <= beta[k])).any(-1) & ~und
            bad |= ~np.isfinite(g).all(-1)
        if bad.any():
            n = int(np.nonzero(bad)[0][0])
            msgs.append(f"{what}: {int(bad.sum())} gaussians with {k} out of budget, e.g. {describe(rows, tr, 0, n)}: "
                        f"got {g[n].tolist()}, truth {ref[k][n].tolist()}, beta {beta[k][n].tolist()}")
    return msgs


# ------------------------------------------------------------------------------------------------------------------
# reporting
def describe(rows, tr, c, n):
    return (f"row {n} (class {tr.cls[n]}, camera {c}, mean={rows['means'][n].tolist()}, quat={rows['quats'][n].tolist()}, "
            f"scale={rows['scales'][n].tolist()}, opacity={float(rows['opacities'][n])!r})")


def check_forward(rows, cfg, tr, radii, means2d, depths, conics, comps, what):
    """GPU / float32 forward outputs [C, N, *] against the truth on decided rows; returns failure messages."""
    msgs = []
    dec = tr.decided
    bad = dec & (radii != tr.radii).any(-1)
    if bad.any():
        idx = np.argwhere(bad)
        msgs.append(f"{what}: {len(idx)} decided rows with wrong radii, e.g. " + "; ".join(
            f"{describe(rows, tr, c, n)}: got {radii[c, n].tolist()}, truth {tr.radii[c, n].tolist()}" for c, n in idx[:3]))
    vis = dec & (tr.radii > 0).all(-1) & ~bad
    for name, got in (("means2d", means2d), ("depths", depths), ("conics", conics), ("compensations", comps)):
        if got is None:
            continue
        ref, beta = tr.values[name], tr.beta[name]
        with np.errstate(invalid="ignore"):
            err = np.abs(got.astype(np.float64) - ref)
            viol = ~(err <= beta)
        if viol.ndim == 3:
            viol = viol.any(-1)
        viol &= vis & np.isfinite(ref if ref.ndim == 2 else ref.sum(-1))
        if viol.any():
            c, n = np.argwhere(viol)[0]
            msgs.append(f"{what}: {int(viol.sum())} decided rows with {name} out of budget, e.g. {describe(rows, tr, c, n)}: "
                        f"got {got[c, n].tolist()}, truth {ref[c, n].tolist()}, beta {np.asarray(beta[c, n]).tolist()}")
    return msgs


def undecided_report(tr):
    """{class: (undecided rows / rows)} over all cameras"""
    out = {}
    for k in np.unique(tr.cls):
        sel = tr.cls == k
        out[str(k)] = float((~tr.decided[:, sel]).mean())
    return out


# ------------------------------------------------------------------------------------------------------------------
# the intersection: a 2D adversarial set and the pixel truth of tile coverage
def adversarial_2d(W2, H2, seed=7, n=400):
    """means2d [1, n, 2], conics [1, n, 3], opacities [1, n], depths [1, n], radii [1, n, 2] (float32 / int32) of
    hostile screen-space gaussians: near-singular conics (disc ~ 0), opacities just above 1/255 (t ~ 0), centres far
    outside, needles spanning more than 64 tiles."""
    rng = np.random.RandomState(seed)
    rows = []
    for i in range(n):
        kind = i % 5
        ang = rng.uniform(0, math.pi)
        l1 = 10.0 ** rng.uniform(-1, 2.5)  # sigma along the major axis, px
        an = 10.0 ** rng.uniform(0, 4) if kind in (0, 3) else 10.0 ** rng.uniform(0, 1)
        if kind == 0:  # needle: long axis up to ~ the canvas
            l1 = rng.uniform(0.2, 1.0) * max(W2, H2) / 3.0
        s1, s2 = l1, max(l1 / an, 0.05)
        cs, sn = math.cos(ang), math.sin(ang)
        cov = np.array([[cs * cs * s1 * s1 + sn * sn * s2 * s2, cs * sn * (s1 * s1 - s2 * s2)],
                        [cs * sn * (s1 * s1 - s2 * s2), sn * sn * s1 * s1 + cs * cs * s2 * s2]])
        cov += 0.3 * np.eye(2) * (kind != 3)  # kind 3: no blur, disc ~ 0 when the needle is thin
        con = np.linalg.inv(cov)
        op = ALPHA_TH * (1 + 10.0 ** rng.uniform(-6, -1)) if kind == 1 else rng.uniform(0.05, 1.0)
        if kind == 2:
            mx, my = rng.uniform(-3 * s1, W2 + 3 * s1), rng.uniform(-3 * s1, H2 + 3 * s1)
        else:
            mx, my = rng.uniform(-0.2 * W2, 1.2 * W2), rng.uniform(-0.2 * H2, 1.2 * H2)
        e = min(EXTEND, math.sqrt(2 * math.log(op / ALPHA_TH)))
        rx, ry = math.ceil(e * math.sqrt(cov[0, 0])), math.ceil(e * math.sqrt(cov[1, 1]))
        rows.append((mx, my, con[0, 0], con[0, 1], con[1, 1], op, rng.uniform(0.5, 50), rx, ry))
    a = np.array(rows)
    f = lambda x: np.ascontiguousarray(x.astype(np.float32)[None])  # noqa: E731
    return dict(means2d=f(a[:, 0:2]), conics=f(a[:, 2:5]), opacities=f(a[:, 5]), depths=f(a[:, 6]),
                radii=np.ascontiguousarray(a[None, :, 7:9].astype(np.int32)))


def required_tiles(means2d, conics, opacities, radii, W2, H2, ts=16, max_pixels=4096):
    """Per (image, gaussian) with positive radii and a positive-definite conic: the tiles holding a *decided* pixel of
    float64 alpha >= 1/255 (sigma <= t / 2 with t = min(2 log(255 op), 3.33^2), the region AccuTile and the radius
    AABB both enumerate), searched in the gaussian's float64 bounding box (subsampled to about `max_pixels` pixel
    centres).  A pixel is decided when |2 sigma - t| exceeds 64 ulp of (|terms| + t), widened by 1 / |disc| for
    near-singular conics.  Returns {(image, gaussian): set(tile ids)}."""
    I, N = means2d.shape[:2]
    tw = -(-W2 // ts)
    out = {}
    f8 = np.float64
    for i in range(I):
        for n in range(N):
            if not (radii[i, n] > 0).all():
                continue
            a, b, c = (f8(v) for v in conics[i, n])
            op = f8(opacities[i, n])
            det = a * c - b * b
            if not (a > 0 and c > 0 and det > 0 and np.isfinite(det) and op >= ALPHA_TH):
                continue
            t = min(2.0 * math.log(op / ALPHA_TH), EXTEND * EXTEND)
            mx, my = (f8(v) for v in means2d[i, n])
            xe, ye = math.sqrt(t * c / det), math.sqrt(t * a / det)
            x0, x1 = max(0, math.floor(mx - xe)), min(W2 - 1, math.ceil(mx + xe))
            y0, y1 = max(0, math.floor(my - ye)), min(H2 - 1, math.ceil(my + ye))
            if x1 < x0 or y1 < y0:
                continue
            step = max(1, math.ceil(math.sqrt((x1 - x0 + 1) * (y1 - y0 + 1) / max_pixels)))
            px = np.arange(x0, x1 + 1, step, dtype=f8)
            py = np.arange(y0, y1 + 1, step, dtype=f8)
            dx = px[None, :] + 0.5 - mx
            dy = py[:, None] + 0.5 - my
            s2 = a * dx * dx + c * dy * dy + 2 * b * dx * dy
            S = np.abs(a) * dx * dx + np.abs(c) * dy * dy + 2 * np.abs(b * dx * dy)
            widen = max(1.0, abs(a * c) / abs(det))
            inside = (s2 <= t) & (np.abs(s2 - t) > 64.0 * ULP * widen * (S + t))
            yy, xx = np.nonzero(inside)
            if len(yy):
                tiles = (py[yy].astype(np.int64) // ts) * tw + px[xx].astype(np.int64) // ts
                out[(i, n)] = set(np.unique(tiles).tolist())
    return out


def listed_tiles(isect_ids, flatten_ids, N, tile_bits):
    """{(image, gaussian): set(tiles)} from isect ids / flatten ids (dense layout, flatten id = image * N + gaussian)"""
    tiles = (np.asarray(isect_ids, np.int64) >> 32) & ((1 << tile_bits) - 1)
    fl = np.asarray(flatten_ids, np.int64)
    out = {}
    for f, t in zip(fl.tolist(), tiles.tolist()):
        out.setdefault((f // N, f % N), set()).add(t)
    return out


def missing_tiles(required, listed):
    """[(image, gaussian, missing tiles)] of the required tiles that are not listed"""
    miss = []
    for key, req in required.items():
        m = req - listed.get(key, set())
        if m:
            miss.append((key[0], key[1], sorted(m)[:5]))
    return miss
