"""Adversarial sweep for the SH colour evaluation of gsplat_b200/csrc/pergauss.cu and its float64 truth (no GPU needed).

N_ROWS Gaussians, every row tagged with its class, in a random order so that warps mix classes, seen and unseen rows:

* direction classes: bulk; exact +-x, +-y, +-z view directions (the cameras sit at the origin, so the view direction
  mean + R^T t is the mean bit for bit); directions 1e-7 to 1e-3 off an axis; |dir| from 0.02 to 1e4; large
  coefficients (|c| ~ 1e2 - 1e3) whose terms cancel to a colour near [0, 1];
* clamp classes: exact float32 ties of max(x + 0.5, 0) -- the trainer's initialisation sh0 = (rgb - 0.5) / C0 of black
  channels, in all three channels or only some -- and rows 1e-7 to 1e-2 of the terms on either side of the kink.

Six cameras at the origin look along +z, +x, -z, +y, -x and -y (signed permutation rotations, 116 degree field of view);
each of PAIRS is two orthogonal cameras whose views overlap, so that a row is seen by both, by one or by neither, and
every signed axis is the optical axis of one camera.  The standalone SH kernels also run under cameras moved off the
origin (OFFSET_CENTRES).

The truth is the oracle (oracle/gso.py) in float64 on the float32 inputs.  Budgets: every quantity is re-evaluated at
N_PERTURB seeded relative perturbations of the float32 inputs of 4 * 2^-24; its budget is 4x the largest deviation plus
ulps of the sum of the absolute values of its terms (sum_k TERM_k |c_k| for a colour, TERM_k bounding the terms of
Y_k).  A colour entry is *decided* when
|x + 0.5| exceeds its budget, or when it is an exact float32 tie by construction; at a tie the contract is float32's,
that of torch.clamp_min: the colour is 0 and the gradient passes.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import gso

f32, f64 = np.float32, np.float64
ULP = 2.0**-24
N_ROWS = 4113  # the last warp is partial
N_PERTURB = 6
SH_C0 = 0.28209479177387814
W = H = 64
FOCAL = 20.0  # half field of view atan(32 / 20) = 58 degrees: orthogonal cameras overlap around their diagonal

# degree x K: both load / store layouts (K * 3 % 4 == 0 for K = 4, 16), NB * 3 % 4 != 0 (degrees 0, 2, 4) and the
# trainer's warm-up (K = 16 with degree < 3, where v_sh beyond (degree + 1)^2 must be exactly 0)
GRID = [(d, K) for d in range(5) for K in sorted({(d + 1) ** 2, 16, 25}) if K >= (d + 1) ** 2]

# camera-space rows of the rotation: R maps the world axis the camera looks along to +z
_ROT = {
    "+z": [[1, 0, 0], [0, 1, 0], [0, 0, 1]],
    "+x": [[0, 0, -1], [0, 1, 0], [1, 0, 0]],
    "-z": [[-1, 0, 0], [0, 1, 0], [0, 0, -1]],
    "+y": [[1, 0, 0], [0, 0, -1], [0, 1, 0]],
    "-x": [[0, 0, 1], [0, 1, 0], [-1, 0, 0]],
    "-y": [[1, 0, 0], [0, 0, 1], [0, -1, 0]],
}
AXES = tuple(_ROT)
PAIRS = ((0, 1), (2, 3), (4, 5))
OFFSET_CENTRES = ((0.3, -0.2, 0.1), (-0.15, 0.25, -0.3))

CLASSES = ("bulk", "axis", "near_axis", "dist", "cancel", "tie", "kink")
N_CLASS = dict(axis=240, near_axis=300, dist=300, cancel=400, tie=400, kink=800)  # bulk fills the rest


def cameras(ids, centres=None):
    """viewmats [C, 4, 4], Ks [C, 3, 3] float32 of the cameras `ids`, at the origin or at `centres`"""
    vm = np.zeros((len(ids), 4, 4), f32)
    for i, c in enumerate(ids):
        R = np.array(_ROT[AXES[c]], f64)
        vm[i, :3, :3] = R
        vm[i, 3, 3] = 1
        if centres is not None:
            vm[i, :3, 3] = -R @ np.asarray(centres[i], f64)
    K = np.array([[FOCAL, 0, W / 2], [0, FOCAL, H / 2], [0, 0, 1]], f32)
    return vm, np.ascontiguousarray(np.broadcast_to(K, (len(ids), 3, 3)))


# per band, a bound of sum |term| of Y_k's float32 evaluation on the unit sphere (Y_6 = 0.946 z^2 - 0.315 cancels to
# nothing near z^2 = 1/3, while its rounding error stays that of 0.315)
TERM = (0.2821, 0.4886, 1.262, 3.0, 8.0)


def band_terms(deg, K=None):
    """[nb] (or [K], zero beyond nb): TERM of each coefficient's band"""
    nb = (deg + 1) ** 2
    t = np.array([TERM[int(math.isqrt(k))] for k in range(nb)])
    return t if K is None else np.concatenate([t, np.zeros(K - nb)])


def terms(deg, coeffs):
    """[N, D]: sum_k TERM_k |c_k|, the size of the terms a colour is summed from"""
    nb = (deg + 1) ** 2
    return np.einsum("k,nkd->nd", band_terms(deg), np.abs(coeffs[:, :nb].astype(f64)))


def basis(deg, means, viewmats):
    """float64 Y_k [..., C, N, NB] of the float32 inputs (the oracle on identity coefficients)"""
    nb = (deg + 1) ** 2
    eye = np.ascontiguousarray(np.broadcast_to(np.eye(nb), (means.shape[-2], nb, nb)))
    return gso.spherical_harmonics(deg, means.astype(f64), viewmats.astype(f64), eye)


def _unit(rng, n):
    v = rng.standard_normal((n, 3))
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def make_rows(deg, K, seed=20261017):
    """dict(cls [N], means [N, 3], quats, scales, opacities, coeffs [N, K, 3], tie [N, 3], side [N, 3]) -- tie marks the
    exact float32 ties, side the side of the kink a "kink" channel was put on (+-1, else 0).  The geometry depends on the
    seed only, the coefficients on (deg, K) too."""
    rng = np.random.RandomState(seed)
    counts = dict(N_CLASS, bulk=N_ROWS - sum(N_CLASS.values()))
    cls = np.concatenate([np.full(counts[c], c, dtype=object) for c in CLASSES])
    N = len(cls)
    u = _unit(rng, N)
    dist = np.exp(rng.uniform(math.log(0.5), math.log(20.0), N))
    ax = cls == "axis"
    a = rng.randint(0, 6, ax.sum())
    e = np.zeros((ax.sum(), 3))
    e[np.arange(ax.sum()), a % 3] = np.where(a < 3, 1.0, -1.0)
    u[ax] = e
    na = cls == "near_axis"
    a = rng.randint(0, 6, na.sum())
    e = np.zeros((na.sum(), 3))
    e[np.arange(na.sum()), a % 3] = np.where(a < 3, 1.0, -1.0)
    perp = _unit(rng, na.sum())
    perp -= (perp * e).sum(-1, keepdims=True) * e
    perp /= np.linalg.norm(perp, axis=-1, keepdims=True)
    eps = np.exp(rng.uniform(math.log(1e-7), math.log(1e-3), na.sum()))
    v = e + eps[:, None] * perp
    u[na] = v / np.linalg.norm(v, axis=-1, keepdims=True)
    dd = cls == "dist"
    dist[dd] = np.exp(rng.uniform(math.log(0.02), math.log(1e4), dd.sum()))
    means = (u * dist[:, None]).astype(f32)  # the axis rows have exactly one non-zero component
    scales = (0.03 * dist[:, None] * rng.uniform(0.5, 1.5, (N, 3))).astype(f32)
    quats = rng.standard_normal((N, 4))
    quats = (quats / np.linalg.norm(quats, axis=-1, keepdims=True)).astype(f32)
    opacities = np.full(N, 0.9, f32)
    perm = rng.permutation(N)
    geo = dict(cls=cls[perm], means=np.ascontiguousarray(means[perm]), quats=quats[perm], scales=scales[perm],
               opacities=opacities)
    geo["coeffs"], geo["tie"], geo["side"] = _coeffs(deg, K, geo["cls"], geo["means"], np.random.RandomState(seed + 101 * deg + K))
    return geo


def _coeffs(deg, K, cls, means, rng):
    N, nb = len(cls), (deg + 1) ** 2
    c = (rng.standard_normal((N, K, 3)) * 0.3).astype(f32)  # bands >= nb: read by nobody
    rgb = rng.uniform(0.05, 1.0, (N, 3)).astype(f32)
    tie, side = np.zeros((N, 3), bool), np.zeros((N, 3))
    t = np.flatnonzero(cls == "tie")
    pattern = np.array([[0, 0, 0], [255, 0, 0], [0, 255, 0], [0, 0, 255], [255, 255, 0], [0, 128, 255]], f32)
    pick = rng.randint(0, len(pattern), len(t))
    pick[: len(t) // 2] = 0  # half black-initialised
    rgb[t] = pattern[pick] / f32(255.0)
    tie[t] = pattern[pick] == 0
    c[:, 0, :] = (rgb - f32(0.5)) / SH_C0  # the trainer's initialisation, in float32
    c[t, 1:nb, :] = 0.0
    Y = basis(deg, means, np.eye(4, dtype=f32)[None])[0]  # [N, nb]: the view direction is the mean for every camera
    for name in ("kink", "cancel"):
        r = np.flatnonzero(cls == name)
        if name == "cancel" and deg > 0:
            mag = np.exp(rng.uniform(math.log(1e2), math.log(1e3), (len(r), nb - 1, 3)))
            c[r, 1:nb, :] = (mag * np.sign(rng.standard_normal(mag.shape))).astype(f32)
            target = rng.uniform(-0.8, 0.3, (len(r), 3))
        elif name == "cancel":
            c[r, 0, :] *= f32(256.0)  # degree 0: no higher band to cancel against, a large colour instead
            continue
        else:
            side[r] = np.where(rng.random_sample((len(r), 3)) < 0.5, -1.0, 1.0)
            delta = np.exp(rng.uniform(math.log(1e-7), math.log(1e-2), (len(r), 3)))
            c[r, 0, :] = f32(-0.5 / SH_C0)
            target = -0.5 + side[r] * delta * terms(deg, c[r])
        S = np.einsum("nk,nkd->nd", Y[r, 1:], c[r, 1:nb].astype(f64))
        c[r, 0, :] = ((target - S) / Y[r, :1]).astype(f32)
    return np.ascontiguousarray(c), tie, side


def _perturb(a, rng):
    return a.astype(f64) * (1.0 + 4.0 * ULP * rng.uniform(-1.0, 1.0, a.shape))


class Truth:
    """float64 colours x = SH (before the + 0.5 and the clamp) of one (degree, rows, cameras) setting, their budgets and
    decisions.  masks [..., C, N] bool (the rows a camera sees; all True for the standalone kernels)."""

    def __init__(self, deg, rows, viewmats, masks, coeffs=None, means=None, seed=7):
        self.deg, self.nb = deg, (deg + 1) ** 2
        self.means = rows["means"] if means is None else means
        self.coeffs = rows["coeffs"] if coeffs is None else coeffs
        self.vm, self.masks = viewmats, masks
        self.x = gso.spherical_harmonics(deg, self.means.astype(f64), viewmats.astype(f64), self.coeffs.astype(f64), masks)
        rng = np.random.RandomState(seed)
        spread = np.zeros_like(self.x)
        for _ in range(N_PERTURB):
            xp = gso.spherical_harmonics(deg, _perturb(self.means, rng), _perturb(viewmats, rng), _perturb(self.coeffs, rng), masks)
            spread = np.maximum(spread, np.abs(xp - self.x))
        self.terms = terms(deg, self.coeffs)
        self.budget = 4.0 * spread + (self.nb + 4) * ULP * self.terms
        D = self.x.shape[-1]
        tie = rows["tie"] if D == 3 and "tie" in rows else np.zeros((self.means.shape[-2], D), bool)
        self.tie = np.broadcast_to(tie, self.x.shape) & masks[..., None]
        self.decided = (np.abs(self.x + 0.5) > self.budget) | self.tie
        self.colour = np.where(self.tie, 0.0, np.maximum(self.x + 0.5, 0.0))
        self.passes = self.tie | (self.x + 0.5 >= 0)  # where the clamp passes the gradient

    def row_decided(self):
        """[N, D]: every camera that sees the row decides channel d (what v_sh[n, :, d] depends on)"""
        return (self.decided | ~self.masks[..., None]).reshape((-1,) + self.x.shape[-2:]).all(0)

    def grads(self, cot, clamp=True, seed=8):
        """float64 (v_coeffs, v_means) of sum(cot * colour) (clamp=True) or sum(cot * x), with their budgets"""
        m = self.masks[..., None]
        vcol = cot.astype(f64) * m * (self.passes if clamp else 1.0)
        ref = gso.spherical_harmonics_bwd(self.deg, self.means.astype(f64), self.vm.astype(f64), self.coeffs.astype(f64),
                                          self.masks, vcol)
        rng = np.random.RandomState(seed)
        spread = [np.zeros_like(ref[0]), np.zeros_like(ref[1])]
        for _ in range(N_PERTURB):
            vp = _perturb(cot, rng) * m * (self.passes if clamp else 1.0)
            gp = gso.spherical_harmonics_bwd(self.deg, _perturb(self.means, rng), _perturb(self.vm, rng),
                                             _perturb(self.coeffs, rng), self.masks, vp)
            spread = [np.maximum(s, np.abs(g - r)) for s, g, r in zip(spread, gp, ref)]
        N, D = self.x.shape[-2:]
        t_sh = band_terms(self.deg)[:, None] * np.abs(vcol).reshape(-1, N, D).sum(0)[:, None, :]
        t_m = dir_grad_terms(self.deg, self.means, self.vm, self.coeffs, vcol).sum(-2)
        b_sh = np.zeros(self.coeffs.shape)
        b_sh[:, : self.nb] = 4.0 * spread[0][:, : self.nb] + (self.nb + 8) * ULP * t_sh
        b_m = 4.0 * spread[1] + (self.nb + 16) * ULP * t_m[..., None]
        return ref, (b_sh, b_m)


def visibility(rows, viewmats, Ks):
    """[C, N] rows the float32 projection keeps (the kernels' radii agree with it bit for bit)"""
    radii = gso.fully_fused_projection(rows["means"], None, rows["quats"], rows["scales"], viewmats, Ks, W, H, 0.3, 0.01,
                                       1e10, 0.0, False, "pinhole", rows["opacities"])[0]
    return (radii > 0).all(-1)


def dir_grad_terms(deg, means, viewmats, coeffs, vcol):
    """[..., C, N]: the size of the terms of one image's view-direction gradient sum_k g_k dY_k/du (I - u u^T) / |dir|,
    g_k = sum_d c_kd vcol_d; dY_k/du of band l is bounded by 2 l^2 on the sphere"""
    nb = (deg + 1) ** 2
    band = np.floor(np.sqrt(np.arange(nb))).astype(f64)
    g = np.einsum("nkd,...nd->...nk", np.abs(coeffs[:, :nb].astype(f64)), np.abs(vcol))
    dirs = means[..., None, :, :].astype(f64) + np.einsum(
        "...ji,...j->...i", viewmats[..., :3, :3].astype(f64), viewmats[..., :3, 3].astype(f64))[..., None, :]
    return (g * 2 * band**2).sum(-1) / np.linalg.norm(dirs, axis=-1)


def undecided_report(tr, cls):
    """{class: (visible entries, undecided entries)} over the entries (camera, row, channel) the cameras see"""
    vis = np.broadcast_to(tr.masks[..., None], tr.x.shape)
    und = vis & ~tr.decided
    out = {}
    for c in CLASSES:
        sel = np.broadcast_to((cls == c)[:, None], tr.x.shape[-2:])
        out[c] = (int((vis & sel).sum()), int((und & sel).sum()))
    return out


def check(got, ref, budget, sel, what):
    """messages for entries of `sel` whose |got - ref| exceeds the budget"""
    got = np.asarray(got, f64)
    bad = sel & ~(np.abs(got - ref) <= budget)
    if not bad.any():
        return []
    i = tuple(np.argwhere(bad)[0])
    return [f"{what}: {int(bad.sum())} of {int(sel.sum())} entries off, first {i}: got {got[i]!r} truth {ref[i]!r} "
            f"budget {budget[i]:.3e}"]
