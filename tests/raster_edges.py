"""Adversarial single-gaussian sweep for the compositing kernels and its float64 truth (no GPU needed).

Every gaussian is rendered ALONE in its own 45 x 37 image (3 x 3 tiles, partial in both directions), and every tile of
that image lists it, so the compositing kernel's block-level cull plus its exact per-pixel test alone decide which
pixels it touches.  The cull must be conservative: it may never skip a (pixel block, gaussian) pair in which some pixel
reaches alpha >= 1/255.  The sweep aims at the inputs where float32 extents go wrong: needles (conic anisotropy up to
1e6), near-isotropic conics with a tiny off-diagonal, sub-pixel gaussians, opacities just above 1/255 or at / above the
0.99 clamp, centres far outside the image, centres placed so that the alpha = 1/255 boundary's extreme point along x, y
or an ellipse axis falls just beyond the nearest pixel of a warp's 8 x 4 pixel block, and a handful of degenerate rows
(non-positive-definite, inf / NaN conics, opacity below 1/255) that take the kernels' "never cull" or "always cull"
branches.

The truth is computed per pixel in float64 from the float32 inputs:
    sigma = 0.5 (a dx^2 + c dy^2) + b dx dy,  alpha = min(0.99, op exp(-sigma)),
    kept if sigma >= 0 and alpha >= 1/255 (else 0),  colour = alpha c + (1 - alpha) bg.
A float32 evaluation of sigma errs by a few units of 2^-24 of the sum of the absolute values of its terms,
S = 0.5 (|a| dx^2 + |c| dy^2) + |b dx dy|; the kernels evaluate the exponent with the conic pre-scaled by log2(e) and
ex2.approx.  The per-pixel budget allows 16 ulp of S for sigma (`dsig`) and 32 ulp for the exponential and the product
with the opacity, so that the relative error of a float32 alpha is at most beta = expm1(dsig + 32 ulp).  A pixel is
*decided* when no discrete decision lies within that budget of flipping: the sign of sigma, the alpha >= 1/255 threshold
and the 0.99 clamp (the last one only matters for the gradient).
"""
from __future__ import annotations

import itertools
import math

import numpy as np

W, H = 45, 37
TW, TH = 3, 3
ULP = 2.0**-24
ALPHA_TH = float(np.float32(1.0 / 255.0))
MAX_ALPHA = float(np.float32(0.99))

L1_GRID = tuple(10.0**e for e in np.arange(-7.0, 2.01, 0.5))  # larger conic eigenvalue: 1e-7 .. 1e2
ANISO = (1.0, 1.0 + 1e-6, 10.0, 1e2, 1e3, 1e4, 1e6)
ANGLES = ("0", "pi/4", "1e-3", "random")
OPACITIES = tuple(float(np.float32(ALPHA_TH * (1.0 + e))) for e in (1e-5, 1e-3, 1e-1)) + (0.5, 0.99, 1.0, 1.5)
# where the centre goes: uniformly over the image (sub-pixel), far outside it, or so that the extreme point of the
# alpha = 1/255 boundary along x / y / the major / the minor conic axis / a random direction lands next to a pixel
PLACEMENTS = ("inside", "far", "x", "y", "u", "v", "dir")

# degenerate rows: (a, b, c, opacity)
_INF, _NAN = float("inf"), float("nan")
DEGENERATE = (
    (0.1, 0.2, 0.1, 0.5),  # det < 0 (saddle)
    (0.1, 0.3, 1.0, 0.99),  # det < 0
    (0.1, 0.1, 0.1, 0.5),  # det == 0 exactly
    (-0.1, 0.0, 0.1, 0.5),  # a < 0
    (0.0, 0.0, 0.1, 1.0),  # a == 0
    (0.1, 0.0, -0.1, 0.5),  # c < 0
    (-0.1, 0.0, -0.1, 0.99),  # negative definite: sigma <= 0 everywhere
    (0.0, 0.0, 0.0, 0.5),  # zero conic
    (_INF, 0.0, 0.1, 0.5),
    (0.1, _INF, 0.1, 0.5),
    (0.1, -_INF, 0.1, 0.5),
    (0.1, 0.0, _INF, 0.99),
    (_INF, _INF, _INF, 0.5),
    (_NAN, 0.0, 0.1, 0.5),
    (0.1, _NAN, 0.1, 0.5),
    (0.1, 0.0, _NAN, 0.5),
    (0.05, 0.01, 0.05, ALPHA_TH * (1.0 - 1e-5)),  # opacity just below 1/255
    (0.05, 0.01, 0.05, 1e-3),
    (0.05, 0.01, 0.05, 0.0),
    (0.05, 0.01, 0.05, -0.5),
    (0.05, 0.01, 0.05, _NAN),
)


def _conic(l1, l2, angle, rng):
    if angle == "pi/4":
        cs = sn = math.sqrt(0.5)
    else:
        th = {"0": 0.0, "1e-3": 1e-3}.get(angle)
        th = rng.uniform(0, math.pi) if th is None else th
        cs, sn = math.cos(th), math.sin(th)
    # Q = R diag(l1, l2) R^T
    return l1 * cs * cs + l2 * sn * sn, (l1 - l2) * sn * cs, l1 * sn * sn + l2 * cs * cs


def _place(kind, a, b, c, op, rng):
    """Centre for one gaussian (float64; rounded to float32 by the caller)."""
    inside = (rng.uniform(-2.0, W + 2.0), rng.uniform(-2.0, H + 2.0))
    if kind == "inside":
        return inside
    if kind == "far":
        return rng.uniform(-500.0, W + 500.0), rng.uniform(-500.0, H + 500.0)
    Q = np.array([[a, b], [b, c]], np.float64)
    if not (a > 0 and c > 0 and a * c - b * b > 0):
        return inside
    L = math.log(255.0 * op)  # boundary: sigma = L
    if kind == "x":
        n = np.array([rng.choice((-1.0, 1.0)), 0.0])
    elif kind == "y":
        n = np.array([0.0, rng.choice((-1.0, 1.0))])
    elif kind in ("u", "v"):
        w, V = np.linalg.eigh(Q)  # ascending: column 1 = larger eigenvalue (u, the short axis)
        n = V[:, 1 if kind == "u" else 0] * rng.choice((-1.0, 1.0))
    else:
        t = rng.uniform(0, 2 * math.pi)
        n = np.array([math.cos(t), math.sin(t)])
    Qn = np.linalg.solve(Q, n)
    d = math.sqrt(2.0 * L / float(n @ Qn)) * Qn  # point of the boundary that is extreme along n
    if not np.isfinite(d).all() or np.abs(d).max() > 700.0:
        return inside
    # the pixel of its warp block (8 x 4) that is nearest to the centre along n: that is where a too tight cull bites
    col = 0 if n[0] > 1e-9 else (7 if n[0] < -1e-9 else rng.randint(8))
    row = 0 if n[1] > 1e-9 else (3 if n[1] < -1e-9 else rng.randint(4))
    px = rng.choice(np.arange(col, W, 8)) + 0.5
    py = rng.choice(np.arange(row, H, 4)) + 0.5
    s = rng.uniform(0.993, 0.9995) if rng.rand() < 0.85 else rng.uniform(1.0005, 1.01)
    return px - s * d[0], py - s * d[1]


def make_sweep(n=1536, seed=20261015, channels=(3, 5)):
    """Seeded sweep of `n` gaussians (plus the degenerate rows), one per image.

    Returns a dict with the kernel inputs (float32 dense layout [I, 1, *]) and per-gaussian labels: `aniso`, `l1`,
    `placement` (NaN / "degenerate" for the degenerate rows), `colors{D}` [I, 1, D] and `bg{D}` [I, D] per channel
    count, `isect_offsets` [I, 3, 3] = arange(I * 9) and `flatten_ids` = repeat(arange(I), 9)."""
    rng = np.random.RandomState(seed)
    grid = list(itertools.product(L1_GRID, ANISO, ANGLES, OPACITIES, PLACEMENTS))
    pick = rng.choice(len(grid), size=n - len(DEGENERATE), replace=False)
    rows, aniso, l1s, place = [], [], [], []
    for i in pick:
        l1, k, ang, op, kind = grid[i]
        a, b, c = (float(np.float32(v)) for v in _conic(l1, l1 / k, ang, rng))
        mx, my = _place(kind, a, b, c, op, rng)
        rows.append((mx, my, a, b, c, op))
        aniso.append(k), l1s.append(l1), place.append(kind)
    for a, b, c, op in DEGENERATE:
        rows.append((rng.uniform(0, W), rng.uniform(0, H), a, b, c, op))
        aniso.append(np.nan), l1s.append(np.nan), place.append("degenerate")
    r = np.array(rows, np.float64)
    I = r.shape[0]
    with np.errstate(over="ignore", invalid="ignore"):
        r32 = r.astype(np.float32)
    out = dict(
        means2d=np.ascontiguousarray(r32[:, None, 0:2]),
        conics=np.ascontiguousarray(r32[:, None, 2:5]),
        opacities=np.ascontiguousarray(r32[:, None, 5]),
        isect_offsets=np.arange(I * TH * TW, dtype=np.int32).reshape(I, TH, TW),
        flatten_ids=np.repeat(np.arange(I, dtype=np.int32), TH * TW),
        aniso=np.array(aniso), l1=np.array(l1s), placement=np.array(place),
    )
    for D in channels:
        out[f"colors{D}"] = rng.random_sample((I, 1, D)).astype(np.float32)
        out[f"bg{D}"] = rng.random_sample((I, D)).astype(np.float32)
    return out


def truth(sw):
    """float64 per-pixel truth and float32 error budget of the sweep, all [I, H, W]:
    alpha (kept alpha, 0 where rejected), alpha_c (min(0.99, op exp(-sigma)) before the threshold), beta (bound on the
    relative error of a float32 alpha), decided (no discrete decision within the budget of flipping)."""
    f8 = np.float64
    m = sw["means2d"][:, 0].astype(f8)
    a, b, c = (sw["conics"][:, 0, k].astype(f8)[:, None, None] for k in range(3))
    op = sw["opacities"][:, 0].astype(f8)[:, None, None]
    dx = m[:, 0, None, None] - (np.arange(W, dtype=f8) + 0.5)[None, None, :]
    dy = m[:, 1, None, None] - (np.arange(H, dtype=f8) + 0.5)[None, :, None]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        sigma = 0.5 * (a * dx * dx + c * dy * dy) + b * dx * dy
        S = 0.5 * (np.abs(a) * dx * dx + np.abs(c) * dy * dy) + np.abs(b * dx * dy)
        dsig = 16.0 * ULP * S
        dl = dsig + 32.0 * ULP  # budget of log(alpha): sigma, ex2.approx, op * vis
        lx = np.log(op) - sigma  # log of op exp(-sigma)
        alpha_c = np.minimum(MAX_ALPHA, op * np.exp(-sigma))
        finite = np.isfinite(sigma) & np.isfinite(S) & (op > 0)
        keep = finite & (sigma >= 0) & (alpha_c >= ALPHA_TH)
        alpha = np.where(keep, alpha_c, 0.0)
        may_pass = finite & (sigma >= -dsig)  # pixels whose sign test can come out positive
        und = finite & (np.abs(sigma) <= dsig) & (S > 0)
        und |= may_pass & (np.abs(lx - math.log(ALPHA_TH)) <= dl)
        und |= may_pass & (np.abs(lx - math.log(MAX_ALPHA)) <= dl)
        beta = np.where(finite, np.expm1(np.minimum(dl, 700.0)), 0.0)
        nan_alpha = np.isnan(op * np.exp(-sigma))
    alpha_c = np.where(finite, np.nan_to_num(alpha_c, nan=0.0), 0.0)
    return dict(alpha=alpha, alpha_c=alpha_c, beta=beta, decided=~und, nan_alpha=nan_alpha)


def colour_truth(alpha, colors, bg):
    """[I, H, W, D] colour of one gaussian over a background."""
    al = alpha[..., None]
    return al * colors.astype(np.float64)[:, None, :, :] + (1.0 - al) * bg.astype(np.float64)[:, None, None, :]


def describe(sw, i, y=None, x=None):
    a, b, c = sw["conics"][i, 0]
    s = (f"gaussian {i} (conic a={a!r} b={b!r} c={c!r}, opacity={sw['opacities'][i, 0]!r}, "
         f"centre={tuple(sw['means2d'][i, 0].tolist())}, anisotropy={sw['aniso'][i]:g}, placement={sw['placement'][i]})")
    return s if y is None else s + f" at pixel (x={x}, y={y})"


def check_render(sw, tr, rc, ra, D, atol=1e-5, what="render", skip=None):
    """Checks a float32 rendering of the sweep (rc [I, H, W, D], ra [I, H, W, 1]) against the truth.

    Decided pixels: alpha within beta * alpha + atol, colour within beta * alpha * (|c| + |bg|) + atol; a pixel whose
    truth alpha is positive but whose rendered alpha is exactly 0 is reported as a dropped pair.  Undecided pixels:
    alpha is 0 or within beta of the unthresholded value.  Returns a list of failure messages (empty = pass)."""
    col, bg = sw[f"colors{D}"], sw[f"bg{D}"]
    ra = np.asarray(ra, np.float64)[..., 0]
    rc = np.asarray(rc, np.float64)
    al, dec, beta = tr["alpha"], tr["decided"], tr["beta"]
    if skip is not None:
        dec = dec & ~skip
    msgs = []
    dropped = dec & (al > 0) & (ra == 0)
    if dropped.any():
        idx = np.argwhere(dropped)
        msgs.append(f"{what}: {len(idx)} dropped pairs in {len(np.unique(idx[:, 0]))} gaussians, e.g. "
                    + "; ".join(describe(sw, i, y, x) + f" truth alpha {al[i, y, x]:.6g}" for i, y, x in idx[:3]))
    bad_a = dec & (np.abs(ra - al) > beta * al + atol)
    ref_c = colour_truth(al, col, bg)
    tol_c = (beta * al)[..., None] * (np.abs(col).max(-1)[:, :, None, None] + np.abs(bg)[:, None, None, :]) + atol
    bad_c = dec & (np.abs(rc - ref_c) > tol_c).any(-1)
    for bad, name, got, ref in ((bad_a, "alpha", ra, al), (bad_c, "colour", rc[..., 0], ref_c[..., 0])):
        if bad.any():
            i, y, x = np.argwhere(bad)[0]
            msgs.append(f"{what}: {int(bad.sum())} decided pixels with a wrong {name}, e.g. {describe(sw, i, y, x)}: "
                        f"got {got[i, y, x]:.8g}, truth {ref[i, y, x]:.8g} (beta {beta[i, y, x]:.3g})")
    und = ~tr["decided"] if skip is None else ~tr["decided"] & ~skip
    ac = tr["alpha_c"]
    bad_u = und & (ra != 0) & (np.abs(ra - ac) > beta * ac + atol)
    if bad_u.any():
        i, y, x = np.argwhere(bad_u)[0]
        msgs.append(f"{what}: {int(bad_u.sum())} undecided pixels neither 0 nor within beta, e.g. {describe(sw, i, y, x)}: "
                    f"got {ra[i, y, x]:.8g}, unthresholded truth {ac[i, y, x]:.8g}")
    return msgs


def undecided_report(sw, tr):
    """Per anisotropy class (and the degenerate rows): (undecided pixels / pixels that are touched or undecided,
    gaussians with an undecided pixel / gaussians).  A pixel is touched when its truth alpha is positive."""
    und = ~tr["decided"]
    touched = tr["alpha"] > 0
    out = {}
    keys = [k for k in ANISO] + ["degenerate"]
    for k in keys:
        sel = np.isnan(sw["aniso"]) if k == "degenerate" else sw["aniso"] == k
        if not sel.any():
            continue
        u, t = und[sel], touched[sel]
        out[k] = (float(u.sum() / max((u | t).sum(), 1)), float(u.any(axis=(1, 2)).mean()))
    return out
