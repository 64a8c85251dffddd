"""Adversarial sweep for the 3DGUT compositing kernels (eval3d_fwd_kernel, eval3d_bwd_kernel, eval3d_finish_kernel of
gsplat_b200/csrc/ut.cu) and for the pixel rays of cam_unproject (camera.cuh), with their float64 truth (no GPU needed).

Compositing images are 45 x 37 (3 x 3 tiles, partial in both directions), one per camera of one call, each with its own
K and view matrix (perfect pinhole), and every tile of an image lists every gaussian of that image in depth order, so
no projection cull hides anything.  Each gaussian belongs to one image.  It is placed relative to the float64 ray of a
chosen pixel: at a distance t along it and a distance lam across it, where dist = |g x a|^2 = lam^2 |g x M e| exactly,
so o * resp at that pixel is whatever the class asks.  Classes (CLASSES): o * resp near 1/255 ("alpha") and near 0.99
("clamp", where the backward takes the branch o * resp <= 0.99); hit_t near 0 ("hit": gaussians straddling the camera
plane or containing the camera); |a| from 1e2 to 1e5 where c = g x a cancels ("cancel": needles, far and tiny
gaussians); stacks whose next_T lands near 1e-4 at a pixel ("stop"); stacks that leave T_final near 1e-4 to 1e-3, where
the backward's T_final = 1 - render_alphas keeps a relative precision of about 2^-24 / T ("saturated"); opacities above
1, unnormalised quaternions, partial-tile pixels and rotated poses ("edges"); "bulk"; and rows the projection would cull
("degenerate": a zero scale, a scale below 1/FLT_MAX, a zero quaternion, non-finite means, which make no contribution,
and an infinite scale, which is a cylinder and does).

Exact ties ("tie"): K = (64, 64, 22.5, 18.5) with the identity pose sends pixel (22, 18)'s ray exactly along (0, 0, 1)
from the origin, so an identity-quaternion gaussian on the axis has c == 0, resp == 1 and alpha == o in float32 as in
float64: o == float32(1/255) and its predecessor; o == 0.99f and its successor; the opacities of surfel_edges'
STOP_OPACITIES, with which next_T == float32(1e-4) exactly at the fifth gaussian; and means at z = 0 off the axis
(hit_t == -0, kept) and z = +-2^-20.  The CPU tests check these ties by an exact float32 emulation of eval_hit (ut.cu is
built with -fmad=false).

Truth: float64 on the float32 inputs, vectorised over (image, pixel, list slot); the thresholds are the float32 values
the kernels compare with; a NaN hit_t or response makes no contribution, nor does a gaussian with a scale whose float32
reciprocal overflows (0 or below 1/FLT_MAX), whose M the kernel cannot form.  Budgets: every quantity is re-evaluated N_PERTURB
times with the float32 inputs (gaussians, colours, backgrounds, view matrices, Ks) perturbed by seeded relative amounts
up to 4 * 2^-24, and with the kernel's own rounding injected at its bound where it does not scale with the inputs:
a = M (o - mu) by 4 ulp of sum |M| |o - mu|, c = g x a by 4 ulp of |g| |a| per component, hit_t by 4 ulp of
sum |g_i a_i|, and the response by (4 + dist / 2) ulp relative (ex2.approx, and the rounding of its argument scaled
by dist).  Each budget is 4x the largest deviation, plus: for next_T, 2 ulp per product taken; for colours and alphas,
2 (L + 2) ulp of the sum of the absolute terms (L the list length); for gradients, K_GRAD ulp of the sum over pixels of
|that pixel's share| (autograd on per-pixel copies of the leaves; K_GRAD bounds the float32 chain of one share and the
butterfly and atomic sums over a 45 x 37 image), plus 2^-23 / T_final of each pixel's share (the backward divides its way
back from T_final = 1 - render_alphas).  A pair is decided when each of its decisions (1/255, 0.99, hit_t >= 0, and for a
pair that composites next_T <= 1e-4) clears its budget, or is an exact tie; a pixel when every pair it reaches is; a
gaussian when every pixel it reaches is.  Decisions are frozen at the central evaluation in the perturbed ones.

Pixel rays (lens_cases): one gaussian centred on the camera, listed on every tile, has alpha == o exactly on every ray
that exists and composites nothing elsewhere, so render_alphas shows the kernel's per-pixel validity.  The truth replays
the kernels' Newton rule in float64 (oracle.ut.Camera.unproject(rule="reference"), oracle.ut.FThetaCamera); a pixel is
decided when each comparison of its rule clears its budget (4x the spread under perturbed K and lens coefficients, plus
the float32 rounding of what it compares).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import ut as U
from tests.surfel_edges import STOP_OPACITIES

f64 = torch.float64
f32 = np.float32
ULP = 2.0**-24
N_PERTURB = 6
K_GRAD = 64
IW, IH = 45, 37
TW, TH = 3, 3
P = IW * IH
CHANNELS = (1, 2, 3, 4, 5, 8, 16, 32)


def F32(v):
    return float(f32(v))


ALPHA_TH = F32(f32(1.0) / f32(255.0))
MAX_ALPHA = F32(0.99)
T_TH = F32(1e-4)
CLASSES = ("alpha", "clamp", "hit", "cancel", "stop", "saturated", "edges", "bulk", "degenerate", "tie")
# undecided share of the pixels and of the gaussians allowed per class: "alpha" places half its gaussians within
# 1e-5 relative of 1/255 at one pixel, below its budget on purpose; one undecided pixel of a "bulk" stack leaves the
# whole stack out of the gradient check
UNDECIDED_MAX = dict(alpha=1e-3, clamp=0.0, hit=0.0, cancel=0.0, stop=0.0, saturated=0.0, edges=0.0, bulk=1e-3,
                     degenerate=0.0, tie=0.0)
G_UNDECIDED_MAX = dict(alpha=0.5, clamp=0.0, hit=0.0, cancel=0.0, stop=0.0, saturated=0.0, edges=0.0, bulk=0.15,
                       degenerate=0.0, tie=0.0)
TIE_K = (64.0, 64.0, 22.5, 18.5)
TIE_PIX = 18 * IW + 22


def _rot(axis, angle):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K


def _qrot(q):
    q = np.asarray(q, np.float64)
    return U.quat_to_rotmat(torch.tensor(q)).numpy()


class Sweep:
    """The images of the compositing sweep: per image its class, K, view matrix and gaussians (mean, quat, scale,
    opacity) in list order; ``ties`` marks the (image, pixel, slot) pairs decided exactly."""

    def __init__(self, seed=20261019):
        self.rng = np.random.RandomState(seed)
        self.images = []

    def image(self, cls, K=None, vm=None):
        rng = self.rng
        if K is None:
            fx = rng.uniform(40, 70)
            K = (fx, fx * rng.uniform(0.9, 1.1), rng.uniform(18, 27), rng.uniform(14, 23))
        if vm is None:
            vm = np.eye(4)
        self.images.append(dict(cls=cls, K=np.array([F32(k) for k in K]), vm=np.asarray(vm, np.float64).astype(f32),
                                gs=[], ties=[], stop_tie=None))
        return len(self.images) - 1

    def ray(self, c, px, py):
        im = self.images[c]
        fx, fy, cx, cy = im["K"]
        vm = im["vm"].astype(np.float64)
        d = np.array([(px + 0.5 - cx) / fx, (py + 0.5 - cy) / fy, 1.0])
        d /= np.linalg.norm(d)
        R, t = vm[:3, :3], vm[:3, 3]
        return -R.T @ t, R.T @ d

    def add(self, c, mean, quat, scale, o):
        self.images[c]["gs"].append((np.asarray(mean, np.float64).astype(f32), np.asarray(quat, np.float64).astype(f32),
                                     np.asarray(scale, np.float64).astype(f32), f32(o)))

    def place(self, c, px, py, t, quat, scale, o, dist):
        """a gaussian at distance t along pixel (px, py)'s ray and across it so that dist = |g x a|^2 there"""
        ro, rd = self.ray(c, px, py)
        e = np.cross(rd, self.rng.standard_normal(3))
        e /= np.linalg.norm(e)
        M = _qrot(quat).T / np.asarray(scale, np.float64)[:, None]
        b = M @ rd
        g = b / np.linalg.norm(b)
        lam = math.sqrt(max(dist, 0.0)) / np.linalg.norm(np.cross(g, M @ e))
        self.add(c, ro + t * rd + lam * e, quat, scale, o)

    def quat(self):
        q = self.rng.standard_normal(4)
        return q / np.linalg.norm(q)

    def pixel(self):
        return self.rng.randint(0, IW), self.rng.randint(0, IH)


def _float32_stop():
    """(slot of the stop, next_T) of STOP_OPACITIES evaluated like the kernel (alpha == o on the axis)"""
    T = f32(1.0)
    for k, o in enumerate(STOP_OPACITIES):
        nxt = f32(T * f32(f32(1.0) - f32(min(f32(MAX_ALPHA), f32(o)))))
        if nxt <= f32(T_TH):
            return k, nxt
        T = nxt
    return None, T


def make_sweep(seed=20261019):
    sw = Sweep(seed)
    rng = sw.rng
    deltas = (1e-2, -1e-2, 1e-3, -1e-3, 1e-4, -1e-4, 3e-5, -3e-5, 1e-5, -1e-5, 1e-6, -1e-7)
    for d in deltas:
        c = sw.image("alpha")
        o = rng.uniform(0.2, 1.0)
        sw.place(c, *sw.pixel(), rng.uniform(1.5, 6), sw.quat(), rng.uniform(0.05, 0.3, 3), o,
                 -2 * math.log(ALPHA_TH * (1 + d) / o))
    for d in deltas[:10]:
        c = sw.image("clamp")
        o = rng.uniform(1.0, 1.5)
        sw.place(c, *sw.pixel(), rng.uniform(1.5, 6), sw.quat(), rng.uniform(0.1, 0.4, 3), o,
                 -2 * math.log(MAX_ALPHA * (1 + d) / o))
    for k in range(8):  # straddling the camera plane (k even) or containing the camera (k odd)
        c = sw.image("hit")
        if k % 2 == 0:
            mean = (rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), rng.uniform(-0.05, 0.05))
            scale = rng.uniform(0.2, 0.6, 3)
        else:
            mean = rng.uniform(-0.1, 0.1, 3)
            scale = rng.uniform(0.5, 2.0, 3)
        sw.add(c, mean, sw.quat(), scale, rng.uniform(0.3, 0.9))
    for k in range(9):  # |a| = t / s from 1e2 to 1e5
        c = sw.image("cancel")
        if k % 3 == 0:  # needle along a random axis
            t, scale = rng.uniform(2, 10), np.array([1e-4, 1e-4, 0.5])[rng.permutation(3)]
        elif k % 3 == 1:  # far
            t = rng.uniform(1e3, 1e4)
            scale = t * rng.uniform(2e-3, 1e-2, 3)
        else:  # tiny
            t, scale = rng.uniform(1, 5), rng.uniform(5e-5, 2e-4, 3)
        sw.place(c, *sw.pixel(), t, sw.quat(), scale, rng.uniform(0.5, 0.95), rng.uniform(0, 3))
    for k, target in enumerate((1e-4 * (1 + d) for d in (1e-2, -1e-2, 1e-3, -1e-3, 3e-4, -3e-4))):
        _stack(sw, "stop", target)
    for target in (1.5e-4, 2.5e-4, 4e-4, 6e-4, 8e-4, 1e-3):
        _stack(sw, "saturated", target)
    for k in range(8):
        vm = np.eye(4)
        if k % 2 == 1:
            vm[:3, :3], vm[:3, 3] = _rot(rng.standard_normal(3), rng.uniform(0.1, 0.5)), rng.uniform(-0.5, 0.5, 3)
        c = sw.image("edges", vm=vm)
        o = (1.5, 3.0, 20.0, 1.2, 2.0, 1.0, 0.7, 5.0)[k]
        q = sw.quat() * (1e-3, 1e3, 1.0, 7.5, 1e-2, 1.0, 40.0, 1.0)[k]
        px, py = (rng.randint(32, IW), rng.randint(32, IH)) if k % 3 != 2 else sw.pixel()
        sw.place(c, px, py, rng.uniform(1.5, 6), q, rng.uniform(0.05, 0.4, 3), o, rng.uniform(0, 4))
    for k in range(12):
        c = sw.image("bulk")
        for t in sorted(rng.uniform(1, 10, rng.randint(1, 5))):
            sw.place(c, *sw.pixel(), t, sw.quat(), rng.uniform(0.05, 0.5, 3) * t / 3, rng.uniform(0.05, 1.0),
                     rng.uniform(0, 6))
    q = np.array([0.9, 0.2, 0.3, 0.1]) / np.linalg.norm([0.9, 0.2, 0.3, 0.1])
    for mean, quat, scale in (((0.0, 0.0, 3.0), q, (0.1, 0.0, 0.1)), ((0.0, 0.0, 3.0), (1, 0, 0, 0), (0.1, 0.0, 0.1)),
                              ((0.0, 0.0, 3.0), q, (0.1, 2e-39, 0.1)), ((0.0, 0.0, 3.0), (0, 0, 0, 0), (0.1, 0.1, 0.1)),
                              ((0.0, 0.0, math.inf), q, (0.3, 0.3, 0.3)), ((0.1, math.nan, 3.0), q, (0.3, 0.3, 0.3)),
                              ((-math.inf, 0.0, 3.0), (1, 0, 0, 0), (0.3, 0.3, 0.3)), ((0.1, 0.0, 3.0), q, (math.inf, 0.2, 0.2))):
        c = sw.image("degenerate", K=TIE_K)
        sw.add(c, mean, quat, scale, 0.8)
    # exact ties on the axis ray of pixel (22, 18)
    ident = (1.0, 0.0, 0.0, 0.0)
    for o in (ALPHA_TH, float(np.nextafter(f32(ALPHA_TH), f32(0))), MAX_ALPHA, float(np.nextafter(f32(MAX_ALPHA), f32(2)))):
        c = sw.image("tie", K=TIE_K)
        sw.add(c, (0.0, 0.0, 2.0), ident, (0.01, 0.01, 0.02), o)
        sw.images[c]["ties"].append((TIE_PIX, 0))
    c = sw.image("tie", K=TIE_K)
    for k, o in enumerate(STOP_OPACITIES):
        sw.add(c, (0.0, 0.0, 1.0 + k), ident, (0.01, 0.01, 0.02), o)
        sw.images[c]["ties"].append((TIE_PIX, k))
    sw.images[c]["stop_tie"] = _float32_stop()[0]
    for z in (0.0, 2.0**-20, -(2.0**-20)):
        c = sw.image("tie", K=TIE_K)
        sw.add(c, (0.01, 0.005, z), ident, (0.02, 0.02, 0.02), 0.9)
        # on the pixels (22 + k, 18 - 2 k) the ray's component along the mean's offset cancels exactly in float32 (y ==
        # -2 x is a power-of-two multiple) as in float64, so hit_t takes the sign of z there (+-0 at z = 0: kept)
        sw.images[c]["ties"].extend(((18 - 2 * k) * IW + 22 + k, 0) for k in range(-9, 10))
    return sw


def _stack(sw, cls, target):
    """3 to 5 gaussians on one pixel's ray; the last one's opacity brings T after it to `target` at that pixel"""
    rng = sw.rng
    c = sw.image(cls)
    px, py = sw.pixel()
    T, n = 1.0, 0
    while T > 0.01 or n < 2:
        al = rng.uniform(0.8, 0.95)
        sw.place(c, px, py, 1.0 + n, sw.quat(), rng.uniform(0.1, 0.4, 3), al, 0.0)
        T, n = T * (1 - float(f32(al))), n + 1
    sw.place(c, px, py, 1.0 + n, sw.quat(), rng.uniform(0.1, 0.4, 3), 1 - target / T, 0.0)


def arrays(sw, D=3, seed=7):
    """float32 inputs of one call: means / quats / scales [N, *], opacities [C, N], colours [C, N, D], backgrounds
    [C, D], Ks [C, 3, 3], viewmats [C, 4, 4], the tile lists, and per gaussian its image and slot."""
    rng = np.random.RandomState(seed + D)
    C = len(sw.images)
    gid, img, slot = [], [], []
    for c, im in enumerate(sw.images):
        for l, _ in enumerate(im["gs"]):
            gid.append((c, l))
            img.append(c)
            slot.append(l)
    N = len(gid)
    means = np.stack([sw.images[c]["gs"][l][0] for c, l in gid]).astype(f32)
    quats = np.stack([sw.images[c]["gs"][l][1] for c, l in gid]).astype(f32)
    scales = np.stack([sw.images[c]["gs"][l][2] for c, l in gid]).astype(f32)
    opac = np.full((C, N), 0.5, f32)
    for n, (c, l) in enumerate(gid):
        opac[c, n] = sw.images[c]["gs"][l][3]
    Ks = np.zeros((C, 3, 3), f32)
    for c, im in enumerate(sw.images):
        fx, fy, cx, cy = im["K"]
        Ks[c] = ((fx, 0, cx), (0, fy, cy), (0, 0, 1))
    vms = np.stack([im["vm"] for im in sw.images]).astype(f32)
    ids, offs = [], []
    first = np.cumsum([0] + [len(im["gs"]) for im in sw.images])
    for c, im in enumerate(sw.images):
        for _ in range(TW * TH):
            offs.append(len(ids))
            ids.extend(c * N + first[c] + l for l in range(len(im["gs"])))
    return dict(means=means, quats=quats, scales=scales, opacities=opac,
                colors=rng.uniform(-0.5, 1.5, (C, N, D)).astype(f32), backgrounds=rng.uniform(0, 1, (C, D)).astype(f32),
                Ks=Ks, viewmats=vms, flatten_ids=np.array(ids, np.int32),
                isect_offsets=np.array(offs, np.int32).reshape(C, TH, TW), img=np.array(img), slot=np.array(slot),
                first=first, L=max(len(im["gs"]) for im in sw.images),
                v_colors=rng.standard_normal((C, IH, IW, D)).astype(f32),
                v_alphas=rng.standard_normal((C, IH, IW, 1)).astype(f32))


def _perturb(arr, k):
    if k == 0:
        return arr
    rng = np.random.RandomState(1000 + k)
    out = dict(arr)
    for key in ("means", "quats", "scales", "opacities", "colors", "backgrounds", "Ks", "viewmats"):
        a = arr[key].astype(np.float64)
        with np.errstate(all="ignore"):
            out[key] = a * (1 + 4 * ULP * rng.uniform(-1, 1, a.shape))
    return out


def _cross(u, v):
    return torch.stack([u[..., 1] * v[..., 2] - u[..., 2] * v[..., 1], u[..., 2] * v[..., 0] - u[..., 0] * v[..., 2],
                        u[..., 0] * v[..., 1] - u[..., 1] * v[..., 0]], -1)


def evaluate(sw, arr, k=0, use_bg=True, masks=None, frozen=None):
    """float64 compositing of every image at perturbation k (0: the float32 inputs themselves).  Returns a dict of
    [C, P, L] pair quantities (raw = o * resp, hit, next_T, use, live), [C, P, *] images and the per-pair leaves
    (autograd: gradients on them are each pixel's share).  ``frozen``: the central evaluation, whose decisions are
    kept."""
    a = _perturb(arr, k)
    C, L = len(sw.images), arr["L"]
    t = lambda key: torch.as_tensor(np.asarray(a[key], np.float64))  # noqa: E731
    first = arr["first"]
    slot_ok = torch.zeros(C, L, dtype=torch.bool)
    gidx = torch.zeros(C, L, dtype=torch.long)
    for c, im in enumerate(sw.images):
        n = len(im["gs"])
        slot_ok[c, :n] = True
        gidx[c, :n] = torch.arange(first[c], first[c] + n)
        gidx[c, n:] = first[c]
    # rays
    Ks, vms = t("Ks"), t("viewmats")
    jj, ii = torch.meshgrid(torch.arange(IW, dtype=f64), torch.arange(IH, dtype=f64), indexing="xy")
    u, v = jj.reshape(-1) + 0.5, ii.reshape(-1) + 0.5
    d = torch.stack([(u[None] - Ks[:, 0, 2, None]) / Ks[:, 0, 0, None], (v[None] - Ks[:, 1, 2, None]) / Ks[:, 1, 1, None],
                     torch.ones(C, P, dtype=f64)], -1)
    d = d / d.norm(dim=-1, keepdim=True)
    R, tt = vms[:, :3, :3], vms[:, :3, 3]
    rd = torch.einsum("cji,cpj->cpi", R, d)[:, :, None]  # [C, P, 1, 3]
    ro = (-torch.einsum("cji,cj->ci", R, tt))[:, None, None]
    leaf = lambda x: x[:, None].expand((C, P) + x.shape[1:]).clone().requires_grad_(True)  # noqa: E731
    means, quats, scales = (leaf(t(key)[gidx]) for key in ("means", "quats", "scales"))
    opac = leaf(torch.gather(t("opacities"), 1, gidx))
    colors = leaf(t("colors")[torch.arange(C)[:, None], gidx])
    bg = t("backgrounds")[:, None].expand(C, P, -1).clone().requires_grad_(True)
    with np.errstate(all="ignore"):
        Rq = U.quat_to_rotmat(quats)
        M = Rq.transpose(-1, -2) / scales[..., :, None]
        w = ro - means
        aa = torch.einsum("cplij,cplj->cpli", M, w)
        b = torch.einsum("cplij,cplj->cpli", M, rd.expand_as(w))
        g = b / b.norm(dim=-1, keepdim=True)
        noise = np.random.RandomState(2000 + k) if k else None
        nz = lambda shape: torch.as_tensor(noise.uniform(-1, 1, shape))  # noqa: E731
        if k:
            aa = aa + nz(aa.shape) * (4 * ULP * torch.einsum("cplij,cplj->cpli", M.abs(), w.abs())).detach()
        hit = -(g * aa).sum(-1)
        cc = _cross(g, aa)
        if k:
            hit = hit + nz(hit.shape) * (4 * ULP * (g * aa).abs().sum(-1)).detach()
            cc = cc + nz(cc.shape) * (4 * ULP * g.norm(dim=-1) * aa.norm(dim=-1)).detach()[..., None]
        dist = (cc * cc).sum(-1)
        resp = torch.exp(-0.5 * dist)
        if k:
            resp = resp * (1 + nz(resp.shape) * ((4 + 0.5 * dist) * ULP).detach())
        raw = opac * resp
        alpha = torch.clamp(raw, max=MAX_ALPHA)
    # a scale whose float32 reciprocal overflows (0, or below 1/FLT_MAX) has no float32 M: no contribution
    with np.errstate(all="ignore"):
        recip_ok = torch.as_tensor(np.isfinite(f32(1.0) / arr["scales"]).all(-1))[gidx]
    ok = (slot_ok & recip_ok)[:, None]
    if masks is not None:
        mpix = torch.as_tensor(np.asarray(masks, bool)).reshape(C, TH, TW).repeat_interleave(16, 1).repeat_interleave(16, 2)
        ok = ok & mpix[:, :IH, :IW].reshape(C, P, 1)
    else:
        mpix = None
    if frozen is None:
        use = (hit >= 0) & (raw >= ALPHA_TH) & ok
    else:
        use = frozen["use"]
    am = torch.where(use, alpha, torch.zeros_like(alpha))
    Tin = torch.cumprod(torch.cat([torch.ones(C, P, 1, dtype=f64), 1 - am], -1), -1)
    if frozen is None:
        stop = use & (Tin[..., 1:] <= T_TH)
        for c, im in enumerate(sw.images):  # the float32 tie: next_T == float32(1e-4) exactly
            if im["stop_tie"] is not None:
                stop[c, TIE_PIX] = False
                stop[c, TIE_PIX, im["stop_tie"]] = True
    else:
        stop = frozen["stop"]
    alive = torch.cumsum(stop.to(torch.int64), -1) == 0
    wgt = am * Tin[..., :-1] * alive
    T = torch.prod(torch.where(alive, 1 - am, torch.ones_like(am)), -1)
    acc = (wgt[..., None] * colors).sum(-2)
    col = acc + T[..., None] * bg if use_bg else acc
    live = torch.cat([torch.ones(C, P, 1, dtype=torch.bool), alive[..., :-1]], -1) & ok
    absum = ((wgt[..., None] * colors).abs().sum(-2) + (T[..., None] * bg).abs() * use_bg).detach()
    return dict(raw=raw.detach(), hit=hit.detach(), next_T=Tin[..., 1:].detach(), use=use, stop=stop, live=live,
                col=col, alpha=1 - T, T=T.detach(), absum=absum, leaves=(means, quats, scales, colors, opac, bg),
                mpix=mpix)


def _spread(x0, xs):
    with np.errstate(all="ignore"):
        dev = torch.stack([(x - x0).abs() for x in xs]).nan_to_num(nan=math.inf)
    return 4 * dev.max(0).values


def truth(sw, arr, use_bg=True, masks=None, grads=True):
    """central float64 results with their budgets and the decided pixels [C, P] and gaussians [N]."""
    ev = [evaluate(sw, arr, 0, use_bg, masks)]
    ev += [evaluate(sw, arr, k, use_bg, masks, frozen=ev[0]) for k in range(1, N_PERTURB + 1)]
    e0 = ev[0]
    C, L = len(sw.images), arr["L"]
    raw, hit, nT, use, live = e0["raw"], e0["hit"], e0["next_T"], e0["use"], e0["live"]
    B_raw = _spread(raw, [e["raw"] for e in ev[1:]])
    B_hit = _spread(hit, [e["hit"] for e in ev[1:]])
    B_T = _spread(nT, [e["next_T"] for e in ev[1:]]) + 2 * ULP * torch.arange(1, L + 1, dtype=f64) * nT
    tie = torch.zeros(C, P, L, dtype=torch.bool)
    for c, im in enumerate(sw.images):
        for p, l in im["ties"]:
            tie[c, p, l] = True
    with np.errstate(all="ignore"):
        clear_a = (raw - ALPHA_TH).abs() > B_raw
        below = raw < ALPHA_TH - B_raw
        dec = (clear_a & ((raw - MAX_ALPHA).abs() > B_raw) & ((hit.abs() > B_hit) | below)
               & (~use | ((nT - T_TH).abs() > B_T)))
        dec = dec | ~torch.isfinite(raw) | ~torch.isfinite(hit) | tie | ~live
    pix_dec = dec.all(-1)
    out = dict(ev=e0, pix_dec=pix_dec, pair_dec=dec, B_raw=B_raw, B_hit=B_hit, B_T=B_T)
    col0, a0 = e0["col"].detach(), e0["alpha"].detach()
    out["col"], out["alpha"] = col0, a0
    out["B_col"] = _spread(col0, [e["col"].detach() for e in ev[1:]]) + 2 * (L + 2) * ULP * e0["absum"]
    out["B_alpha"] = _spread(a0, [e["alpha"].detach() for e in ev[1:]]) + 2 * (L + 1) * ULP
    if not grads:
        return out
    vcol = torch.as_tensor(arr["v_colors"].astype(np.float64)).reshape(C, P, -1)
    val = torch.as_tensor(arr["v_alphas"].astype(np.float64)).reshape(C, P)
    G = []
    for e in ev:
        loss = (e["col"] * vcol).sum() + (e["alpha"] * val).sum()
        with np.errstate(all="ignore"):
            G.append(torch.autograd.grad(loss, e["leaves"], allow_unused=True))
    names = ("means", "quats", "scales", "colors", "opacities", "backgrounds")
    c_of, l_of = torch.as_tensor(arr["img"]), torch.as_tensor(arr["slot"])
    tf = e0["T"].clamp_min(T_TH)  # [C, P]
    # per gaussian: share [N, P, *] of each pixel
    grads_out, budgets = {}, {}
    for i, name in enumerate(names):
        def per_g(gr):
            if name == "backgrounds":
                return gr
            return gr[c_of, :, l_of]
        shares = [per_g(gg[i] if gg[i] is not None else torch.zeros_like(e0["leaves"][i])).nan_to_num(nan=0.0) for gg in G]
        tot = [s.sum(1) for s in shares]
        absum = shares[0].abs().sum(1)
        tfac = (shares[0].abs() * (2 * ULP / (tf[c_of] if name != "backgrounds" else tf)).reshape(
            shares[0].shape[:2] + (1,) * (shares[0].dim() - 2))).sum(1)
        grads_out[name] = tot[0]
        budgets[name] = _spread(tot[0], tot[1:]) + K_GRAD * ULP * absum + tfac
    out["grads"], out["B_grads"] = grads_out, budgets
    # a gaussian is decided when every pixel it reaches is
    reach = live[c_of, :, l_of]
    out["g_dec"] = (pix_dec[c_of] | ~reach).all(1)
    out["bg_dec"] = pix_dec.all(1)
    return out


def classes(sw):
    return np.array([im["cls"] for im in sw.images])


# ------------------------------------------------------------------------------------------------------------------
# pixel rays
def lens_cases():
    """{name: dict(camera kwargs for rasterize_to_pixels_eval3d (numpy), oracle camera, valid [H*W], decided [H*W])}:
    ut_edges' distorted pinhole (k1 = float32(0.8) - 1 folds near normalised radius 0.86, inside the image) and fisheye
    (negative k1 ends the monotone range inside the image), one FTheta calibration with the forward polynomial as the
    reference, and linear maps with |c - e d| = 3 * 2^-28 (valid) and 2 * 2^-28 (singular)."""
    from tests import scene
    k1 = F32(f32(0.8) - f32(1))
    out = {}
    jj, ii = np.meshgrid(np.arange(IW, dtype=np.float64), np.arange(IH, dtype=np.float64), indexing="xy")
    u, v = jj.reshape(-1) + 0.5, ii.reshape(-1) + 0.5
    specs = {
        "distorted": ("pinhole", (20.0, 22.0, 21.5, 17.0), dict(radial=(k1, 0, 0, 0, 0, 0), tangential=(2.0**-7, -(2.0**-8)))),
        "fisheye": ("fisheye", (14.0, 16.0, 22.0, 18.5), dict(radial=(-0.2, 0.0, 0.0, 0.0))),
    }
    for name, (kind, (fx, fy, cx, cy), co) in specs.items():
        K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], f32)
        co = {key: np.array(val, f32) for key, val in co.items()}
        runs = []
        for kp in range(N_PERTURB + 1):
            rng = np.random.RandomState(3000 + kp)
            pert = lambda x: x.astype(np.float64) * (1 + (4 * ULP * rng.uniform(-1, 1, x.shape) if kp else 0))  # noqa: E731
            cam = U.Camera(kind, pert(K), IW, IH, **{key: pert(val) for key, val in co.items()})
            d, ok = cam.unproject(torch.tensor(u), torch.tensor(v), rule="reference")
            runs.append((cam, d, ok, cam.trace))
        cam, d, ok, tr = runs[0]
        rho = torch.as_tensor(np.hypot((u - cx) / fx, (v - cy) / fy))  # normalised radius of the distorted point
        dec = torch.ones(len(u), dtype=torch.bool)
        if kind == "pinhole":
            # float32 rounding of what each comparison takes: the residual x0 - D(x) at 6 ulp of the point's size
            # (icD x + offset: four roundings of icD ~ 1 + |k1| rho^2, one of the product, one of the difference),
            # through J^-1 into the step, plus the float32 iterate's drift of 1 ulp of rho per step; icD and det at
            # 8 ulp of their terms (each of size ~1 + |k1| rho^2)
            size = rho * (1 + abs(k1) * rho * rho)
            rnd = {"step": 6 * ULP * size * (1 + tr["jinv"].nan_to_num(nan=0.0)) + ULP * 5 * rho,
                   "det": 8 * ULP * (1 + abs(k1) * rho * rho) ** 2 * 4, "icd": 8 * ULP * (1 + abs(k1) * rho * rho)}
            thr = {"step": 1e-6, "det": 1e-6, "icd": 0.0}
        else:
            # the step (f(t) - delta) / f'(t): its numerator at 6 ulp of t (1 + |k1| t^2) + delta (four roundings of
            # f, one of the difference), over |f'(t)|, and the iterate's own rounding of 2 ulp of t (Newton does not let it
            # accumulate); t against 0
            # and max_angle at 16 ulp of the angle, which also bounds the float32 bisection of f' that gives the
            # kernel's max_angle
            t_fin = tr["t"]
            fe_d = cam._dfe(t_fin).abs().clamp_min(1e-12)
            rnd = {"step": 6 * ULP * (t_fin.abs() * (1 + 0.2 * t_fin * t_fin) + rho) / fe_d + 2 * ULP * t_fin.abs()}
            sp_t = _spread(t_fin, [r[3]["t"] for r in runs[1:]])
            conv = (tr["step"] < 1e-6).any(0)  # t decides only where the iteration converged
            dec = dec & ((t_fin.abs() > sp_t + 16 * ULP * t_fin.abs()) | (t_fin == 0) | ~conv)
            thr = {"step": 1e-6}
            dec = dec & (((t_fin - cam.max_angle).abs()
                         > 16 * ULP * cam.max_angle + sp_t) | ~conv)
        for key in thr:
            x0 = tr[key].abs() if key == "det" else tr[key]
            sp = _spread(x0, [(r[3][key].abs() if key == "det" else r[3][key]) for r in runs[1:]])
            with np.errstate(all="ignore"):
                m = (x0 - thr[key]).abs() > sp + rnd[key]
            dec = dec & (m | torch.isnan(x0)).all(0)
        out[name] = dict(camera_model=kind, K=K, coeffs={U_KEYS[key]: val[None] for key, val in co.items()}, cam=cam,
                         valid=ok.numpy(), decided=dec.numpy())
    # FTheta: the oracle replays the kernel's rule; the last Newton step against 1e-6
    cal = scene.calibrations()["cross_left_120fov"]
    params, pp, _ = scene.scaled(cal, IW)
    params = dict(params, reference_poly=U.ANGLE_TO_PIXELDIST)
    K = np.array([[1, 0, pp[0]], [0, 1, pp[1]], [0, 0, 1]], f32)
    cam = U.FThetaCamera(params, K, IW, IH)
    dirs, ok = cam.unproject(torch.tensor(u), torch.tensor(v))
    ls = cam.last_step
    # the last step (fw(th) - delta) / fw'(th): its numerator at 6 ulp of sum |c_k th^k| + delta, over |fw'(th)|,
    # and the iterate's drift of 1 ulp of th per step
    th = torch.atan2(dirs[:, :2].norm(dim=-1), dirs[:, 2])
    fw = params["angle_to_pixeldist_poly"]
    terms = sum(abs(c) * th.abs() ** n for n, c in enumerate(fw))
    dfw = U.poly(U.dpoly(fw), th).abs().clamp_min(1e-12)
    dec = (ls - 1e-6).abs() > 6 * ULP * terms / dfw + 3 * ULP * th.abs()
    out["ftheta"] = dict(camera_model="ftheta", K=K, ftheta=params, cam=cam, valid=ok.numpy(), decided=dec.numpy())
    for name, k in (("linear_valid", 3), ("linear_singular", 2)):
        e = 1.0 - k * 2.0**-24  # c = d = 1/16: c - e d = k 2^-28, exact in float32 and float64
        prm = dict(pixeldist_to_angle_poly=[0.0, 1e-10, 0, 0, 0, 0], angle_to_pixeldist_poly=[0.0, 1e10, 0, 0, 0, 0],
                   max_angle=1.5, linear_cde=[1.0 / 16, 1.0 / 16, e], reference_poly=U.PIXELDIST_TO_ANGLE)
        K = np.array([[1, 0, 22.0], [0, 1, 18.0], [0, 0, 1]], f32)
        cam = U.FThetaCamera(prm, K, IW, IH)
        _, ok = cam.unproject(torch.tensor(u), torch.tensor(v))
        out[name] = dict(camera_model="ftheta", K=K, ftheta=prm, cam=cam, valid=ok.numpy(),
                         decided=np.ones(len(u), bool))
    return out


U_KEYS = {"radial": "radial_coeffs", "tangential": "tangential_coeffs", "thin": "thin_prism_coeffs"}
# undecided share of the pixels per lens: the fisheye's pixels beyond its monotone range wander in Newton (steps of
# order 1) before converging to a negative angle or not at all, and their step sequences are not stable under the
# input perturbations, so most of them stay undecided
LENS_UNDECIDED_MAX = dict(distorted=0.25, fisheye=0.72, ftheta=0.01, linear_valid=0.0, linear_singular=0.0)


def subset(sw, per_class=2):
    """the first `per_class` images of every class, for the channel sweep"""
    out = Sweep()
    seen = {}
    for im in sw.images:
        if seen.get(im["cls"], 0) < per_class:
            seen[im["cls"]] = seen.get(im["cls"], 0) + 1
            out.images.append(im)
    return out


def tile_masks(sw, seed=11):
    """[C, TH, TW] tile masks with two tiles of every image masked out"""
    rng = np.random.RandomState(seed)
    m = np.ones((len(sw.images), TH * TW), bool)
    for c in range(len(sw.images)):
        m[c, rng.choice(TH * TW, 2, replace=False)] = False
    return m.reshape(-1, TH, TW)


def no_contribution(sw, arr):
    """[N] gaussians that contribute nothing anywhere by rule (non-finite float32 M or mean)"""
    with np.errstate(all="ignore"):
        bad_s = ~np.isfinite(f32(1.0) / arr["scales"]).all(-1)
        bad_q = (arr["quats"] == 0).all(-1)
        bad_m = ~np.isfinite(arr["means"]).all(-1)
    return bad_s | bad_q | bad_m
