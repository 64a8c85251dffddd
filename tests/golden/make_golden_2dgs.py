#!/usr/bin/env python
"""Generate tests/golden/ref_2dgs.npz and ref_signatures_2dgs.json from the REFERENCE ITSELF (2DGS).

Runs only where the reference sources are available, like make_golden.py, whose nerfacc shim it imports.  The
reference's pure-PyTorch twins are evaluated on the CPU in float64:

  * gsplat/cuda/_torch_impl_2dgs.py  _fully_fused_projection_2dgs  (projection; outputs and autograd gradients)
  * gsplat/cuda/_torch_impl_2dgs.py  accumulate_2dgs               (compositing of a pair list; autograd gradients)

The pair list fed to accumulate_2dgs is every (gaussian, pixel) pair of a small scene whose gaussians overlap little,
front to back per pixel: the twin has no alpha threshold and no transmittance stop, so the fixture keeps those two
decisions away from every pair (tests/test_2dgs_cpu.py states what it allows for).

Usage:  python tests/golden/make_golden_2dgs.py        (from the repo root)
"""
import ast
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (reference on sys.path, nerfacc shim installed)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import gsplat  # noqa: E402
from gsplat.cuda._torch_impl_2dgs import _fully_fused_projection_2dgs, accumulate_2dgs  # noqa: E402

GSPLAT = os.path.dirname(os.path.abspath(gsplat.__file__))  # the reference package make_golden.py put on the path

f64 = torch.float64


def make_signatures():
    out = {}
    for path, names in (
        (os.path.join(GSPLAT, "cuda", "_wrapper.py"), ("fully_fused_projection_2dgs", "rasterize_to_pixels_2dgs")),
        (os.path.join(GSPLAT, "rendering.py"), ("rasterization_2dgs",)),
    ):
        tree = ast.parse(open(path).read())
        for node in ast.walk(tree):
            if isinstance(node, ast.FunctionDef) and node.name in names:
                a = node.args
                out[node.name] = {"params": [x.arg for x in a.posonlyargs + a.args + a.kwonlyargs], "n_defaults": len(a.defaults)}
    with open(os.path.join(HERE, "ref_signatures_2dgs.json"), "w") as f:
        json.dump({"params": out}, f, indent=1)
    print("wrote ref_signatures_2dgs.json")


def make_projection(rng):
    """2 cameras looking down +z at surfels in front of them; a few rows behind the near plane and off-screen."""
    N, C, W, H = 64, 2, 64, 48
    means = np.stack([rng.uniform(-1.2, 1.2, N), rng.uniform(-0.9, 0.9, N), rng.uniform(2.0, 6.0, N)], -1)
    means[:3, 2] = [-1.0, 0.005, 3.0]
    means[2, 0] = 40.0  # off-screen
    quats = rng.standard_normal((N, 4))
    scales = rng.uniform(0.02, 0.12, (N, 3))
    viewmats = np.tile(np.eye(4), (C, 1, 1))
    viewmats[1, :3, 3] = [0.1, -0.05, 0.2]
    ang = 0.1
    viewmats[1, :3, :3] = [[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]]
    Ks = np.tile(np.array([[60.0, 0, W / 2], [0, 60.0, H / 2], [0, 0, 1]]), (C, 1, 1))
    t = {k: torch.tensor(v, dtype=f64, requires_grad=True) for k, v in dict(means=means, quats=quats, scales=scales, viewmats=viewmats).items()}
    radii, means2d, depths, rt, normals = _fully_fused_projection_2dgs(t["means"], t["quats"], t["scales"], t["viewmats"], torch.tensor(Ks, dtype=f64), W, H)
    cot = {k: torch.tensor(rng.standard_normal(v.shape)) for k, v in dict(means2d=means2d, depths=depths, rt=rt, normals=normals).items()}
    vis = (radii > 0).all(-1)
    loss = sum(((o * cot[k]) * vis.reshape(vis.shape + (1,) * (o.dim() - vis.dim()))).sum()
               for k, o in dict(means2d=means2d, depths=depths, rt=rt, normals=normals).items())
    g = torch.autograd.grad(loss, [t["means"], t["quats"], t["scales"], t["viewmats"]])
    return dict(
        p_means=means, p_quats=quats, p_scales=scales, p_viewmats=viewmats, p_Ks=Ks, p_width=np.int64(W), p_height=np.int64(H),
        p_radii=radii.numpy(), p_means2d=means2d.detach().numpy(), p_depths=depths.detach().numpy(), p_ray_transforms=rt.detach().numpy(),
        p_normals=normals.detach().numpy(), p_v_means2d=cot["means2d"].numpy(), p_v_depths=cot["depths"].numpy(),
        p_v_ray_transforms=cot["rt"].numpy(), p_v_normals=cot["normals"].numpy(), p_g_means=g[0].numpy(), p_g_quats=g[1].numpy(),
        p_g_scales=g[2].numpy(), p_g_viewmats=g[3].numpy(),
    )


def make_compositing(rng):
    """One camera, 24 x 20 pixels, 12 surfels facing the camera at different depths; every pixel gets every surfel whose
    alpha there is >= 1/255 (decided in float64 by the twin's own formula), front to back."""
    N, W, H, D = 12, 24, 20, 4
    means = np.stack([rng.uniform(-0.25, 0.25, N), rng.uniform(-0.2, 0.2, N), np.linspace(2.0, 4.0, N)], -1)
    quats = np.concatenate([np.ones((N, 1)), rng.uniform(-0.3, 0.3, (N, 3))], -1)
    scales = rng.uniform(0.03, 0.08, (N, 3))
    Ks = np.array([[[40.0, 0, W / 2], [0, 40.0, H / 2], [0, 0, 1]]])
    vm = np.eye(4)[None]
    with torch.no_grad():
        radii, means2d, depths, rt, normals = _fully_fused_projection_2dgs(*(torch.tensor(a, dtype=f64) for a in (means, quats, scales, vm, Ks)), W, H)
    opac = rng.uniform(0.2, 0.6, (1, N))
    colors = np.concatenate([rng.uniform(0, 1, (1, N, D - 1)), depths.numpy()[..., None]], -1)
    m2 = torch.tensor(means2d.numpy(), requires_grad=True)
    rtt = torch.tensor(rt.numpy(), requires_grad=True)
    op = torch.tensor(opac, requires_grad=True)
    co = torch.tensor(colors, requires_grad=True)
    nr = torch.tensor(normals.numpy(), requires_grad=True)
    # pair list: the twin's own alpha per (pixel, gaussian), thresholded at 1/255, sorted by depth per pixel
    pix = torch.arange(W * H)
    px, py = (pix % W + 0.5).double(), (pix // W + 0.5).double()
    hu = -rtt[0, None, :, 0, :] + rtt[0, None, :, 2, :] * px[:, None, None]
    hv = -rtt[0, None, :, 1, :] + rtt[0, None, :, 2, :] * py[:, None, None]
    s = torch.cross(hu, hv, dim=-1)
    g3 = (s[..., 0] / s[..., 2]) ** 2 + (s[..., 1] / s[..., 2]) ** 2
    d = torch.stack([px, py], -1)[:, None, :] - m2[0, None]
    g2 = 2 * (d ** 2).sum(-1)
    al = torch.clamp_max(op[0, None] * torch.exp(-0.5 * torch.minimum(g3, g2)), 0.99).detach()
    keep = al >= 1.0 / 255.0
    order = torch.argsort(depths[0])
    p_l, g_l = [], []
    for p in range(W * H):
        for gi in order.tolist():
            if keep[p, gi]:
                p_l.append(p), g_l.append(gi)
    g_t, p_t = torch.tensor(g_l), torch.tensor(p_l)
    i_t = torch.zeros_like(g_t)
    rc, ra, rn = accumulate_2dgs(m2, rtt, op, co, nr, g_t, p_t, i_t, W, H)
    cot = [torch.tensor(rng.standard_normal(x.shape)) for x in (rc, ra, rn)]
    g = torch.autograd.grad(sum((a * b).sum() for a, b in zip((rc, ra, rn), cot)), [m2, rtt, op, co, nr])
    amin = float(al[keep].min())
    return dict(
        c_means2d=means2d.numpy(), c_ray_transforms=rt.numpy(), c_opacities=opac, c_colors=colors, c_normals=normals.numpy(),
        c_radii=radii.numpy(), c_depths=depths.numpy(), c_width=np.int64(W), c_height=np.int64(H), c_render_colors=rc.detach().numpy(),
        c_render_alphas=ra.detach().numpy(), c_render_normals=rn.detach().numpy(), c_v_render_colors=cot[0].numpy(),
        c_v_render_alphas=cot[1].numpy(), c_v_render_normals=cot[2].numpy(), c_g_means2d=g[0].numpy(), c_g_ray_transforms=g[1].numpy(),
        c_g_opacities=g[2].numpy(), c_g_colors=g[3].numpy(), c_g_normals=g[4].numpy(), c_n_pairs=np.int64(len(g_l)),
        c_min_alpha=np.float64(amin), c_min_transmittance=np.float64(1.0 - ra.detach().max()),
    )


if __name__ == "__main__":
    rng = np.random.RandomState(20261016)
    make_signatures()
    out = make_projection(rng)
    out.update(make_compositing(rng))
    make_golden.save("ref_2dgs.npz", **out)
