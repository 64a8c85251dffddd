"""The 3DGUT compositing kernels against the float64 truth of tests/eval3d_edges.py: per pixel on the decided pixels
and per gaussian on the decided gaussians (v_means, v_quats, v_scales, v_colors, v_opacities, v_backgrounds), every
channel count with and without backgrounds and with masked tiles, and the per-pixel validity of the pixel rays under
the distorted pinhole, the fisheye and FTheta.  Undecided pixels and gaussians are counted and bounded per class."""
import numpy as np
import pytest
import torch

import gsplat_b200 as gs
from tests import eval3d_edges as E

pytestmark = pytest.mark.gpu
DEV = "cuda"
SWEEP = E.make_sweep()
NAMES = ("means", "quats", "scales", "colors", "opacities", "backgrounds")


def _t(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)


def _run(arr, use_bg, masks=None):
    leaves = [_t(arr[k], True) for k in NAMES]
    bg = leaves[5] if use_bg else None
    rc, ra = gs.rasterize_to_pixels_eval3d(
        leaves[0], leaves[1], leaves[2], leaves[3], leaves[4], _t(arr["viewmats"]), _t(arr["Ks"]), E.IW, E.IH, 16,
        _t(arr["isect_offsets"]), _t(arr["flatten_ids"]), backgrounds=bg,
        masks=None if masks is None else _t(masks), camera_model="pinhole")
    loss = (rc * _t(arr["v_colors"])).sum() + (ra * _t(arr["v_alphas"])).sum()
    loss.backward()
    grads = {k: (l.grad if l.grad is not None else torch.zeros_like(l)).cpu().double() for k, l in zip(NAMES, leaves)}
    return rc.detach().cpu().double(), ra.detach().cpu().double(), grads


def _check(sw, arr, use_bg, masks=None, report=None):
    tr = E.truth(sw, arr, use_bg=use_bg, masks=masks)
    rc, ra, grads = _run(arr, use_bg, masks)
    C, D = len(sw.images), arr["colors"].shape[-1]
    cls = E.classes(sw)
    pd = tr["pix_dec"]
    for name, g in grads.items():
        assert torch.isfinite(g).all(), f"non-finite {name} gradient"
    err_c = (rc.reshape(C, E.P, D) - tr["col"]).abs() > tr["B_col"]
    err_a = (ra.reshape(C, E.P) - tr["alpha"]).abs() > tr["B_alpha"]
    bad = (err_c.any(-1) | err_a) & pd
    assert not bad.any(), f"{int(bad.sum())} decided pixels off budget, images {sorted(set(np.nonzero(bad.numpy())[0].tolist()))}"
    if masks is not None:
        mp = torch.as_tensor(masks).repeat_interleave(16, 1).repeat_interleave(16, 2)[:, :E.IH, :E.IW].reshape(C, E.P)
        bgv = torch.as_tensor(arr["backgrounds"].astype(np.float64)) if use_bg else torch.zeros(C, D, dtype=torch.float64)
        out = rc.reshape(C, E.P, D)[~mp]
        assert torch.equal(out, bgv[:, None].expand(C, E.P, D)[~mp]) and (ra.reshape(C, E.P)[~mp] == 0).all()
    # per gaussian
    img, n = torch.as_tensor(arr["img"]), torch.arange(len(arr["img"]))
    kern = {"means": grads["means"], "quats": grads["quats"], "scales": grads["scales"],
            "colors": grads["colors"][img, n], "opacities": grads["opacities"][img, n]}
    gdec = tr["g_dec"]
    for name, kv in kern.items():
        tv, bv = tr["grads"][name], tr["B_grads"][name]
        off = ((kv - tv).abs() > bv).reshape(len(n), -1).any(-1) & gdec
        assert not off.any(), (f"v_{name} off budget on gaussians {torch.nonzero(off).flatten().tolist()[:10]}: kernel "
                               f"{kv[off][:3].tolist()} truth {tv[off][:3].tolist()} budget {bv[off][:3].tolist()}")
    if use_bg:
        off = ((grads["backgrounds"] - tr["grads"]["backgrounds"]).abs() > tr["B_grads"]["backgrounds"]).any(-1) & tr["bg_dec"]
        assert not off.any(), f"v_backgrounds off budget on images {torch.nonzero(off).flatten().tolist()}"
    # gaussians that contribute nothing by rule get exactly zero gradients
    none = torch.as_tensor(E.no_contribution(sw, arr))
    for name, kv in kern.items():
        assert (kv[none] == 0).all(), f"v_{name} of a non-contributing gaussian"
    # undecided counts per class
    gcls = cls[arr["img"]]
    for c in E.CLASSES:
        m = torch.as_tensor(cls == c)
        if not m.any():
            continue
        und_p = float((~pd[m]).float().mean())
        und_g = float((~gdec[torch.as_tensor(gcls == c)]).float().mean())
        if report is not None:
            report.append((c, D, use_bg, int((~pd[m]).sum()), int(pd[m].numel()), int((~gdec[torch.as_tensor(gcls == c)]).sum()),
                           int((gcls == c).sum())))
        assert und_p <= E.UNDECIDED_MAX[c], (c, und_p)
        assert und_g <= E.G_UNDECIDED_MAX[c] + 1e-12, (c, und_g)


def test_sweep_against_float64():
    report = []
    _check(SWEEP, E.arrays(SWEEP, 3), True, report=report)
    for r in report:
        print("class %-10s D=%d bg=%d undecided pixels %d / %d, gaussians %d / %d" % r)


SUB = E.subset(SWEEP)


@pytest.mark.parametrize("D", E.CHANNELS)
@pytest.mark.parametrize("use_bg", [True, False])
def test_channels_backgrounds_and_masks(D, use_bg):
    _check(SUB, E.arrays(SUB, D), use_bg, masks=E.tile_masks(SUB))


@pytest.mark.parametrize("lens", ["distorted", "fisheye", "ftheta", "linear_valid", "linear_singular"])
def test_pixel_ray_validity(lens):
    case = E.lens_cases()[lens]
    o = 0.5
    kw = dict(camera_model=case["camera_model"])
    if case["camera_model"] == "ftheta":
        kw["ftheta_coeffs"] = gs.FThetaCameraDistortionParameters(**case["ftheta"])
    else:
        kw.update({k: _t(v) for k, v in case["coeffs"].items()})
    offs = torch.zeros(1, E.TH, E.TW, dtype=torch.int32, device=DEV)
    offs.view(-1)[:] = torch.arange(E.TH * E.TW, dtype=torch.int32)
    fids = torch.zeros(E.TH * E.TW, dtype=torch.int32, device=DEV)
    _, ra = gs.rasterize_to_pixels_eval3d(
        _t(np.zeros((1, 3), np.float32)), _t(np.array([[1, 0, 0, 0]], np.float32)), _t(np.ones((1, 3), np.float32)),
        _t(np.ones((1, 1, 1), np.float32)), _t(np.full((1, 1), o, np.float32)), _t(np.eye(4, dtype=np.float32)[None]),
        _t(case["K"][None]), E.IW, E.IH, 16, offs, fids, **kw)
    got = ra.reshape(-1).cpu().numpy()
    want = np.where(case["valid"], np.float32(o), np.float32(0))
    dec = case["decided"]
    print(f"{lens}: valid {int(case['valid'].sum())}, undecided {int((~dec).sum())} / {dec.size}")
    assert np.isin(got, (0.0, np.float32(o))).all()
    bad = (got != want) & dec
    assert not bad.any(), f"{int(bad.sum())} decided pixels disagree on ray validity, first {np.nonzero(bad)[0][:8]}"
    assert (~dec).mean() <= E.LENS_UNDECIDED_MAX[lens]
