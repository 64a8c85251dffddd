"""The sweep of tests/eval3d_edges.py is what it claims (no GPU): every class is present and mostly decided, the ties lie
exactly on their thresholds in a float32 emulation of eval_hit, the vectorised truth equals oracle.ut.eval3d_render, the
replayed unprojection rule agrees with the converged oracle ray wherever it says valid, and the budgets are small."""
import numpy as np
import pytest
import torch

from oracle import ut as U
from tests import eval3d_edges as E

f32 = np.float32


@pytest.fixture(scope="module")
def sweep():
    sw = E.make_sweep()
    arr = E.arrays(sw, 3)
    return sw, arr, E.truth(sw, arr)


def test_classes_present_and_mostly_decided(sweep):
    sw, arr, tr = sweep
    cls = E.classes(sw)
    gcls = cls[arr["img"]]
    for c in E.CLASSES:
        m = cls == c
        assert m.sum() >= 4, c
        assert float((~tr["pix_dec"][torch.as_tensor(m)]).float().mean()) <= E.UNDECIDED_MAX[c], c
        assert float((~tr["g_dec"][torch.as_tensor(gcls == c)]).float().mean()) <= E.G_UNDECIDED_MAX[c] + 1e-12, c
    # every gaussian composites somewhere, except the ones that by rule cannot (ties below their threshold aside)
    none = E.no_contribution(sw, arr)
    used = tr["ev"]["use"].any(1)  # [C, L]
    for n in range(len(none)):
        if gcls[n] != "tie":
            assert bool(used[arr["img"][n], arr["slot"][n]]) != bool(none[n]), n


def _emulate_hit(mean, quat, scale, o, d):
    """eval_hit of ut.cu in float32 (ut.cu is built with -fmad=false), identity quaternions only, origin 0"""
    assert tuple(quat) == (1, 0, 0, 0)
    inv = f32(1) / scale
    w = (f32(0) - mean).astype(f32)
    a = (inv * w).astype(f32)
    b = (inv * d).astype(f32)
    l2 = f32(f32(b[0] * b[0] + b[1] * b[1]) + b[2] * b[2])
    g = (b * (f32(1) / np.sqrt(l2))).astype(f32)
    hit = -f32(f32(f32(g[0] * a[0]) + f32(g[1] * a[1])) + f32(g[2] * a[2]))
    c = np.array([g[1] * a[2] - g[2] * a[1], g[2] * a[0] - g[0] * a[2], g[0] * a[1] - g[1] * a[0]], f32)
    dist = f32(f32(c[0] * c[0] + c[1] * c[1]) + c[2] * c[2])
    return hit, dist, f32(o) if dist == 0 else None


def test_ties_are_exact(sweep):
    sw, arr, tr = sweep
    seen = 0
    for c, im in enumerate(sw.images):
        if im["cls"] != "tie":
            continue
        fx, fy, cx, cy = im["K"]
        for p, l in im["ties"]:
            i, j = divmod(p, E.IW)
            x, y = f32(f32(j + 0.5) - f32(cx)) / f32(fx), f32(f32(i + 0.5) - f32(cy)) / f32(fy)
            inv = f32(1) / np.sqrt(f32(f32(x * x + y * y) + f32(1)))
            d = np.array([x * inv, y * inv, inv], f32)
            mean, quat, scale, o = im["gs"][l]
            hit, dist, alpha = _emulate_hit(mean, quat, scale, o, d)
            z = float(mean[2])
            if p == E.TIE_PIX and mean[0] == 0:
                assert dist == 0 and hit > 0 and alpha == f32(o)  # alpha == o exactly, on its threshold
            else:
                assert (hit == 0) if z == 0 else (np.sign(hit) == np.sign(z)), (c, p, hit)
                assert float(tr["ev"]["hit"][c, p, l]) == 0 if z == 0 else np.sign(float(tr["ev"]["hit"][c, p, l])) == np.sign(z)
            seen += 1
    ops = [im["gs"][0][3] for im in sw.images if im["cls"] == "tie"]
    assert f32(E.ALPHA_TH) in ops and np.nextafter(f32(E.ALPHA_TH), f32(0)) in ops
    assert f32(E.MAX_ALPHA) in ops and np.nextafter(f32(E.MAX_ALPHA), f32(2)) in ops
    k, nT = E._float32_stop()
    assert k == len(E.STOP_OPACITIES) - 1 and nT == f32(E.T_TH)
    assert seen > 10


def test_truth_equals_oracle_render(sweep):
    sw, arr, tr = sweep
    cls = E.classes(sw)
    pick = [int(np.nonzero(cls == c)[0][0]) for c in ("alpha", "clamp", "stop", "edges", "bulk", "hit")]
    N = len(arr["img"])
    t = lambda x: torch.as_tensor(np.asarray(x, np.float64))  # noqa: E731
    for c in pick:
        fx, fy, cx, cy = sw.images[c]["K"]
        cam = U.Camera("pinhole", [[fx, 0, cx], [0, fy, cy], [0, 0, 1]], E.IW, E.IH)
        col, alp, _ = U.eval3d_render(t(arr["means"]), t(arr["quats"]), t(arr["scales"]), t(arr["colors"]).reshape(-1, 3),
                                      t(arr["opacities"]).reshape(-1), t(arr["viewmats"][c]), cam,
                                      torch.as_tensor(arr["isect_offsets"]), arr["flatten_ids"].tolist(), len(sw.images),
                                      N, c, background=t(arr["backgrounds"][c]))
        # the oracle thresholds and clamps alpha at 1/255 and 0.99 in float64, the sweep at their float32 values as the
        # kernels do: 0.99 differs by 1e-8
        away = ((tr["ev"]["raw"][c] - E.ALPHA_TH).abs() > 1e-9).all(-1)
        assert away.float().mean() > 0.99
        assert torch.allclose(col.reshape(E.P, 3)[away], tr["col"][c][away], rtol=0, atol=1e-7), c
        assert torch.allclose(alp.reshape(E.P)[away], tr["alpha"][c][away], rtol=0, atol=1e-7), c


def test_replayed_rule_agrees_with_converged_ray():
    for name, case in E.lens_cases().items():
        if case["camera_model"] == "ftheta":
            continue
        cam = case["cam"]
        jj, ii = np.meshgrid(np.arange(E.IW) + 0.5, np.arange(E.IH) + 0.5, indexing="xy")
        u, v = torch.tensor(jj.reshape(-1)), torch.tensor(ii.reshape(-1))
        d_ref, ok_ref = cam.unproject(u, v, rule="reference")
        d_conv, ok_conv = cam.unproject(u, v)
        both = ok_ref & ok_conv
        assert both.sum() >= 0.9 * ok_ref.sum(), name
        assert ((d_ref - d_conv).norm(dim=-1)[both] < 1e-5).all(), name
        assert case["valid"].any() and not case["valid"].all(), name  # the image straddles the rule's edge
    lc = E.lens_cases()
    assert lc["linear_valid"]["valid"].all() and not lc["linear_singular"]["valid"].any()


def test_budgets_are_small(sweep):
    sw, arr, tr = sweep
    pd = tr["pix_dec"]
    rel = tr["B_col"][pd] / tr["col"][pd].abs().clamp_min(1e-2)
    assert float(rel.median()) < 1e-5 and float(tr["B_alpha"][pd].median()) < 1e-5
    dec = tr["pair_dec"] & tr["ev"]["use"]
    assert float((tr["B_raw"][dec] / tr["ev"]["raw"][dec]).median()) < 3e-5
    for name, b in tr["B_grads"].items():
        g = tr["grads"][name]
        assert float((b / g.abs().clamp_min(1e-6)).median()) < 1e-3, name
