"""The SH colour kernels on the adversarial sweep of tests/sh_edges.py, against its float64 truth.

* fused_project_sh, C = 1 and the three camera pairs (both ONE_CAM instantiations), with and without the row records:
  colours within budget on every decided entry, 0 below the kink and at exact ties; the rgb word of the row record is
  the colour; the colours equal spherical_harmonics followed by clamp_min bit for bit.
* Its backward under a colour cotangent alone: v_quats and v_scales exactly 0, v_sh and v_means (the SH term alone)
  within budget on every decided row, the gradient passing at exact ties; every entry written (NaN-filled gradient
  buffers), v_sh beyond (degree + 1)^2 exactly 0.
* spherical_harmonics (dense, masked, batch dims [2]) and spherical_harmonics_rows for D in {1, 3, 4, 32} under cameras
  off the origin: colours, v_coeffs, v_means and v_viewmats (through the per-image direction sums).
* rasterization() + l1_loss on the black-initialised garden: the fused path, packed=True and pose gradients give the
  same v_sh, and every visible tied channel gets a gradient on all three.
* Quaternions and SH coefficients at a 4-byte offset in their buffer give what their aligned copies give.
"""
import numpy as np
import pytest
import torch

from tests import scene
from tests import sh_edges as se

pytestmark = pytest.mark.gpu
dev = "cuda"
f32 = np.float32
IDS = [f"deg{d}-K{K}" for d, K in se.GRID]
CAMS = [(0,)] + list(se.PAIRS)


@pytest.fixture(scope="module")
def gs():
    import gsplat_b200

    return gsplat_b200


@pytest.fixture(scope="module", params=se.GRID, ids=IDS)
def case(request):
    deg, K = request.param
    return deg, se.make_rows(deg, K)


def _t(a, grad=False):
    return torch.tensor(np.ascontiguousarray(a), device=dev).requires_grad_(grad)


def _n(t):
    return t.detach().cpu().double().numpy()


def _nan_allocator(name, like):
    return None if like is None else torch.full_like(like, float("nan"))


@pytest.mark.parametrize("ids", CAMS, ids=lambda v: "cams" + "".join(map(str, v)))
def test_fused_tie_and_kink_vs_truth(gs, case, ids):
    deg, rows = case
    vm, Ks = se.cameras(ids)
    C, N = len(ids), se.N_ROWS
    P = {k: _t(rows[k], k in ("means", "quats", "scales", "coeffs")) for k in ("means", "quats", "scales", "opacities", "coeffs")}
    args = (P["means"], P["quats"], P["scales"], P["opacities"], P["coeffs"], _t(vm), _t(Ks), se.W, se.H, deg)
    ro = gs.ops.RowSideOutputs(16, se.W // 16, se.H // 16)
    outs = [gs.fused_project_sh(*args, rows_out=ro), gs.fused_project_sh(*args)]
    radii, col = outs[0][0], outs[0][4]
    for o in outs[1:]:
        assert torch.equal(o[0], radii) and torch.equal(o[4], col)
    vis = (_n(radii) > 0).all(-1)
    assert np.array_equal(vis, se.visibility(rows, vm, Ks)), "radii vs the float32 projection"
    assert torch.equal(ro.rows[..., 12:15][radii[..., 0] > 0], col[radii[..., 0] > 0]), "row record rgb word"
    tr = se.Truth(deg, rows, vm, vis)
    got = _n(col)
    sel = tr.decided & vis[..., None]
    msgs = se.check(got, tr.colour, tr.budget, sel, "colour")
    below = sel & (tr.colour == 0)
    assert (got[below] == 0).all(), "0 below the kink and at exact ties"
    assert (got[~vis] == 0).all()
    # the same unit's standalone kernel followed by torch's clamp
    seen = radii[..., 0] > 0
    ref = torch.clamp_min(gs.spherical_harmonics(deg, P["means"].detach(), _t(vm), P["coeffs"].detach()) + 0.5, 0.0)
    ndiff = int((ref[seen] != col[seen]).sum())
    assert ndiff == 0, f"{ndiff} colours differ from spherical_harmonics + clamp_min, max {float((ref - col)[seen].abs().max()):.3e}"
    # backward: a colour cotangent alone
    cot = np.random.RandomState(3).standard_normal((C, N, 3)).astype(f32)
    gs.ops.set_gradient_allocator(_nan_allocator)
    try:
        gm, gq, gsc, gsh = torch.autograd.grad((col * _t(cot)).sum(), (P["means"], P["quats"], P["scales"], P["coeffs"]))
    finally:
        gs.ops.set_gradient_allocator(None)
    for g, name in ((gm, "v_means"), (gq, "v_quats"), (gsc, "v_scales"), (gsh, "v_sh")):
        assert not torch.isnan(g).any(), f"{name}: {int(torch.isnan(g).sum())} entries never written"
    assert (gq == 0).all() and (gsc == 0).all()
    nb = (deg + 1) ** 2
    assert (gsh[:, nb:] == 0).all()
    (r_sh, r_m), (b_sh, b_m) = tr.grads(cot)
    rd = tr.row_decided()
    msgs += se.check(_n(gsh), r_sh, b_sh, np.broadcast_to(rd[:, None, :], r_sh.shape), "v_sh")
    msgs += se.check(_n(gm), r_m, b_m, np.broadcast_to(rd.all(-1)[:, None], r_m.shape), "v_means")
    # the clamp passes the gradient at exact ties: every visible tied channel's v_sh[:, 0] is the cotangent's sum times Y0
    tie = tr.tie.any(0)
    assert tie.sum() >= 100
    v0 = _n(gsh)[:, 0, :]
    y0sum = (cot.astype(np.float64) * vis[..., None]).sum(0) * se.SH_C0
    assert np.allclose(v0[tie], y0sum[tie], rtol=1e-5, atol=1e-6), "v_sh of tied channels"
    assert (np.abs(v0[tie]) > 0).mean() > 0.99
    assert not msgs, "\n".join(msgs)


@pytest.mark.parametrize("D", [1, 3, 4, 32])
@pytest.mark.parametrize("deg", [0, 1, 3, 4])
def test_standalone_sh_vs_truth(gs, deg, D):
    """dense (masked, batch dims [2]) and row SH kernels under cameras off the origin; N * D is not a multiple of 32"""
    K = 25 if deg == 4 else 16
    rows = se.make_rows(deg, K)
    N = se.N_ROWS
    vm2, _ = se.cameras((0, 1), se.OFFSET_CENTRES)
    vm = np.stack([vm2, vm2[::-1]])  # batch [2]: the second element sees through the cameras in the other order
    means = np.stack([rows["means"], rows["means"] * f32(0.5)])
    reps = (D + 2) // 3
    coeffs = np.concatenate([rows["coeffs"] * f32(2.0**i) for i in range(reps)], -1)[..., :D]  # exact scalings
    masks = np.random.RandomState(D).random_sample((2, 2, N)) < 0.7
    tr = se.Truth(deg, dict(rows, coeffs=coeffs), vm, masks, coeffs=coeffs, means=means)
    cot = np.random.RandomState(5).standard_normal((2, 2, N, D)).astype(f32)
    (r_c, r_m), (b_c, b_m) = tr.grads(cot, clamp=False)
    tm, tvm, tc = _t(means, True), _t(vm, True), _t(coeffs, True)
    out = gs.spherical_harmonics(deg, tm, tvm, tc, masks=_t(masks))
    msgs = se.check(_n(out), np.where(masks[..., None], tr.x, 0.0), np.where(masks[..., None], tr.budget, 0.0),
                    np.ones(tr.x.shape, bool), "dense colour")
    gm, gv, gc = torch.autograd.grad((out * _t(cot)).sum(), (tm, tvm, tc))
    msgs += se.check(_n(gc), r_c, b_c, np.ones(r_c.shape, bool), "dense v_coeffs")
    msgs += se.check(_n(gm), r_m, b_m, np.ones(r_m.shape, bool), "dense v_means")
    # v_viewmats = (t S^T | R S) with S the image's sum of view-direction gradients; S from the truth per image
    from oracle import gso

    ref_v = np.zeros((2, 2, 4, 4))
    tol_v = np.zeros((2, 2, 4, 4))
    for b in range(2):
        for c in range(2):
            vcol = cot[b, c : c + 1].astype(np.float64) * masks[b, c : c + 1, :, None]
            _, vd = gso.spherical_harmonics_bwd(deg, means[b].astype(np.float64), vm[b, c : c + 1].astype(np.float64),
                                                coeffs.astype(np.float64), masks[b, c : c + 1], vcol)
            terms = se.dir_grad_terms(deg, means[b], vm[b, c : c + 1], coeffs, vcol)[0]
            S, Sabs = vd.sum(0), np.abs(vd).sum(0) + (deg + 1) ** 2 * terms.sum()
            R, t = vm[b, c, :3, :3].astype(np.float64), vm[b, c, :3, 3].astype(np.float64)
            ref_v[b, c, :3, :3], ref_v[b, c, :3, 3] = t[:, None] * S[None], R @ S
            # float32 atomics over ceil(N * D / 32) warps, plus the per-row budgets
            tol_v[b, c, :3, :3] = np.abs(t)[:, None] * Sabs[None]
            tol_v[b, c, :3, 3] = np.abs(R) @ Sabs
    tol_v = 512 * se.ULP * tol_v
    msgs += se.check(_n(gv), ref_v, tol_v, np.ones(ref_v.shape, bool), "dense v_viewmats")
    # packed rows of the same masks
    b_ids, c_ids, g_ids = (torch.tensor(x, device=dev) for x in np.nonzero(masks))
    tm2, tvm2, tc2 = _t(means, True), _t(vm, True), _t(coeffs, True)
    rows_out = gs.ops.spherical_harmonics_rows(deg, tm2, tvm2, tc2, b_ids, c_ids, g_ids)
    assert torch.equal(rows_out, out.detach()[masks]), "rows == dense on the same rows"
    gm2, gv2, gc2 = torch.autograd.grad((rows_out * _t(cot[masks])).sum(), (tm2, tvm2, tc2))
    msgs += se.check(_n(gc2), r_c, b_c + 4 * se.ULP * np.abs(r_c), np.ones(r_c.shape, bool), "rows v_coeffs")
    msgs += se.check(_n(gm2), r_m, b_m, np.ones(r_m.shape, bool), "rows v_means")
    msgs += se.check(_n(gv2), ref_v, tol_v, np.ones(ref_v.shape, bool), "rows v_viewmats")
    assert not msgs, "\n".join(msgs)


@pytest.mark.parametrize("sh_degree", [0, 3])
def test_paths_agree_on_black_garden(gs, sh_degree):
    """Every channel of the garden initialised black (sh0 = (0 - 0.5) / C0, higher bands 0) sits exactly on the kink.
    The fused path, packed=True and the pose-gradient path must pass the gradient there alike (as torch.clamp_min does):
    the same v_sh within 1e-4 relative L2 (compositing sums its gradient with float atomics), and a non-zero gradient
    for every channel of every Gaussian with a non-zero colour gradient."""
    sc = scene.make_scene(n_max=30000, sh_degree=3)
    K = (sh_degree + 1) ** 2
    sh = np.zeros((sc["means"].shape[0], K, 3), f32)
    sh[:, 0, :] = (np.zeros_like(sc["colors"]) - f32(0.5)) / scene.SH_C0
    W, H = 256, 192
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:2]
    P = {k: _t(sc[k]) for k in ("means", "quats", "scales", "opacities")}
    target = torch.rand((2, H, W, 3), device=dev, generator=torch.Generator(dev).manual_seed(0))
    grads = {}
    for path in ("fused", "packed", "pose"):
        coeffs = _t(sh, True)
        rc, _, meta = gs.rasterization(P["means"], P["quats"], P["scales"], P["opacities"], coeffs,
                                       _t(sc["viewmats"][:2], path == "pose"), _t(Ks), W, H, sh_degree=sh_degree,
                                       packed=path == "packed")
        assert (rc == 0).all(), "black Gaussians on a black background"
        gs.l1_loss(rc, target).backward()
        grads[path] = coeffs.grad
        if path == "fused":
            vis = (meta["radii"] > 0).all(-1).any(0)
    g = grads["fused"]
    assert vis.sum() > 1000
    seen = vis & (g[:, 0].abs() > 0).any(-1)
    assert seen.sum() > 0.9 * vis.sum(), f"only {int(seen.sum())} of {int(vis.sum())} visible Gaussians get a gradient"
    for path in ("packed", "pose"):
        rel = float((grads[path] - g).norm() / g.norm())
        assert rel < 1e-4, f"{path} vs fused v_sh: relative L2 {rel:.3e}"
        assert ((grads[path][:, 0].abs() > 0) == (g[:, 0].abs() > 0)).float().mean() > 0.999
    assert (g[seen][:, 0] != 0).all(), "every channel of a Gaussian with a colour gradient"


@pytest.mark.parametrize("C", [1, 2])
def test_offset_views_equal_aligned_copies(gs, C):
    """quats and SH coefficients carved at a 4-byte offset from flat buffers (contiguous views, 4-byte aligned) render
    and differentiate exactly like their aligned copies"""
    a = 1 << 20  # never dereferenced: an empty call returns before any CUDA call
    if gs._cabi.lib().gsb200_project_sh_fwd(1, 0, 1, 0, a, a + 4, a, a, a, a, a, 16, 16, 0.3, 0.01, 1e10, 0.0, 0, a, a, a,
                                            a, None, a, None) != -1:
        pytest.skip("this library does not check the alignment of its 128-bit accesses")
    deg, K = 3, 16
    rows = se.make_rows(deg, K)
    N = se.N_ROWS
    vm, Ks = se.cameras((0,) if C == 1 else se.PAIRS[0])
    q_flat, sh_flat = torch.zeros(N * 4 + 1, device=dev), torch.zeros(N * K * 3 + 1, device=dev)
    q_flat[1:] = _t(rows["quats"]).reshape(-1)
    sh_flat[1:] = _t(rows["coeffs"]).reshape(-1)
    outs = []
    for aligned in (True, False):
        q = q_flat[1:].view(N, 4)
        sh = sh_flat[1:].view(N, K, 3)
        assert q.is_contiguous() and q.data_ptr() % 16 == 4
        if aligned:
            q, sh = q.clone(), sh.clone()
        q.requires_grad_(True)
        sh.requires_grad_(True)
        m = _t(rows["means"], True)
        o = gs.fused_project_sh(m, q, _t(rows["scales"]), _t(rows["opacities"]), sh, _t(vm), _t(Ks), se.W, se.H, deg)
        cot = torch.randn(o[4].shape, device=dev, generator=torch.Generator(dev).manual_seed(1))
        grads = torch.autograd.grad((o[4] * cot).sum() + o[1].sum(), (m, q, sh))
        outs.append((o[0], o[1], o[4]) + grads)
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
