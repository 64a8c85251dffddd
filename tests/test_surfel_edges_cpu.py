"""The 2DGS sweep of tests/surfel_edges.py checks itself without a GPU: every projection class is present and mostly
decided, oracle/surfel.py run in float32 (the kernels' stand-in) agrees with the float64 truth within the budgets on
every decided row, forward and backward, the exact-tie compositing images tie in float32, and the oracle culls the rows
whose ray transform is beyond float32's range."""
import numpy as np
import pytest
import torch

from oracle import surfel
from tests import surfel_edges as se

# undecided shares per class under camera 0, whose frame the rows are built in (the sweep meets them with a margin of
# about 0.1): ceil, cosv, near / far, off-screen and radius_clip rows sit at their thresholds on purpose, a quarter to
# a half of them inside the budget; dist ~ 0 rows at 1e-2 of dist's terms have radii of 1e4 pixels and more, whose
# float32 ceil is uncertain
MAX_UNDECIDED = {"ceil": 0.55, "cosv": 0.5, "dist~0": 0.55, "far": 0.5, "near": 0.5, "offscreen": 0.6, "radius_clip": 0.55}


@pytest.fixture(scope="module")
def rows():
    return se.make_rows()


def test_classes_present_and_mostly_decided(rows):
    tr = se.truth(rows, 1)
    rep = se.undecided_report(tr)
    print("\ncamera 0 (rows, undecided, rows):", rep)
    for cls, m in se.CLASS_MIN.items():
        assert rep[cls][0] >= m, (cls, rep[cls])
        assert rep[cls][1] <= MAX_UNDECIDED.get(cls, 0.25) * rep[cls][2], (cls, rep[cls])
    # the floor rows reach the GPU: decided and visible, most of them on the 1e-4 floor in one axis or both
    fl = (tr.cls == "floor") & tr.decided[0] & tr.vis[0]
    floored = tr.q["ext"][0] < se.FLOOR
    print("floor rows decided and visible:", int(fl.sum()), "floored on one axis:", int((fl & floored.any(-1)).sum()),
          "on both:", int((fl & floored.all(-1)).sum()))
    assert fl.sum() >= 12 and (fl & floored.any(-1)).sum() >= 10 and (fl & floored.all(-1)).sum() >= 5
    assert ((tr.cls == "dist==0") & tr.decided[0] & ~tr.vis[0]).sum() >= 8
    tr2 = se.truth(rows, 2)
    print("C = 2 (rows, undecided pairs, pairs):", se.undecided_report(tr2))
    assert tr2.decided.mean() > 0.6  # camera 1 sees rows built for camera 0's thresholds: 0.69


@pytest.mark.parametrize("C,clip", [(1, 0.0), (2, 0.0), (1, se.RCLIP)])
def test_float32_oracle_within_budgets(rows, C, clip):
    tr = se.truth(rows, C, clip)
    vm, Ks = se.camera_arrays(C)
    out = [o.numpy() for o in surfel.project(*(torch.tensor(v) for v in (rows["means"], rows["quats"], rows["scales"], vm, Ks)),
                                             se.W, se.H, se.NEAR, se.FAR, clip)]
    # torch's float -> int32 conversion does not saturate (the kernels' cvt.rzi.s32.f32 does)
    out[0] = np.where(out[0] == np.iinfo(np.int32).min, se.INT32_MAX, out[0])
    msgs = se.check_projection(rows, tr, *out, what=f"float32 oracle C={C} clip={clip}")
    assert not msgs, "\n".join(msgs)
    if clip:
        cl = (tr.cls == "radius_clip")[None] & tr.decided
        assert ((tr.radii[cl] == clip).all(-1) | (tr.radii[cl] == 0).all(-1)).any(), "no row with radius == radius_clip"


def test_float32_oracle_backward_within_budgets(rows):
    C = 2
    tr = se.truth(rows, C)
    ref, beta, cot = se.grad_truth(rows, tr, 0.0, se.cotangents((C, rows["means"].shape[0])))
    vm, Ks = se.camera_arrays(C)
    leaves = [torch.tensor(v, requires_grad=True) for v in (rows["means"], rows["quats"], rows["scales"], vm)]
    out = surfel.project(*leaves, torch.tensor(Ks), se.W, se.H, se.NEAR, se.FAR)
    loss = sum((o * torch.tensor(cot[k])).sum() for o, k in zip(out[1:], ("means2d", "depths", "ray_transforms", "normals")))
    g = torch.autograd.grad(loss, leaves)
    got = dict(v_means=g[0].numpy(), v_quats=g[1].numpy(), v_scales=g[2].numpy(), v_viewmats=g[3].numpy())
    msgs = se.check_grads(rows, tr, got, ref, beta, "float32 oracle")
    assert not msgs, "\n".join(msgs)


def test_tie_images_tie_in_float32():
    ti = se.tie_images()
    for dt in (torch.float32, torch.float64):
        m2 = torch.tensor(ti["means2d"][0, 0], dtype=dt)
        rt = torch.tensor(ti["ray_transforms"][0, 0], dtype=dt)
        px = torch.arange(se.IW, dtype=dt) + 0.5
        py = torch.arange(se.IH, dtype=dt) + 0.5
        py, px = torch.meshgrid(py, px, indexing="ij")
        hu = px[..., None] * rt[2] - rt[0]
        hv = py[..., None] * rt[2] - rt[1]
        s = torch.linalg.cross(hu, hv, dim=-1)
        g3 = (s[..., 0] / s[..., 2]) ** 2 + (s[..., 1] / s[..., 2]) ** 2
        g2 = 2.0 * ((m2[0] - px) ** 2 + (m2[1] - py) ** 2)
        assert torch.equal(g3, g2), dt
    last, T = se.stop_chain_float32()
    f = np.float32
    assert last == 3 and f(T * f(f(1) - f(se.STOP_OPACITIES[4]))) == f(se.T_TH)
    assert f(1) - f(0.5) == f(0.5)
    # the clamp image: raw alpha above 0.99 at the farthest pixel
    u = (np.array([se.IW, se.IH]) / 1024.0) ** 2
    assert np.exp(-0.5 * u.sum()) > se.MAX_ALPHA
    # the filter image: g2 < g3 at every pixel (no pixel centre on the surfel's centre, where both are 0)
    m2, rt = ti["means2d"][4, 0].astype(np.float64), ti["ray_transforms"][4, 0].astype(np.float64)
    d = np.stack(np.meshgrid(np.arange(se.IW) + 0.5, np.arange(se.IH) + 0.5), -1) - m2
    uv = d @ np.linalg.inv(rt[:2, :2]).T
    assert ((uv**2).sum(-1) > 2.0 * (d**2).sum(-1)).all()


def test_oracle_culls_float32_overflow():
    ov = se.overflow_rows()
    vm, Ks = se.camera_arrays(1)
    args = [torch.tensor(v) for v in (ov["means"], ov["quats"], ov["scales"], vm, Ks)]
    with np.errstate(all="ignore"):
        r64 = surfel.project(*(a.double() for a in args), se.W, se.H, se.NEAR, se.FAR)
    assert (r64[0] == 0).all(), "the oracle culls rows beyond float32's range"
    with np.errstate(all="ignore"):
        M = surfel.project(*(a.double() for a in args[:2]), args[2].double() * 1e-30, *(a.double() for a in args[3:]), se.W, se.H)[3]
    assert (M != 0).any(), "the same rows at ordinary scales are visible"
