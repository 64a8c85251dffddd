"""The SH sweep of tests/sh_edges.py checks itself without a GPU: its premises hold (the tie rows tie in float32, the
kink rows sit on their intended side, every signed axis is seen exactly, warps mix seen and unseen rows), the float32
oracle (the kernels' stand-in) stays within the budgets on every decided entry, forward and backward, and most entries
are decided.  The fused SH entry points reject misaligned quaternion and SH pointers before any CUDA call."""
import numpy as np
import pytest
import torch

from oracle import gso
from tests import sh_edges as se

f32 = np.float32
# undecided entries per class: the kink rows sit 1e-7 to 1e-2 of their terms from the kink on purpose (about a quarter
# are inside the budget); the cancelling rows carry terms up to 1e5 around a colour of order 1 (15 % undecided at
# degree 4)
MAX_UNDECIDED = {"kink": 0.4, "cancel": 0.25}
CAMS = [(0,)] + list(se.PAIRS)


@pytest.fixture(scope="module", params=se.GRID, ids=[f"deg{d}-K{K}" for d, K in se.GRID])
def case(request):
    deg, K = request.param
    return deg, se.make_rows(deg, K)


def test_premises(case):
    deg, rows = case
    N, cls, c = se.N_ROWS, rows["cls"], rows["coeffs"]
    assert rows["means"].shape[0] == N and N % 32 != 0
    # ties: black channels of the trainer's initialisation, x = Y0 c0 == -0.5 exactly in float32 (the higher bands are 0)
    t = rows["tie"]
    assert t.sum() >= 300 and (t.all(-1) & (cls == "tie")).sum() >= 150 and (t.any(-1) & ~t.all(-1)).sum() >= 50
    assert (f32(se.SH_C0) * c[:, 0][t] == f32(-0.5)).all()
    assert (c[:, 1 : (deg + 1) ** 2][np.broadcast_to(t[:, None], c[:, 1 : (deg + 1) ** 2].shape)] == 0).all()
    vm, _ = se.cameras((0,))
    x32 = gso.spherical_harmonics(deg, rows["means"], vm, c)[0]
    assert (x32[t] + f32(0.5) == 0).all(), "the float32 oracle ties"
    # kink rows: float64 x + 0.5 on the intended side
    x64 = gso.spherical_harmonics(deg, rows["means"].astype(np.float64), vm.astype(np.float64), c.astype(np.float64))[0]
    k = rows["side"] != 0
    assert k.sum() >= 2000 and (np.sign(x64[k] + 0.5) == rows["side"][k]).all()
    # exact axis rows: one non-zero component; each signed axis is the optical axis of a camera that sees a row on it
    ax = cls == "axis"
    assert ((rows["means"][ax] != 0).sum(-1) == 1).all()
    for i, name in enumerate(se.AXES):
        j, sgn = "xyz".index(name[1]), 1.0 if name[0] == "+" else -1.0
        on = ax & (np.sign(rows["means"][:, j]) == sgn)
        vm1, Ks1 = se.cameras((i,))
        assert (se.visibility(rows, vm1, Ks1)[0] & on).sum() >= 10, name
    for ids in se.PAIRS:
        vis = se.visibility(rows, *se.cameras(ids))
        both, one, none = vis.all(0), vis.sum(0) == 1, ~vis.any(0)
        assert both.sum() >= 200 and one.sum() >= 1000 and none.sum() >= 1000, ids
        seen = vis.any(0)[: N // 32 * 32].reshape(-1, 32)
        assert (seen.any(-1) & ~seen.all(-1)).mean() > 0.9, "warps mix seen and unseen rows"
        assert seen.any() and vis.any(0)[N // 32 * 32 :].any(), "the partial last warp has a seen row"


@pytest.mark.parametrize("ids", CAMS, ids=lambda v: "cams" + "".join(map(str, v)))
def test_mostly_decided(case, ids):
    deg, rows = case
    vm, Ks = se.cameras(ids)
    tr = se.Truth(deg, rows, vm, se.visibility(rows, vm, Ks))
    rep = se.undecided_report(tr, rows["cls"])
    print(f"\ndegree {deg} cameras {ids} (visible entries, undecided):", rep)
    for c, (n, u) in rep.items():
        assert n >= 100, (c, n)
        assert u <= MAX_UNDECIDED.get(c, 0.0) * n, (c, n, u)


def _oracle32_vs_truth(deg, rows, vm, vis, clamp):
    tr = se.Truth(deg, rows, vm, vis)
    x32 = gso.spherical_harmonics(deg, rows["means"], vm, rows["coeffs"], vis).astype(np.float64)
    sel = tr.decided & vis[..., None]
    msgs = []
    if clamp:
        col32 = np.maximum(x32 + 0.5, 0.0)
        msgs += se.check(col32, tr.colour, tr.budget, sel, "colour")
    else:
        msgs += se.check(x32, tr.x, tr.budget, vis[..., None] & np.ones_like(sel), "x")
    cot = np.random.RandomState(3).standard_normal(tr.x.shape).astype(f32)
    ref, (b_sh, b_m) = tr.grads(cot, clamp)
    v_col = cot * vis[..., None] * (((x32 + 0.5) >= 0) if clamp else 1.0)
    g_sh, g_m = gso.spherical_harmonics_bwd(deg, rows["means"], vm, rows["coeffs"], vis, v_col.astype(f32))
    rd = tr.row_decided() if clamp else np.ones(tr.x.shape[-2:], bool)
    msgs += se.check(g_sh, ref[0], b_sh, np.broadcast_to(rd[:, None, :], g_sh.shape), "v_sh")
    msgs += se.check(g_m, ref[1], b_m, np.broadcast_to(rd.all(-1)[:, None], g_m.shape), "v_means")
    return msgs


@pytest.mark.parametrize("ids", CAMS, ids=lambda v: "cams" + "".join(map(str, v)))
def test_float32_oracle_within_budgets(case, ids):
    deg, rows = case
    vm, Ks = se.cameras(ids)
    msgs = _oracle32_vs_truth(deg, rows, vm, se.visibility(rows, vm, Ks), True)
    assert not msgs, "\n".join(msgs)


def test_float32_oracle_within_budgets_off_origin(case):
    """the standalone kernels' setting: cameras off the origin, every row evaluated, no clamp"""
    deg, rows = case
    vm, _ = se.cameras((0, 1), se.OFFSET_CENTRES)
    msgs = _oracle32_vs_truth(deg, rows, vm, np.ones((2, se.N_ROWS), bool), False)
    assert not msgs, "\n".join(msgs)


def test_fused_entry_points_check_alignment():
    """quats, sh_coeffs, v_quats and v_sh are moved with 128-bit accesses: a pointer that is not 16-byte aligned is
    GSB200_E_INVALID, returned before any CUDA call (before project_sh_fwd_rows clears its totals)."""
    from gsplat_b200 import _cabi

    L = _cabi.lib()
    a = 1 << 20  # never dereferenced

    def fwd(q, sh):
        return L.gsb200_project_sh_fwd(1, 4, 16, 3, a, q, a, a, sh, a, a, 16, 16, 0.3, 0.01, 1e10, 0.0, 0, a, a, a, a, None, a, None)

    def fwd_rows(q, sh):
        return L.gsb200_project_sh_fwd_rows(1, 4, 16, 3, a, q, a, a, sh, a, a, 16, 16, 0.3, 0.01, 1e10, 0.0, 16, 1, 1, a, a,
                                           a, a, a, a, a, a, None)

    def bwd(q, sh, vq=a, vsh=a):
        return L.gsb200_project_sh_bwd(1, 4, 16, 3, a, q, a, sh, a, a, 16, 16, 0.3, a, a, None, a, a, 2, a, 1, a, 3, a, 3,
                                       None, a, vq, a, vsh, None, None)

    for call in (fwd, fwd_rows, bwd):
        for off in (4, 8, 12):
            assert call(a + off, a) == -1, (call.__name__, "quats", off)
            assert call(a, a + off) == -1, (call.__name__, "sh", off)
    for off in (4, 8, 12):
        assert bwd(a, a, vq=a + off) == -1
        assert bwd(a, a, vsh=a + off) == -1


def test_gradient_allocator_alignment_is_checked():
    """a gradient segment at a 4-byte offset in its buffer is refused, not handed to the 128-bit stores"""
    from gsplat_b200 import ops

    like = torch.zeros(10, 4)
    flat = torch.zeros(41)
    try:
        ops.set_gradient_allocator(lambda name, t: flat[1:].view(10, 4) if name == "quats" else None)
        with pytest.raises(RuntimeError, match="mismatching tensor for 'quats'"):
            ops._alloc_grad("quats", like)
        ops.set_gradient_allocator(lambda name, t: flat[:40].view(10, 4))
        assert ops._alloc_grad("quats", like).data_ptr() == flat.data_ptr()
    finally:
        ops.set_gradient_allocator(None)
